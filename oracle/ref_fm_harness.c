/* ref_fm_harness.c — synchronous driver around the UNMODIFIED reference rx_fm DSP.
 *
 * TEST INFRASTRUCTURE.  Built only when /root/reference is present (oracle/Makefile,
 * target _ref/libref_fm.so).  It #includes the reference translation unit where it lies
 * (-I/root/reference/src) so that file-static items (rtlsdr_callback, atan_lut, do_exit)
 * are visible, renames its main(), and drives
 *     rtlsdr_callback()  (src/rtl_fm.c:828)   then   full_demod()  (src/rtl_fm.c:759)
 * once per chunk, exactly as the dongle/demod threads do (src/rtl_fm.c:899, :923), but
 * synchronously (SURVEY.md F12: the threaded pipeline has no back-pressure).
 * Nothing here is copied from the reference; the reference code is compiled from its own
 * files.  Only tests/, smoke() and bench.py's cpu_baseline/reference arm may load this.
 */
#define main rtl_fm_reference_main
#include "rtl_fm.c"
#undef main

#include <time.h>

typedef struct {
	int mode;             /* 0 fm, 1 am, 2 usb, 3 lsb, 4 raw            (src/rtl_fm.c:1320-1342) */
	int downsample;       /* demod.downsample                            (:142, :968-971) */
	int downsample_passes;/* demod.downsample_passes                     (:146, :970) */
	int comp_fir_size;    /* demod.comp_fir_size (-F arg)                (:147, :1307) */
	int custom_atan;      /* 0 std 1 fast 2 lut 3 ale                    (:148, :1309-1319) */
	int output_scale;     /* demod.output_scale                          (:144, :988-992) */
	int post_downsample;  /* demod.post_downsample (-o)                  (:143, :1265) */
	int deemph;           /* demod.deemph                                (:149) */
	int deemph_a;         /* demod.deemph_a                              (:1412) */
	int rate_out;         /* demod.rate_out (-s value)                   (:137, :1257) */
	int rate_out2;        /* demod.rate_out2 (-r) or -1                  (:138, :1261) */
	int squelch_level;    /* demod.squelch_level (-l)                    (:145, :1250) */
	int dc_block_audio;   /* -E adc                                      (:152, :1284) */
	int adc_block_const;  /* 9                                           (:1106) */
	int dc_block_raw;     /* -E rdc                                      (:153, :1286) */
	int rdc_block_const;  /* -q, default 9                               (:1110, :1303) */
	int offset_tuning;    /* dongle.offset_tuning: skip rotate16_90      (:118, :854) */
} ref_fm_params;

static int g_inited = 0;

static void reset_static_deemph_avg(void)
{
	/* deemph_filter keeps `static int avg` (src/rtl_fm.c:669, SURVEY F9).  One step with
	 * deemph_a == 1 and input 0 sets avg += (0-avg)/1, i.e. exactly 0. */
	int save_a = demod.deemph_a, save_len = demod.result_len;
	int16_t save0 = demod.result[0];
	demod.deemph_a = 1; demod.result_len = 1; demod.result[0] = 0;
	deemph_filter(&demod);
	demod.deemph_a = save_a; demod.result_len = save_len; demod.result[0] = save0;
}

int ref_fm_configure(const ref_fm_params *p)
{
	if (!g_inited) {
		dongle_init(&dongle);
		demod_init(&demod);
		output_init(&output);
		controller_init(&controller);
		g_inited = 1;
	}
	memset(demod.lowpassed, 0, sizeof demod.lowpassed);
	memset(demod.result, 0, sizeof demod.result);
	memset(demod.lp_i_hist, 0, sizeof demod.lp_i_hist);
	memset(demod.lp_q_hist, 0, sizeof demod.lp_q_hist);
	memset(demod.droop_i_hist, 0, sizeof demod.droop_i_hist);
	memset(demod.droop_q_hist, 0, sizeof demod.droop_q_hist);
	memset(dongle.buf16, 0, sizeof dongle.buf16);
	demod.lp_len = 0; demod.result_len = 0;
	demod.now_r = demod.now_j = demod.pre_r = demod.pre_j = 0;
	demod.prev_index = 0; demod.now_lpr = 0; demod.prev_lpr_index = 0;
	demod.dc_avg = demod.dc_avgI = demod.dc_avgQ = 0;
	demod.squelch_hits = 11; demod.conseq_squelch = 10; demod.squelch_zero = 0;
	demod.terminate_on_squelch = 0;
	switch (p->mode) {
	case 0: demod.mode_demod = &fm_demod; break;
	case 1: demod.mode_demod = &am_demod; break;
	case 2: demod.mode_demod = &usb_demod; break;
	case 3: demod.mode_demod = &lsb_demod; break;
	case 4: demod.mode_demod = &raw_demod; break;
	default: return -1;
	}
	demod.downsample = p->downsample;
	demod.downsample_passes = p->downsample_passes;
	demod.comp_fir_size = p->comp_fir_size;
	demod.custom_atan = p->custom_atan;
	demod.output_scale = p->output_scale;
	demod.post_downsample = p->post_downsample;
	demod.deemph = p->deemph;
	demod.deemph_a = p->deemph_a;
	demod.rate_in = p->rate_out * p->post_downsample;
	demod.rate_out = p->rate_out;
	demod.rate_out2 = p->rate_out2;
	demod.squelch_level = p->squelch_level;
	demod.dc_block_audio = p->dc_block_audio;
	demod.adc_block_const = p->adc_block_const;
	demod.dc_block_raw = p->dc_block_raw;
	demod.rdc_block_const = p->rdc_block_const;
	dongle.offset_tuning = p->offset_tuning;
	dongle.mute = 0;
	dongle.demod_target = &demod;
	if (p->custom_atan == 2 && !atan_lut) { atan_lut_init(); }
	reset_static_deemph_avg();
	printLevels = 0;
	do_exit = 0;
	return 0;
}

/* Runs the reference's own CLI derivation (main(): src/rtl_fm.c:1255-1258, :1305-1308,
 * :1331-1341, :1371, :1410-1415 and optimal_settings(): :960-997) and reports the derived
 * kernel parameters, so the host-side mirror in rx_tools_b200/fm.py can be checked. */
int ref_fm_derive(int mode, int rate_s, int rate_r, int use_F, int comp_fir_size, int custom_atan,
                  int post_downsample, int deemph, int time_constant_us, int wbfm_preset,
                  int offset_tuning, ref_fm_params *out, int *capture_rate, int *capture_freq_offset)
{
	ref_fm_params p0;
	memset(&p0, 0, sizeof p0);
	p0.mode = mode; p0.downsample = 1; p0.output_scale = 1; p0.post_downsample = 1;
	p0.rate_out = 24000; p0.rate_out2 = -1; p0.adc_block_const = 9; p0.rdc_block_const = 9;
	ref_fm_configure(&p0);
	demod_init(&demod);             /* CLI defaults */
	controller_init(&controller);
	switch (mode) {
	case 0: demod.mode_demod = &fm_demod; break;
	case 1: demod.mode_demod = &am_demod; break;
	case 2: demod.mode_demod = &usb_demod; break;
	case 3: demod.mode_demod = &lsb_demod; break;
	case 4: demod.mode_demod = &raw_demod; break;
	}
	if (wbfm_preset) {              /* -M wbfm, src/rtl_fm.c:1331-1341 */
		controller.wb_mode = 1;
		demod.mode_demod = &fm_demod;
		demod.rate_in = 170000; demod.rate_out = 170000; demod.rate_out2 = 32000;
		demod.custom_atan = 1; demod.deemph = 1; demod.squelch_level = 0;
	}
	if (rate_s > 0) { demod.rate_in = rate_s; demod.rate_out = rate_s; }   /* -s after -M */
	if (rate_r > 0) { demod.rate_out2 = rate_r; }
	if (use_F) { demod.downsample_passes = 1; demod.comp_fir_size = comp_fir_size; }
	if (custom_atan >= 0) { demod.custom_atan = custom_atan; }
	if (deemph >= 0) { demod.deemph = deemph; }
	demod.post_downsample = post_downsample;
	dongle.offset_tuning = offset_tuning;
	demod.rate_in *= demod.post_downsample;
	optimal_settings(100000000, demod.rate_in);
	if (demod.deemph) {
		double tc = (double)time_constant_us * 1e-6;
		demod.deemph_a = (int)round(1.0/((1.0-exp(-1.0/(demod.rate_out * tc)))));
	}
	out->mode = mode;
	out->downsample = demod.downsample;
	out->downsample_passes = demod.downsample_passes;
	out->comp_fir_size = demod.comp_fir_size;
	out->custom_atan = demod.custom_atan;
	out->output_scale = demod.output_scale;
	out->post_downsample = demod.post_downsample;
	out->deemph = demod.deemph;
	out->deemph_a = demod.deemph_a;
	out->rate_out = demod.rate_out;
	out->rate_out2 = demod.rate_out2;
	out->squelch_level = demod.squelch_level;
	out->dc_block_audio = demod.dc_block_audio;
	out->adc_block_const = demod.adc_block_const;
	out->dc_block_raw = demod.dc_block_raw;
	out->rdc_block_const = demod.rdc_block_const;
	out->offset_tuning = dongle.offset_tuning;
	*capture_rate = (int)dongle.rate;
	*capture_freq_offset = (int)((long long)dongle.freq - 100000000LL);
	return 0;
}

/* One stream, chunk by chunk.  in: interleaved CS16, n_int16 values.  chunk_int16: int16
 * count handed to rtlsdr_callback per call (<= MAXIMUM_BUF_LENGTH).  out receives the
 * concatenated demod.result[0..result_len).  per-chunk result_len / squelch_hits are
 * optional.  Returns number of int16 written to out, or -1 on overflow of out_cap. */
long ref_fm_run(const int16_t *in, size_t n_int16, size_t chunk_int16,
                int16_t *out, size_t out_cap, int *chunk_result_len, int *chunk_squelch_hits)
{
	static int16_t tmp[MAXIMUM_BUF_LENGTH];
	size_t pos = 0, w = 0, c = 0;
	if (chunk_int16 == 0 || chunk_int16 > MAXIMUM_BUF_LENGTH) { return -2; }
	while (pos < n_int16) {
		size_t len = n_int16 - pos;
		if (len > chunk_int16) { len = chunk_int16; }
		memcpy(tmp, in + pos, len * 2);          /* callback may write into buf (mute) */
		rtlsdr_callback(tmp, (uint32_t)len, &dongle);
		full_demod(&demod);
		if (w + (size_t)demod.result_len > out_cap) { return -1; }
		memcpy(out + w, demod.result, 2 * (size_t)demod.result_len);
		w += (size_t)demod.result_len;
		if (chunk_result_len) { chunk_result_len[c] = demod.result_len; }
		if (chunk_squelch_hits) { chunk_squelch_hits[c] = demod.squelch_hits; }
		pos += len; c++;
	}
	return (long)w;
}

/* Per-chunk `sr` of the -L statistics (src/rtl_fm.c:792-806): the level counters are file-scope
 * statics of the included source; with the print period pushed out of reach, levelSum grows by
 * exactly sr per full_demod() call.  Output PCM is discarded.  Returns the chunk count. */
long ref_fm_run_levels(const int16_t *in, size_t n_int16, size_t chunk_int16, int *levels)
{
	static int16_t tmp[MAXIMUM_BUF_LENGTH];
	size_t pos = 0, c = 0;
	if (chunk_int16 == 0 || chunk_int16 > MAXIMUM_BUF_LENGTH) { return -2; }
	printLevels = 1 << 30; printLevelNo = 1 << 30; levelSum = 0.0; levelMax = 0; levelMaxMax = 0;
	while (pos < n_int16) {
		size_t len = n_int16 - pos;
		double before = levelSum;
		if (len > chunk_int16) { len = chunk_int16; }
		memcpy(tmp, in + pos, len * 2);
		rtlsdr_callback(tmp, (uint32_t)len, &dongle);
		full_demod(&demod);
		levels[c] = (int)(levelSum - before);
		pos += len; c++;
	}
	printLevels = 0; printLevelNo = 1; levelSum = 0.0; levelMax = 0; levelMaxMax = 0;
	return (long)c;
}

/* Same loop, timed (for the cpu_baseline / --impl reference legs of bench.py).  rtlsdr_callback only reads
 * its buffer while dongle.mute == 0 (src/rtl_fm.c:839-843), so every chunk is handed over where it lies,
 * exactly what the dongle thread does with the readStream buffer (:894-899).  Returns seconds. */
double ref_fm_time(const int16_t *in, size_t n_int16, size_t chunk_int16, int repeats, long *n_out)
{
	struct timespec t0, t1;
	long total = 0;
	int r;
	dongle.mute = 0;
	clock_gettime(CLOCK_MONOTONIC, &t0);
	for (r = 0; r < repeats; r++) {
		size_t pos = 0;
		while (pos < n_int16) {
			size_t len = n_int16 - pos;
			if (len > chunk_int16) { len = chunk_int16; }
			rtlsdr_callback((int16_t *)(in + pos), (uint32_t)len, &dongle);
			full_demod(&demod);
			total += demod.result_len;
			pos += len;
		}
	}
	clock_gettime(CLOCK_MONOTONIC, &t1);
	if (n_out) { *n_out = total; }
	return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}

/* The reference's own discriminators over n quads (ar, aj, br, bj) of int32: form 0 polar_discriminant, 1
 * polar_disc_fast, 2 polar_disc_lut, 3 esbensen.  Quads the reference cannot evaluate -- it would crash the process --
 * are not handed to it: skipped[i] = 1 and out[i] = 0.  Those are polar_disc_lut's (cj << 8) == INT_MIN with |cr| = 1
 * (a table read at INT_MIN, or INT_MIN / -1), fast_atan2's cr == cj == INT_MIN (a division by zero) and esbensen's
 * divisors 0 and -1.  Returns the number skipped, or -1 for an unknown form. */
long ref_fm_disc_many(int form, const int32_t *quads, size_t n, int32_t *out, uint8_t *skipped)
{
	size_t i;
	long n_skip = 0;
	if (form < 0 || form > 3) { return -1; }
	if (form == 2 && !atan_lut) { atan_lut_init(); }
	for (i = 0; i < n; i++) {
		const int ar = quads[4 * i], aj = quads[4 * i + 1], br = quads[4 * i + 2], bj = quads[4 * i + 3];
		int cr, cj, bad = 0, den;
		multiply(ar, aj, br, -bj, &cr, &cj);
		if (form == 1) { bad = cr == INT32_MIN && cj == INT32_MIN; }
		if (form == 2) { bad = cr != 0 && cj != 0 && (int)((unsigned)cj << atan_lut_coef) == INT32_MIN && (cr == 1 || cr == -1); }
		if (form == 3) { den = ar * ar + aj * aj + 1; bad = den == 0 || den == -1; }
		skipped[i] = (uint8_t)bad;
		if (bad) { out[i] = 0; n_skip++; continue; }
		switch (form) {
		case 0: out[i] = polar_discriminant(ar, aj, br, bj); break;
		case 1: out[i] = polar_disc_fast(ar, aj, br, bj); break;
		case 2: out[i] = polar_disc_lut(ar, aj, br, bj); break;
		default: out[i] = esbensen(ar, aj, br, bj); break;
		}
	}
	return n_skip;
}

/* Table exports so the host-side builders can be pinned against the reference's. */
int ref_fm_atan_lut(int *dst, int n)
{
	int i;
	if (!atan_lut) { atan_lut_init(); }
	for (i = 0; i < n && i < atan_lut_size; i++) { dst[i] = atan_lut[i]; }
	return atan_lut_size;
}
int ref_fm_cic9(int row, int *dst10)
{
	int i;
	if (row < 0 || row > CIC_TABLE_MAX) { return -1; }
	for (i = 0; i < 10; i++) { dst10[i] = cic_9_tables[row][i]; }
	return 0;
}
