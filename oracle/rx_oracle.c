/* rx_oracle.c — CPU restatement ("port") of the rx_tools hot path.
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load this library; the product
 * (rx_tools_b200 / librxb200.so) never links, imports or calls it.
 *
 * It restates, in plain C and as an explicit per-stream state object (the reference keeps
 * everything in file-scope globals), the algorithm of rxseger/rx_tools @ 811b21c:
 *   rx_fm   : stream-callback DSP body  src/rtl_fm.c:844-857  +  full_demod() :759-824
 *   rx_power: scanner() per-hop body    src/rtl_power.c:709-771 (+ rms_power :403-429)
 * Every function cites the reference lines it follows.  PARITY PIN: the reference ships no
 * golden vectors or tests (SURVEY.md §4); this port is pinned against the reference code
 * itself, compiled unmodified into oracle/_ref/ (oracle/Makefile) — tests/test_oracle_pin.py
 * runs both on the same seeded inputs, and tests/golden/ holds the resulting vectors.
 *
 * Integer semantics: "int" is 32-bit two's complement with wrap (built with -fwrapv),
 * ">>" of negatives is arithmetic, stores to int16_t truncate — as on the x86 build of
 * the reference.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <time.h>

#define ORX_MAX_CHUNK 262144      /* MAXIMUM_BUF_LENGTH, src/rtl_fm.c:80-82 */
#define ORX_MAX_PASSES 10         /* lp_i_hist[10][6], src/rtl_fm.c:130 */

/* ------------------------------------------------------------------ parameters */
typedef struct {
	int mode;              /* 0 fm 1 am 2 usb 3 lsb 4 raw        src/rtl_fm.c:1320-1342 */
	int downsample;        /* boxcar length                      :142 */
	int downsample_passes; /* half-band passes (-F)              :146 */
	int comp_fir_size;     /* 9 enables the droop FIR            :147, :771 */
	int custom_atan;       /* 0 std 1 fast 2 lut 3 ale           :148 */
	int output_scale;      /* am/usb/lsb gain                    :144 */
	int post_downsample;   /* -o                                 :143 */
	int deemph;            /*                                    :149 */
	int deemph_a;          /*                                    :1412 */
	int rate_out;          /*                                    :137 */
	int rate_out2;         /* <=0 disables low_pass_real         :138, :820 */
	int squelch_level;     /*                                    :145 */
	int dc_block_audio;    /*                                    :152 */
	int adc_block_const;   /*                                    :1106 */
	int dc_block_raw;      /*                                    :153 */
	int rdc_block_const;   /*                                    :1110 */
	int offset_tuning;     /* 1: no fs/4 rotation                :118, :854 */
} orx_fm_params;

typedef struct {
	orx_fm_params p;
	/* carried state, one copy per stream (reference: struct demod_state, :128-153) */
	int box_i, box_q, box_fill;          /* now_r, now_j, prev_index */
	int16_t hb_i[ORX_MAX_PASSES][6];     /* lp_i_hist */
	int16_t hb_q[ORX_MAX_PASSES][6];     /* lp_q_hist */
	int16_t droop_i[9], droop_q[9];      /* droop_[iq]_hist */
	int last_i, last_q;                  /* pre_r, pre_j */
	int deemph_avg;                      /* static avg inside deemph_filter, :669 */
	int lpr_acc, lpr_phase;              /* now_lpr, prev_lpr_index */
	int adc_avg;                         /* dc_avg */
	int rdc_avg_i, rdc_avg_q;            /* dc_avgI, dc_avgQ */
	int squelch_hits;
	int want_levels, last_level;   /* -L: per-chunk rms kept for the caller */
	int *atan_tab;                       /* atan_lut, :91-93 */
	int16_t *iq;                         /* lowpassed[] */
	int16_t *pcm;                        /* result[] */
	int iq_len, pcm_len;                 /* lp_len, result_len (int16 counts) */
} orx_fm;

/* cic_9_tables restated: 9-tap droop-compensation coefficients, scaled 2^15, one row per
 * number of half-band passes; element 0 is the tap count (src/rtl_fm.c:287-300). */
static const int k_droop9[11][10] = {
	{0, 0, 0, 0, 0, 0, 0, 0, 0, 0},
	{9, -156,  -97, 2798, -15489, 61019, -15489, 2798,  -97, -156},
	{9, -128, -568, 5593, -24125, 74126, -24125, 5593, -568, -128},
	{9, -129, -639, 6187, -26281, 77511, -26281, 6187, -639, -129},
	{9, -122, -612, 6082, -26353, 77818, -26353, 6082, -612, -122},
	{9, -120, -602, 6015, -26269, 77757, -26269, 6015, -602, -120},
	{9, -120, -582, 5951, -26128, 77542, -26128, 5951, -582, -120},
	{9, -119, -580, 5931, -26094, 77505, -26094, 5931, -580, -119},
	{9, -119, -578, 5921, -26077, 77484, -26077, 5921, -578, -119},
	{9, -119, -577, 5917, -26067, 77473, -26067, 5917, -577, -119},
	{9, -199, -362, 5303, -25505, 77489, -25505, 5303, -362, -199},
};

int orx_droop9(int row, int *dst10)
{
	if (row < 0 || row > 10) { return -1; }
	memcpy(dst10, k_droop9[row], sizeof k_droop9[row]);
	return 0;
}

/* atan table: entry i = (int)(atan(i/256)/3.14159 * 2^14), 131072 entries
 * (atan_lut_init, src/rtl_fm.c:515-526; note 3.14159, not M_PI). */
#define ORX_ATAN_SIZE 131072
#define ORX_ATAN_COEF 8
void orx_build_atan_table(int *dst)
{
	int i;
	for (i = 0; i < ORX_ATAN_SIZE; i++) {
		dst[i] = (int)(atan((double)i / (double)(1 << ORX_ATAN_COEF)) / 3.14159 * (double)(1 << 14));
	}
}

/* deemph_a = round(1/(1-exp(-1/(rate_out*tc)))) (src/rtl_fm.c:1410-1412) */
int orx_deemph_a(int rate_out, int time_constant_us)
{
	double tc = (double)time_constant_us * 1e-6;
	return (int)round(1.0 / ((1.0 - exp(-1.0 / (rate_out * tc)))));
}

/* ------------------------------------------------------------------ rx_fm stages */

/* CS16 -> "8-bit range" squeeze done in floating point by the callback
 * (src/rtl_fm.c:845-847).  C conversion to int16_t truncates toward zero. */
int16_t orx_scale_sample(int16_t x)
{
	return (int16_t)((double)x / 32767.0 * 128.0 + 0.4);
}

/* -E rdc: per-chunk mean of I and of Q blended into a running mean, then subtracted
 * (dc_block_raw_filter, src/rtl_fm.c:699-721). */
static void raw_dc_block(orx_fm *o, int16_t *b, int len)
{
	int64_t si = 0, sq = 0;
	int k, mi, mq, w = o->p.rdc_block_const;
	for (k = 0; k < len; k += 2) { si += b[k]; sq += b[k + 1]; }
	mi = (int)(si / (len / 2));
	mq = (int)(sq / (len / 2));
	mi = (mi + o->rdc_avg_i * w) / (w + 1);
	mq = (mq + o->rdc_avg_q * w) / (w + 1);
	for (k = 0; k < len; k += 2) {
		b[k] = (int16_t)(b[k] - mi);
		b[k + 1] = (int16_t)(b[k + 1] - mq);
	}
	o->rdc_avg_i = mi;
	o->rdc_avg_q = mq;
}

/* fs/4 up-mix: complex sample n of THE CHUNK is multiplied by j^n
 * (rotate16_90, src/rtl_fm.c:309-327: groups of four pairs (I,Q),(-Q,I),(-I,-Q),(Q,-I)). */
static void quarter_rate_rotate(int16_t *b, int len)
{
	int n;
	for (n = 0; 2 * n + 1 < len; n++) {
		int16_t re = b[2 * n], im = b[2 * n + 1];
		switch (n & 3) {
		case 1: b[2 * n] = (int16_t)(-im); b[2 * n + 1] = re; break;
		case 2: b[2 * n] = (int16_t)(-re); b[2 * n + 1] = (int16_t)(-im); break;
		case 3: b[2 * n] = im; b[2 * n + 1] = (int16_t)(-re); break;
		default: break;
		}
	}
}

/* Boxcar decimator with carried phase and partial sums (low_pass, src/rtl_fm.c:351-371). */
static void boxcar_decimate(orx_fm *o)
{
	int rd, wr = 0;
	for (rd = 0; rd < o->iq_len; rd += 2) {
		o->box_i += o->iq[rd];
		o->box_q += o->iq[rd + 1];
		if (++o->box_fill < o->p.downsample) { continue; }
		o->iq[wr] = (int16_t)o->box_i;
		o->iq[wr + 1] = (int16_t)o->box_q;
		o->box_i = o->box_q = 0;
		o->box_fill = 0;
		wr += 2;
	}
	o->iq_len = wr;
}

/* One [1 5 10 10 5 1]/16 half-band pass over one component of the interleaved buffer
 * (fifth_order, src/rtl_fm.c:411-440).  x points at the component, elements are 2 apart,
 * `span` is the reference's `length` argument (an int16 count).  The six-sample window is
 * int16; the weighted sum is formed in int, shifted right 4 and stored back as int16.
 * Window at entry = h[1..5] ++ x[0]; it then advances two input samples per output while
 * 4*k < span; the final window is archived in h[0..5].  When span/2 is even the last input
 * sample of the call is never read (SURVEY F7). */
static void halfband_pass(int16_t *x, int span, int16_t h[6])
{
	int16_t w[6];
	int k;
	w[0] = h[1]; w[1] = h[2]; w[2] = h[3]; w[3] = h[4]; w[4] = h[5]; w[5] = x[0];
	x[0] = (int16_t)((w[0] + (w[1] + w[4]) * 5 + (w[2] + w[3]) * 10 + w[5]) >> 4);
	for (k = 1; 4 * k < span; k++) {
		w[0] = w[2]; w[1] = w[3]; w[2] = w[4]; w[3] = w[5];
		w[4] = x[4 * k - 2];
		w[5] = x[4 * k];
		x[2 * k] = (int16_t)((w[0] + (w[1] + w[4]) * 5 + (w[2] + w[3]) * 10 + w[5]) >> 4);
	}
	memcpy(h, w, sizeof w);
}

/* 9-tap symmetric droop FIR over the PREVIOUS nine samples of one component
 * (generic_fir, src/rtl_fm.c:442-465); the current input only enters the history. */
static void droop_fir9(int16_t *x, int span, const int *c, int16_t h[9])
{
	int d;
	for (d = 0; d < span; d += 2) {
		int16_t in = x[d];
		int acc = (h[0] + h[8]) * c[1] + (h[1] + h[7]) * c[2] + (h[2] + h[6]) * c[3]
		        + (h[3] + h[5]) * c[4] + h[4] * c[5];
		x[d] = (int16_t)(acc >> 15);
		memmove(h, h + 1, 8 * sizeof h[0]);
		h[8] = in;
	}
}

/* rms of a buffer with the DC term removed in floating point (rms, src/rtl_fm.c:739-757). */
static int buffer_rms(const int16_t *s, int len, int step)
{
	long sum = 0, sq = 0;
	double dc, err;
	int k;
	for (k = 0; k < len; k += step) { long v = s[k]; sum += v; sq += v * v; }
	dc = (double)(sum * step) / (double)len;
	err = sum * 2 * dc - dc * dc * len;
	return (int)sqrt((sq - err) / len);
}

/* x[n] * conj(x[n-1]) (multiply with negated bj, src/rtl_fm.c:470-474, :480). */
static void conj_product(int ar, int aj, int br, int bj, int *cr, int *cj)
{
	*cr = ar * br - aj * (-bj);
	*cj = aj * br + ar * (-bj);
}

/* polar_discriminant, src/rtl_fm.c:476-483 */
int orx_disc_std(int ar, int aj, int br, int bj)
{
	int cr, cj;
	conj_product(ar, aj, br, bj, &cr, &cj);
	return (int)(atan2((double)cj, (double)cr) / 3.14159 * (double)(1 << 14));
}

/* polar_discriminant, and *near = 1 when its value v = atan2(cj, cr) / 3.14159 * 2^14 (glibc) lies within 2^-30 of an
 * integer: the
 * only operands where an atan2 that differs from glibc's in the last few ulps (CUDA's: |v| < 2^14, so a few ulps of
 * atan2 move v by < 2^-35) can truncate to a different integer.  atan2(0, x >= 0) is exactly +0 in every libm and does not count. */
static int disc_std_near(int ar, int aj, int br, int bj, int *near)
{
	int cr, cj;
	double v;
	conj_product(ar, aj, br, bj, &cr, &cj);
	v = atan2((double)cj, (double)cr) / 3.14159 * (double)(1 << 14);
	*near = !(cj == 0 && cr >= 0) && fabs(v - rint(v)) < 0x1p-30;
	return (int)v;
}

/* polar_discriminant evaluations of chain runs (fm_discriminate: -A std samples and every chunk's first sample) that
 * were near an integer, since the last orx_std_near_count() */
static long g_std_near = 0;
static int disc_std_counted(int ar, int aj, int br, int bj)
{
	int near, v = disc_std_near(ar, aj, br, bj, &near);
	g_std_near += near;
	return v;
}
long orx_std_near_count(void)
{
	long c = g_std_near;
	g_std_near = 0;
	return c;
}

/* fast_atan2 + polar_disc_fast, src/rtl_fm.c:485-513.  pi == 1<<14. */
int orx_fast_atan2(int y, int x)
{
	const int q1 = 1 << 12, q3 = 3 * (1 << 12);
	int ya = y < 0 ? -y : y, ang;
	if (x == 0 && y == 0) { return 0; }
	if (x >= 0) { ang = q1 - q1 * (x - ya) / (x + ya); }
	else        { ang = q3 - q1 * (x + ya) / (ya - x); }
	return y < 0 ? -ang : ang;
}
int orx_disc_fast(int ar, int aj, int br, int bj)
{
	int cr, cj;
	conj_product(ar, aj, br, bj, &cr, &cj);
	return orx_fast_atan2(cj, cr);
}

/* polar_disc_lut, src/rtl_fm.c:528-564.  One deviation: where (cj << 8) is INT_MIN and |cr| = 1 the reference reads
 * atan_lut[INT_MIN] (cr = 1) or divides INT_MIN by -1 (cr = -1) and crashes; here, as in the library, the quotient
 * INT_MIN takes the linear-range branch (include/rxb200.h, RXB200_ATAN_LUT). */
int orx_disc_lut(const int *tab, int ar, int aj, int br, int bj)
{
	int cr, cj, q, qa, num;
	conj_product(ar, aj, br, bj, &cr, &cj);
	if (cr == 0 || cj == 0) {
		if (cr == 0 && cj == 0) { return 0; }
		if (cr == 0) { return cj > 0 ? (1 << 13) : -(1 << 13); }
		return cr > 0 ? 0 : (1 << 14);
	}
	num = (int)((unsigned)cj << ORX_ATAN_COEF);
	if (num == INT32_MIN && (cr == 1 || cr == -1)) { return cj > 0 ? (1 << 13) : -(1 << 13); }
	q = num / cr;
	qa = q < 0 ? -q : q;
	if (qa >= ORX_ATAN_SIZE) { return cj > 0 ? (1 << 13) : -(1 << 13); }
	if (q > 0) { return cj > 0 ? tab[q] : tab[q] - (1 << 14); }
	return cj > 0 ? (1 << 14) - tab[-q] : -tab[-q];
}

/* esbensen, src/rtl_fm.c:566-582 */
int orx_disc_ale(int ar, int aj, int br, int bj)
{
	int dr = (br - ar) * 2, dj = (bj - aj) * 2;
	int cj = bj * dr - br * dj;
	return 2608 * cj / (ar * ar + aj * aj + 1);
}

/* n quads (ar, aj, br, bj) of int32 through one discriminator, numbered as rxb200_fm_disc_device's forms: 0 std, 1 fast,
 * 2 lut (tab: the atan table), 3 ale, 4 atan2 and 5 the fp64 form (both polar_discriminant here), 6 and 7 the int16 that
 * the row and stream front ends store (fast_atan2's, stored), 8 the AM envelope (int16)sqrt(ar^2 + aj^2).  near (may
 * be NULL) receives disc_std_near()'s flag for every quad.  Returns 0, or -1 for an unknown form. */
int orx_disc_many(int form, const int32_t *quads, size_t n, const int *tab, int32_t *out, uint8_t *near)
{
	size_t i;
	if (form < 0 || form > 8 || (form == 2 && !tab)) { return -1; }
	for (i = 0; i < n; i++) {
		const int ar = quads[4 * i], aj = quads[4 * i + 1], br = quads[4 * i + 2], bj = quads[4 * i + 3];
		int v;
		switch (form) {
		case 1: v = orx_disc_fast(ar, aj, br, bj); break;
		case 2: v = orx_disc_lut(tab, ar, aj, br, bj); break;
		case 3: v = orx_disc_ale(ar, aj, br, bj); break;
		case 6: case 7: v = (int16_t)orx_disc_fast(ar, aj, br, bj); break;
		case 8: v = (int16_t)sqrt(ar * ar + aj * aj); break;      /* am_demod, src/rtl_fm.c:617-632 */
		default: v = orx_disc_std(ar, aj, br, bj); break;
		}
		out[i] = v;
		if (near) {
			int f;
			disc_std_near(ar, aj, br, bj, &f);
			near[i] = (uint8_t)f;
		}
	}
	return 0;
}

/* fm_demod, src/rtl_fm.c:584-615: first output of every chunk uses the atan2 path whatever
 * the selected mode (SURVEY F8). */
static void fm_discriminate(orx_fm *o)
{
	const int16_t *lp = o->iq;
	int k, v = 0;
	o->pcm[0] = (int16_t)disc_std_counted(lp[0], lp[1], o->last_i, o->last_q);
	for (k = 2; k < o->iq_len - 1; k += 2) {
		switch (o->p.custom_atan) {
		case 0: v = disc_std_counted(lp[k], lp[k + 1], lp[k - 2], lp[k - 1]); break;
		case 1: v = orx_disc_fast(lp[k], lp[k + 1], lp[k - 2], lp[k - 1]); break;
		case 2: v = orx_disc_lut(o->atan_tab, lp[k], lp[k + 1], lp[k - 2], lp[k - 1]); break;
		case 3: v = orx_disc_ale(lp[k], lp[k + 1], lp[k - 2], lp[k - 1]); break;
		}
		o->pcm[k / 2] = (int16_t)v;
	}
	if (o->iq_len == 0) {
		/* A chunk that completes no boxcar: :612-613 read lowpassed[-2], lowpassed[-1], the high half of
		 * struct demod_state's `thread` (:126-127).  The reference harness never starts that thread, so both are 0. */
		o->last_i = o->last_q = 0;
	} else {
		o->last_i = lp[o->iq_len - 2];
		o->last_q = lp[o->iq_len - 1];
	}
	o->pcm_len = o->iq_len / 2;
}

/* am/usb/lsb/raw, src/rtl_fm.c:617-665.  The int16 cast binds before the multiply. */
static void envelope_modes(orx_fm *o)
{
	const int16_t *lp = o->iq;
	int k;
	if (o->p.mode == 4) {
		memcpy(o->pcm, lp, (size_t)o->iq_len * 2);
		o->pcm_len = o->iq_len;
		return;
	}
	for (k = 0; k < o->iq_len; k += 2) {
		int v;
		if (o->p.mode == 1) {
			v = lp[k] * lp[k] + lp[k + 1] * lp[k + 1];
			o->pcm[k / 2] = (int16_t)((int16_t)sqrt(v) * o->p.output_scale);
		} else if (o->p.mode == 2) {
			v = lp[k] + lp[k + 1];
			o->pcm[k / 2] = (int16_t)((int16_t)v * o->p.output_scale);
		} else {
			v = lp[k] - lp[k + 1];
			o->pcm[k / 2] = (int16_t)((int16_t)v * o->p.output_scale);
		}
	}
	o->pcm_len = o->iq_len / 2;
}

/* -o N: per-chunk group sums plus the stray copy one slot past the end
 * (low_pass_simple, src/rtl_fm.c:373-387). */
static int group_sum_inplace(int16_t *s, int len, int step)
{
	int g, t, acc;
	for (g = 0; g < len; g += step) {
		acc = 0;
		for (t = 0; t < step; t++) { acc += (int)s[g + t]; }
		s[g / step] = (int16_t)acc;
	}
	s[g / step + 1] = s[g / step];
	return len / step;
}

/* de-emphasis IIR with round-to-nearest integer step (deemph_filter, src/rtl_fm.c:667-682). */
static void deemphasis(orx_fm *o)
{
	int k, a = o->p.deemph_a, d;
	for (k = 0; k < o->pcm_len; k++) {
		d = o->pcm[k] - o->deemph_avg;
		o->deemph_avg += (d > 0) ? (d + a / 2) / a : (d - a / 2) / a;
		o->pcm[k] = (int16_t)o->deemph_avg;
	}
}

/* -E adc (dc_block_audio_filter, src/rtl_fm.c:684-697). */
static void audio_dc_block(orx_fm *o)
{
	int64_t s = 0;
	int k, m, w = o->p.adc_block_const;
	for (k = 0; k < o->pcm_len; k++) { s += o->pcm[k]; }
	m = (int)(s / o->pcm_len);
	m = (m + o->adc_avg * w) / (w + 1);
	for (k = 0; k < o->pcm_len; k++) { o->pcm[k] = (int16_t)(o->pcm[k] - m); }
	o->adc_avg = m;
}

/* -r: rational boxcar resampler, divisor is the INTEGER ratio (low_pass_real,
 * src/rtl_fm.c:389-409). */
static void output_resample(orx_fm *o)
{
	int rd, wr = 0, fast = o->p.rate_out, slow = o->p.rate_out2;
	for (rd = 0; rd < o->pcm_len; rd++) {
		o->lpr_acc += o->pcm[rd];
		o->lpr_phase += slow;
		if (o->lpr_phase < fast) { continue; }
		o->pcm[wr++] = (int16_t)(o->lpr_acc / (fast / slow));
		o->lpr_phase -= fast;
		o->lpr_acc = 0;
	}
	o->pcm_len = wr;
}

/* callback body + full_demod for one chunk (src/rtl_fm.c:844-857, :759-824). */
static void fm_chunk(orx_fm *o, const int16_t *in, int len)
{
	int k, p, P = o->p.downsample_passes;
	for (k = 0; k < len; k++) { o->iq[k] = orx_scale_sample(in[k]); }
	if (o->p.dc_block_raw) { raw_dc_block(o, o->iq, len); }
	if (!o->p.offset_tuning) { quarter_rate_rotate(o->iq, len); }
	o->iq_len = len;

	if (P) {
		for (p = 0; p < P; p++) {
			halfband_pass(o->iq, o->iq_len >> p, o->hb_i[p]);
			halfband_pass(o->iq + 1, (o->iq_len >> p) - 1, o->hb_q[p]);
		}
		o->iq_len >>= P;
		if (o->p.comp_fir_size == 9 && P <= 10) {
			droop_fir9(o->iq, o->iq_len, k_droop9[P], o->droop_i);
			droop_fir9(o->iq + 1, o->iq_len - 1, k_droop9[P], o->droop_q);
		}
	} else {
		boxcar_decimate(o);
	}
	o->last_level = 0;
	if (o->p.squelch_level) {
		int level = buffer_rms(o->iq, o->iq_len, 1);
		o->last_level = level;
		if (level < o->p.squelch_level) {
			o->squelch_hits++;
			memset(o->iq, 0, (size_t)o->iq_len * 2);
		} else {
			o->squelch_hits = 0;
		}
	}
	/* -L statistics input (src/rtl_fm.c:792-794): reuse the squelch's rms unless it was 0 */
	if (o->want_levels && !o->last_level) { o->last_level = buffer_rms(o->iq, o->iq_len, 1); }
	if (o->p.mode == 0) { fm_discriminate(o); } else { envelope_modes(o); }
	if (o->p.mode == 4) { return; }
	if (o->p.post_downsample > 1) { o->pcm_len = group_sum_inplace(o->pcm, o->pcm_len, o->p.post_downsample); }
	if (o->p.deemph) { deemphasis(o); }
	if (o->p.dc_block_audio) { audio_dc_block(o); }
	if (o->p.rate_out2 > 0) { output_resample(o); }
}

orx_fm *orx_fm_new(const orx_fm_params *p)
{
	orx_fm *o = (orx_fm *)calloc(1, sizeof *o);
	if (!o) { return NULL; }
	o->p = *p;
	o->squelch_hits = 11;                       /* demod_init, src/rtl_fm.c:1091 */
	o->iq = (int16_t *)calloc(ORX_MAX_CHUNK + 64, 2);
	o->pcm = (int16_t *)calloc(ORX_MAX_CHUNK + 64, 2);
	if (p->custom_atan == 2) {
		o->atan_tab = (int *)malloc(sizeof(int) * ORX_ATAN_SIZE);
		orx_build_atan_table(o->atan_tab);
	}
	return o;
}

void orx_fm_free(orx_fm *o)
{
	if (!o) { return; }
	free(o->atan_tab); free(o->iq); free(o->pcm); free(o);
}

/* Whole stream, chunk by chunk; same contract as ref_fm_run in ref_fm_harness.c. */
long orx_fm_run(orx_fm *o, const int16_t *in, size_t n_int16, size_t chunk_int16,
                int16_t *out, size_t out_cap, int *chunk_result_len, int *chunk_squelch_hits)
{
	size_t pos = 0, w = 0, c = 0;
	if (chunk_int16 == 0 || chunk_int16 > ORX_MAX_CHUNK) { return -2; }
	while (pos < n_int16) {
		size_t len = n_int16 - pos;
		if (len > chunk_int16) { len = chunk_int16; }
		fm_chunk(o, in + pos, (int)len);
		if (w + (size_t)o->pcm_len > out_cap) { return -1; }
		memcpy(out + w, o->pcm, 2 * (size_t)o->pcm_len);
		w += (size_t)o->pcm_len;
		if (chunk_result_len) { chunk_result_len[c] = o->pcm_len; }
		if (chunk_squelch_hits) { chunk_squelch_hits[c] = o->squelch_hits; }
		pos += len; c++;
	}
	return (long)w;
}

/* Per-chunk level (the `sr` of src/rtl_fm.c:792-806); same contract as ref_fm_run_levels. */
long orx_fm_run_levels(orx_fm *o, const int16_t *in, size_t n_int16, size_t chunk_int16, int *levels)
{
	size_t pos = 0, c = 0;
	if (chunk_int16 == 0 || chunk_int16 > ORX_MAX_CHUNK) { return -2; }
	o->want_levels = 1;
	while (pos < n_int16) {
		size_t len = n_int16 - pos;
		if (len > chunk_int16) { len = chunk_int16; }
		fm_chunk(o, in + pos, (int)len);
		levels[c] = o->last_level;
		pos += len; c++;
	}
	o->want_levels = 0;
	return (long)c;
}

double orx_fm_time(orx_fm *o, const int16_t *in, size_t n_int16, size_t chunk_int16, int repeats, long *n_out)
{
	struct timespec t0, t1;
	long total = 0;
	int r;
	clock_gettime(CLOCK_MONOTONIC, &t0);
	for (r = 0; r < repeats; r++) {
		size_t pos = 0;
		while (pos < n_int16) {
			size_t len = n_int16 - pos;
			if (len > chunk_int16) { len = chunk_int16; }
			fm_chunk(o, in + pos, (int)len);
			total += o->pcm_len;
			pos += len;
		}
	}
	clock_gettime(CLOCK_MONOTONIC, &t1);
	if (n_out) { *n_out = total; }
	return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}

/* ------------------------------------------------------------------ rx_power */

typedef struct {
	int bin_e;             /* log2 FFT length                    src/rtl_power.c:94 */
	int buf_len;           /* int16 per hop buffer               :104, :504-507 */
	int downsample;        /*                                    :97 */
	int downsample_passes; /*                                    :98 */
	int comp_fir_size;     /* global comp_fir_size               :116 */
	int boxcar;            /* global boxcar                      :115 */
	int peak_hold;         /* global peak_hold                   :117 */
} orx_power_params;

/* Sinewave[i] = round(32767 sin(2 pi i / N)), i < 3N/4 (sine_table, src/rtl_power.c:240-254) */
void orx_sine_table(int log2n, int16_t *dst)
{
	int n = 1 << log2n, i;
	for (i = 0; i < n * 3 / 4; i++) {
		dst[i] = (int16_t)(int)round(32767 * sin((double)i * 2.0 * M_PI / n));
	}
}

/* window shapes, src/rtl_power.c:322-401; table entry = (int)(256*w) (:1034-1037).
 * id: 0 rectangle 1 hamming 2 blackman 3 blackman-harris 4 hann-poisson 5 youssef
 *     6 kaiser(==1) 7 bartlett 8 plain Hann (not in the reference; SURVEY F4). */
static double window_value(int id, int i, int length)
{
	double n1 = (double)(length - 1), w;
	switch (id) {
	case 1: return 25.0 / 46.0 - (21.0 / 46.0) * cos(2 * i * M_PI / n1);
	case 2: return 7938.0 / 18608.0 - (9240.0 / 18608.0) * cos(2 * i * M_PI / n1)
	             + (1430.0 / 18608.0) * cos(4 * i * M_PI / n1);
	case 3: return 0.35875 - 0.48829 * cos(2 * i * M_PI / n1) + 0.14128 * cos(4 * i * M_PI / n1)
	             - 0.01168 * cos(6 * i * M_PI / n1);
	case 4: return 0.5 * (1 - cos(2 * M_PI * i / n1))
	             * pow(M_E, (-2.0 * (double)abs((int)(n1 - 1 - 2 * i))) / n1);
	case 5: w = 0.35875 - 0.48829 * cos(2 * i * M_PI / n1) + 0.14128 * cos(4 * i * M_PI / n1)
	          - 0.01168 * cos(6 * i * M_PI / n1);
	        return w * pow(M_E, (-0.0025 * (double)abs((int)(n1 - 1 - 2 * i))) / n1);
	case 7: w = (i - n1 / 2) / ((double)length / 2); if (w < 0) { w = -w; } return 1 - w;
	case 8: return 0.5 * (1 - cos(2 * M_PI * i / n1));
	default: return 1.0;
	}
}
void orx_window_table(int id, int length, int *dst)
{
	int i;
	for (i = 0; i < length; i++) { dst[i] = (int)(256 * window_value(id, i, length)); }
}

/* FIX_MPY, src/rtl_power.c:256-262: (a*b)>>14, then halve rounding the dropped bit up. */
static int16_t q15_mul(int16_t a, int16_t b)
{
	int c = ((int)a * (int)b) >> 14;
	return (int16_t)((c >> 1) + (c & 1));
}

/* In-place radix-2 decimation-in-time FFT on interleaved int16, every stage halves
 * (fix_fft, src/rtl_power.c:264-320).  sine has 3N/4 entries for N = 2^log2_wave. */
int orx_fix_fft(int16_t *iq, int m, const int16_t *sine, int log2_wave)
{
	int n = 1 << m, nw = 1 << log2_wave, rev = 0, idx, half, span, tw_shift, a, b, g;
	if (n > nw) { return -1; }
	/* bit-reversal permutation (:275-290) */
	for (idx = 1; idx <= n - 1; idx++) {
		int bit = n;
		do { bit >>= 1; } while (rev + bit > n - 1);
		rev = (rev & (bit - 1)) + bit;
		if (rev <= idx) { continue; }
		{ int16_t t = iq[2 * idx]; iq[2 * idx] = iq[2 * rev]; iq[2 * rev] = t; }
		{ int16_t t = iq[2 * idx + 1]; iq[2 * idx + 1] = iq[2 * rev + 1]; iq[2 * rev + 1] = t; }
	}
	tw_shift = log2_wave - 1;
	for (half = 1; half < n; half = span) {
		span = half << 1;
		for (g = 0; g < half; g++) {
			int16_t wr = (int16_t)(sine[(g << tw_shift) + nw / 4] >> 1);
			int16_t wi = (int16_t)(((int16_t)(-sine[g << tw_shift])) >> 1);
			for (a = g; a < n; a += span) {
				int16_t tr, ti, qr, qi;
				b = a + half;
				tr = (int16_t)(q15_mul(wr, iq[2 * b]) - q15_mul(wi, iq[2 * b + 1]));
				ti = (int16_t)(q15_mul(wr, iq[2 * b + 1]) + q15_mul(wi, iq[2 * b]));
				qr = (int16_t)(iq[2 * a] >> 1);
				qi = (int16_t)(iq[2 * a + 1] >> 1);
				iq[2 * b] = (int16_t)(qr - tr);
				iq[2 * b + 1] = (int16_t)(qi - ti);
				iq[2 * a] = (int16_t)(qr + tr);
				iq[2 * a + 1] = (int16_t)(qi + ti);
			}
		}
		tw_shift--;
	}
	return 0;
}

/* stateless half-band with its "ease-in" head (rx_power's fifth_order,
 * src/rtl_power.c:582-607): int temporaries, first three outputs special-cased (including
 * the d-used-twice expression), loop from i = 12. */
static void power_halfband(int16_t *x, int span)
{
	int a = x[0], b = x[2], c = x[4], d = x[6], e = x[8], f = x[10], i;
	x[0] = (int16_t)(((a + b) * 10 + (c + d) * 5 + d + f) >> 4);
	x[2] = (int16_t)(((b + c) * 10 + (a + d) * 5 + e + f) >> 4);
	x[4] = (int16_t)((a + (b + e) * 5 + (c + d) * 10 + f) >> 4);
	for (i = 12; i < span; i += 4) {
		a = c; b = d; c = e; d = f;
		e = x[i - 2];
		f = x[i];
		x[i / 2] = (int16_t)((a + (b + e) * 5 + (c + d) * 10 + f) >> 4);
	}
}

/* stateless droop FIR: first nine samples pass through (src/rtl_power.c:626-654). */
static void power_droop9(int16_t *x, int span, const int *c)
{
	int h[9], d, k;
	for (d = 0; d < 18; d += 2) { h[d / 2] = x[d]; }
	for (d = 18; d < span; d += 2) {
		int in = x[d];
		int acc = (h[0] + h[8]) * c[1] + (h[1] + h[7]) * c[2] + (h[2] + h[6]) * c[3]
		        + (h[3] + h[5]) * c[4] + h[4] * c[5];
		x[d] = (int16_t)(acc >> 15);
		for (k = 0; k < 8; k++) { h[k] = h[k + 1]; }
		h[8] = in;
	}
}

/* remove_dc, src/rtl_power.c:609-624: the sum of one component is divided by `span`
 * (the int16 count), not by the number of samples summed. */
static void power_remove_dc(int16_t *x, int span)
{
	int64_t s = 0;
	int16_t m;
	int i;
	for (i = 0; i < span; i += 2) { s += x[i]; }
	m = (int16_t)(s / (int64_t)span);
	if (m == 0) { return; }
	for (i = 0; i < span; i += 2) { x[i] = (int16_t)(x[i] - m); }
}

/* rms_power, src/rtl_power.c:403-429 (bin_e == 0 hops). */
static void power_rms_hop(const orx_power_params *p, const int16_t *buf, int64_t *avg, int *samples)
{
	int64_t sq = 0, sum = 0;
	double dc, err;
	int i;
	for (i = 0; i < p->buf_len; i++) { int v = buf[i]; sum += v; sq += (int64_t)v * v; }
	dc = (double)sum / (double)p->buf_len;
	err = sum * 2 * dc - dc * dc * p->buf_len;
	sq -= (int64_t)round(err);
	if (!p->peak_hold) { avg[0] += sq; } else if (sq > avg[0]) { avg[0] = sq; }
	*samples += 1;
}

/* One hop buffer through scanner()'s per-hop body (src/rtl_power.c:709-771).
 * buf = the first buf_len int16 that readStream left in ts->buf16 (SURVEY F10);
 * work must hold buf_len int16; avg has 2^bin_e entries and is accumulated into. */
void orx_power_hop(const orx_power_params *p, const int *window, const int16_t *sine,
                   const int16_t *buf, int16_t *work, int64_t *avg, int *samples)
{
	int n = 1 << p->bin_e, ds = p->downsample, used, off, j, pass;
	if (n == 1) { power_rms_hop(p, buf, avg, samples); return; }
	memcpy(work, buf, (size_t)p->buf_len * 2);
	if (p->boxcar && ds > 1) {
		/* src/rtl_power.c:723-733: slot k accumulates (with int16 wrap) samples
		 * [k*ds, (k+1)*ds); sources are zeroed. */
		int rd = 2, wr = 0;
		while (rd < p->buf_len) {
			work[wr] = (int16_t)(work[wr] + work[rd]);
			work[wr + 1] = (int16_t)(work[wr + 1] + work[rd + 1]);
			work[rd] = 0; work[rd + 1] = 0;
			rd += 2;
			if (rd % (ds * 2) == 0) { wr += 2; }
		}
	} else if (p->downsample_passes) {
		for (pass = 0; pass < p->downsample_passes; pass++) {
			power_halfband(work, p->buf_len >> pass);
			power_halfband(work + 1, (p->buf_len >> pass) - 1);
		}
		if (p->comp_fir_size == 9 && p->downsample_passes <= 10) {
			power_droop9(work, p->buf_len >> pass, k_droop9[p->downsample_passes]);
			power_droop9(work + 1, (p->buf_len >> pass) - 1, k_droop9[p->downsample_passes]);
		}
	}
	used = p->buf_len / ds;
	power_remove_dc(work, used);
	power_remove_dc(work + 1, used - 1);
	for (off = 0; off < used; off += 2 * n) {
		for (j = 0; j < n; j++) {
			work[off + 2 * j] = (int16_t)((int32_t)work[off + 2 * j] * window[j]);
			work[off + 2 * j + 1] = (int16_t)((int32_t)work[off + 2 * j + 1] * window[j]);
		}
		orx_fix_fft(work + off, p->bin_e, sine, p->bin_e);
		for (j = 0; j < n; j++) {
			int64_t re = work[off + 2 * j], im = work[off + 2 * j + 1];
			int64_t pw = re * re + im * im;
			if (!p->peak_hold) { avg[j] += pw; } else if (pw > avg[j]) { avg[j] = pw; }
		}
		*samples += ds;
	}
}

/* n_pass sweeps over n_hops hops: hop_bufs = int16[n_pass][n_hops][buf_len];
 * avg = int64[n_hops][2^bin_e] (accumulated into), samples = int[n_hops]. */
void orx_power_scan(const orx_power_params *p, const int *window, const int16_t *sine,
                    const int16_t *hop_bufs, int n_pass, int n_hops, int64_t *avg, int *samples)
{
	int16_t *work = (int16_t *)malloc((size_t)p->buf_len * 2 + 64);
	int n = 1 << p->bin_e, s, h;
	for (s = 0; s < n_pass; s++) {
		for (h = 0; h < n_hops; h++) {
			orx_power_hop(p, window, sine, hop_bufs + ((size_t)s * n_hops + h) * p->buf_len,
			              work, avg + (size_t)h * n, samples + h);
		}
	}
	free(work);
}

double orx_power_time(const orx_power_params *p, const int *window, const int16_t *sine,
                      const int16_t *hop_bufs, int n_pass, int n_hops, int64_t *avg, int *samples, int repeats)
{
	struct timespec t0, t1;
	int r;
	clock_gettime(CLOCK_MONOTONIC, &t0);
	for (r = 0; r < repeats; r++) { orx_power_scan(p, window, sine, hop_bufs, n_pass, n_hops, avg, samples); }
	clock_gettime(CLOCK_MONOTONIC, &t1);
	return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}

/* ------------------------------------------------------------------ rx_sdr conversions
 * Restatement of the recorder loop's format conversions (src/rtl_sdr.c:348-391).  PARITY UNPINNED by
 * execution: the conversions live inline in rx_sdr's main() and cannot be called; the CS8 expression is the
 * same one rx_fm's callback uses (pinned through libref_fm), the others are single C expressions. */
void orx_sdr_cs16_to_cs8(const int16_t *src, size_t n_int16, uint8_t *dst)
{
	size_t i;
	for (i = 0; i < n_int16; i++) { dst[i] = (uint8_t)(int)((int16_t)src[i] / 32767.0 * 128.0 + 0.4); }       /* :369 */
}
void orx_sdr_cs16_to_cu8(const int16_t *src, size_t n_int16, uint8_t *dst)
{
	size_t i;
	for (i = 0; i < n_int16; i++) { dst[i] = (uint8_t)(int)((int16_t)src[i] / 32767.0 * 128.0 + 127.4); }     /* :377 */
}
void orx_sdr_cs16_to_cf32(const int16_t *src, size_t n_int16, float *dst)
{
	size_t i;
	for (i = 0; i < n_int16; i++) { dst[i] = src[i] * 1.0f / 32767; }                                         /* :385, SHRT_MAX */
}
void orx_sdr_cs12_to_cs16(const uint8_t *src, size_t n_complex, int16_t *dst)
{
	size_t i;
	for (i = 0; i < n_complex; i++) {                                                                            /* :354-362 */
		uint8_t b0 = src[3 * i], b1 = src[3 * i + 1], b2 = src[3 * i + 2];
		dst[2 * i + 0] = (int16_t)((b1 << 12) | (b0 << 4));
		dst[2 * i + 1] = (int16_t)((b2 << 8) | (b1 & 0xf0));
	}
}
