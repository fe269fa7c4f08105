/* rx_power_b200 — drop-in for rx_tools' rx_power whose per-hop DSP runs on an H100 through librxb200.so.
 *
 * Same command line (option string of src/rtl_power.c:848), same CSV rows
 * ("date, time, Hz low, Hz high, Hz step, samples, dB, dB, ..."), same SoapySDR CS16 stream surface.
 * Host logic is our own: plan (rxb200_power_plan_range == frequency_range()), retune + flush read per
 * hop, one readStream per hop buffer; the window x fix_fft x power-accumulate of every hop of a sweep is
 * ONE rxb200_power_accumulate() call, the report is rxb200_power_read_db() (csv_dbm's arithmetic on the
 * device) + rxb200_power_format_db_row().
 *
 * Several GPUs: RXB200_GPUS=n (environment, so the reference's option string stays as it is) shards the hops over
 * n GPUs of this box through rxb200_power_group_* -- every GPU transforms the hops it owns, ONE NCCL all-gather
 * collates the spectrum rows in hop order before the report loop (src/rtl_power.c:1047-1050).
 *
 * Capture mode: RXB200_CAPTURE_RATE=<max Hz> takes every hop of a sweep from ONE wideband capture instead of a retune
 * and a read per hop.  The device is tuned once to the centre of the hops, at M times the hop rate, and read without
 * pause; each pass of M * buf_len int16 goes through rxb200_power_mix_accumulate, whose NCO down-converter makes every
 * hop's buffer on the GPU.  A pass counts as a sweep.
 *
 * Tile mode: RXB200_TILE_RATE=<max Hz> takes a sweep wider than one capture in tiles of consecutive hops
 * (rxb200_power_plan_tiles).  Per sweep, each tile is one retune to its centre, one flush read, and one burst of the
 * filter's lead plus one pass, gathered from reads of any length and handed to rxb200_power_mix_accumulate_burst for
 * the tile's hops.  A failed read drops that tile's burst for the sweep, as hop mode skips a hop.
 *
 * RXB200_DEVICE_RATE=<Hz> with capture or tile mode: the device runs at that rate instead of R.  The plan is
 * rxb200_power_plan_capture_at's or rxb200_power_plan_tiles_at's (the decimation leaves the resampler's guard band;
 * tiles shrink to fit the device; a capture plan above the device rate exits 1 before the device is opened).  The
 * device is asked for R_dev, and the rate it reports is what the plan and the resampler start from.  Capture mode reads
 * passes of the device samples that emit one pass of M * buf_len int16 (rxb200_resample_in_len) into a handle with
 * rxb200_power_mix_set_device_rate; tile mode reads bursts of rxb200_power_mix_burst_in_len device int16 into a handle
 * with rxb200_power_mix_set_burst_device_rate.
 *
 * RXB200_DEVICE_FORMAT=CS16|CS8|CU8|CS12 with capture or tile mode: the stream is opened in that format, passes and
 * bursts are gathered as the same counts of elements in it, and the handle widens them to CS16 on the GPU
 * (rxb200_power_mix_set_input_format), so the CSV is that of the same run on the widened CS16 stream.  An unknown
 * value, or the variable without capture or tile mode, exits 1 before the device is opened.
 */
#include <math.h>
#include <signal.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>
#include "sdr_util.h"
#include "rxb200.h"

#define BUFFER_DUMP 16384            /* elements flushed after a retune, src/rtl_power.c:71-72, :568 */

static volatile sig_atomic_t g_stop = 0;
static int g_in_fmt = RXB200_IN_CS16;            /* the device's format (RXB200_DEVICE_FORMAT), capture and tile mode */
static const char *g_in_name = SOAPY_SDR_CS16;   /* its SoapySDR name, the stream's format */
static void on_signal(int s) { (void)s; g_stop++; }

static void usage(void)
{
	fprintf(stderr,
		"rx_power_b200, rx_power with the FFT on an H100 GPU\n\n"
		"Use:\trx_power_b200 -f freq_range [-options] [filename]\n"
		"\t-f lower:upper:bin_size [Hz]\n"
		"\t[-i integration_interval (default: 10 seconds)] [-1 single-shot] [-e exit_timer]\n"
		"\t[-d device] [-C channel] [-a antenna] [-g gain] [-p ppm_error]\n"
		"\t[-w rectangle|hamming|blackman|blackman-harris|hann-poisson|youssef|kaiser|bartlett]\n"
		"\t[-c crop_percent] [-F fir_size] [-P peak hold] [-D direct_sampling] [-O offset tuning]\n"
		"\t[-S tuner_sleep_usec] [-R tuner_retry_max]\n"
		"\tfilename ('-' means stdout)\n"
		"environment: RXB200_GPUS=n shards the hops over n GPUs; RXB200_CAPTURE_RATE=max_Hz takes every hop from one\n"
		"\tcapture of at most max_Hz samples/s, tuned once to the centre of the sweep (one GPU);\n"
		"\tRXB200_TILE_RATE=max_Hz takes a wider sweep in tiles of hops, one retune and one burst of at most max_Hz\n"
		"\tsamples/s per tile (one GPU); RXB200_DEVICE_RATE=Hz (with either) runs the device at that rate and resamples\n"
		"\tits stream to the capture's rate on the GPU; RXB200_DEVICE_FORMAT=CS16|CS8|CU8|CS12 (with either) reads the\n"
		"\tdevice in that format and widens it to CS16 on the GPU\n");
	exit(1);
}

static int window_id(const char *name)
{
	static const char *names[] = {"rectangle", "hamming", "blackman", "blackman-harris", "hann-poisson", "youssef", "kaiser", "bartlett"};
	for (int i = 0; i < 8; i++) { if (!strcmp(name, names[i])) { return i; } }
	return -1;
}

/* ---- report (:1044-1058): csv_dbm()'s rows of every hop from the accumulators of pw, then the date/time prefix */
static int report(FILE *out, rxb200_power *pw, const rxb200_power_plan *plan, double *db, int row_len, int *samples,
                  char *row, size_t row_cap, const char *tstr)
{
	const rxb200_power_params *pp = &plan->params;
	if (rxb200_power_read_db(pw, plan->rate, plan->crop, db, (size_t)row_len, samples) != RXB200_OK) { fprintf(stderr, "rxb200: %s\n", rxb200_last_error()); return -1; }
	int have = 0;
	for (int i = 0; i < pp->n_hops; i++) { have |= samples[i]; }
	if (have) {
		for (int i = 0; i < pp->n_hops; i++) {
			int n = rxb200_power_format_db_row(db + (size_t)i * row_len, pp->bin_e, plan->first_freq + (int64_t)i * plan->freq_step, plan->rate,
			                                pp->downsample, plan->crop, samples[i], row, row_cap);
			if (n < 0) { fprintf(stderr, "rxb200: %s\n", rxb200_last_error()); break; }
			fprintf(out, "%s, ", tstr);
			fwrite(row, 1, (size_t)n, out);
		}
		fflush(out);
	}
	return 0;
}

static void time_string(char *tstr, size_t cap, time_t now)
{
	struct tm cal;
	localtime_r(&now, &cal);
	strftime(tstr, cap, "%Y-%m-%d, %H:%M:%S", &cal);
	if (getenv("RXB200_FIXED_TIME")) { snprintf(tstr, cap, "%s", getenv("RXB200_FIXED_TIME")); }
}

/* The set-up every mode shares: the device, its stream, the signal handlers, the -D / -O / -g / -p settings, then the
 * output file.  NULL (reported on stderr) when the device or the file cannot be opened. */
static FILE *open_radio(const char *dev_query, size_t channel, const char *antenna, const char *gain_str, int ppm,
                        int direct_sampling, int offset_tuning, const char *filename, SoapySDRDevice **devp,
                        SoapySDRStream **streamp)
{
	if (sdr_open(dev_query, channel, g_in_name, devp, streamp) != 0) { fprintf(stderr, "Failed to open sdr device matching '%s'.\n", dev_query); return NULL; }
	SoapySDRDevice *dev = *devp;
	if (antenna && SoapySDRDevice_setAntenna(dev, SOAPY_SDR_RX, channel, antenna) != 0) { fprintf(stderr, "Failed to set antenna"); }
	SoapySDRDevice_activateStream(dev, *streamp, 0, 0, 0);
	struct sigaction sa; memset(&sa, 0, sizeof sa); sa.sa_handler = on_signal;
	sigaction(SIGINT, &sa, NULL); sigaction(SIGTERM, &sa, NULL); sigaction(SIGQUIT, &sa, NULL);
	signal(SIGPIPE, SIG_IGN);
	if (direct_sampling) { SoapySDRDevice_writeSetting(dev, "direct_samp", direct_sampling == 1 ? "1" : "2"); }
	if (offset_tuning) { SoapySDRDevice_writeSetting(dev, "offset_tune", "true"); }
	sdr_set_gain(dev, channel, gain_str);
	SoapySDRDevice_setFrequencyCorrection(dev, SOAPY_SDR_RX, channel, (double)ppm);
	FILE *out = !strcmp(filename, "-") ? stdout : fopen(filename, "wb");
	if (!out) { fprintf(stderr, "Failed to open %s\n", filename); }
	return out;
}

/* retune() (:548-580): tune to f, sleep -S, then one flush read of BUFFER_DUMP elements with -R tries */
static void retune(SoapySDRDevice *dev, SoapySDRStream *stream, size_t channel, int64_t f, int16_t *dump,
                   int tuner_sleep_usec, int tuner_retry_max)
{
	SoapySDRKwargs none = {0, NULL, NULL};
	if (SoapySDRDevice_setFrequency(dev, SOAPY_SDR_RX, channel, (double)f, &none) != 0) {
		fprintf(stderr, "Error: failed to set frequency %lli Hz\n", (long long)f);
		return;
	}
	usleep((useconds_t)tuner_sleep_usec);
	int r = -1, flags = 0; long long tn = 0; void *bp[] = {dump};
	for (int a = 0; a < tuner_retry_max && r < 0; a++) { r = SoapySDRDevice_readStream(dev, stream, bp, BUFFER_DUMP, &flags, &tn, 1000000); }
	if (r < 0) { fprintf(stderr, "Error: bad retune at %lli Hz, r=%d (try increasing -S or -R).\n", (long long)f, r); }
}

/* Capture or tile mode's plan and handle.  tiles: tile mode, its plan rxb200_power_plan_tiles's, else capture mode's
 * rxb200_power_plan_capture's; each the _at planner's when dev_rate is not 0, with the resampler from that rate
 * attached to the handle (to its bursts in tile mode).  limit is the mode's variable, RXB200_TILE_RATE's or
 * RXB200_CAPTURE_RATE's value.  Prints the mode's banner and the device rate's line; nonzero, reported on stderr, when
 * a plan or the handle is refused. */
struct power_setup {
	rxb200_power_mix *pm;
	rxb200_power_tiling tl;      /* tile mode */
	int64_t fc;                  /* capture mode: the centre */
	int decim, rate;             /* M and R = M plan->rate */
	int rs_up, rs_down;          /* capture mode at a device rate: the resampler's L/N (0: none attached) */
};
static int power_setup(int tiles, const rxb200_power_plan *plan, const int *window_coefs, const char *limit,
                       long long dev_rate, struct power_setup *ps)
{
	const rxb200_power_params *pp = &plan->params;
	const char *mode = tiles ? "Tile mode" : "Capture mode", *var = tiles ? "RXB200_TILE_RATE" : "RXB200_CAPTURE_RATE";
	memset(ps, 0, sizeof *ps);
	int *offs = (int *)malloc(sizeof(int) * (size_t)pp->n_hops);
	rxb200_fm_capture_plan cp;
	int rc, T;
	if (tiles) {
		rc = dev_rate ? rxb200_power_plan_tiles_at(plan, atoll(limit), dev_rate, &ps->tl, offs)
		              : rxb200_power_plan_tiles(plan, atoll(limit), &ps->tl, offs);
		ps->decim = ps->tl.decim; ps->rate = ps->tl.capture_rate; T = ps->tl.n_taps;
	} else {
		rc = dev_rate ? rxb200_power_plan_capture_at(plan, atoll(limit), dev_rate, &cp, offs)
		              : rxb200_power_plan_capture(plan, atoll(limit), &cp, offs);
		ps->fc = cp.centre_hz; ps->decim = cp.decim; ps->rate = cp.capture_rate; T = cp.n_taps;
	}
	if (rc == RXB200_EINVAL && !tiles) {         /* the rate the span needs is above the cap (the message names it) */
		fprintf(stderr, "Capture mode: %s, above RXB200_CAPTURE_RATE=%s.\n", rxb200_last_error(), limit);
		free(offs);
		return 1;
	}
	if (rc != RXB200_OK) { fprintf(stderr, "%s: %s (%s=%s).\n", mode, rxb200_last_error(), var, limit); free(offs); return 1; }
	if (tiles) {
		fprintf(stderr, "Tile mode: %d tiles of up to %d hops, %d Hz, decimation %d, %d taps\n", ps->tl.n_tiles,
		        ps->tl.hops_per_tile, ps->tl.capture_rate, ps->tl.decim, ps->tl.n_taps);
	} else {
		fprintf(stderr, "Capture mode: %lld Hz centred at %lli Hz, decimation %lld, %d taps\n", (long long)ps->rate,
		        (long long)ps->fc, (long long)ps->decim, T);
	}
	/* the resampler spans the widest tile (each offset is from its own tile's centre), or every hop */
	long long span = 0;
	for (int i = 0; i < pp->n_hops; i++) { span = 2 * (long long)abs(offs[i]) > span ? 2 * (long long)abs(offs[i]) : span; }
	rxb200_resampler rs = {1, 1, 0, NULL, 15};
	if (dev_rate && device_resampler(dev_rate, ps->rate, span + plan->rate, &rs) != 0) { free(offs); return 1; }
	int32_t *taps = (int32_t *)malloc(sizeof(int32_t) * (size_t)T);
	rxb200_ddc_lowpass(ps->decim, T, 15, taps);
	const rxb200_ddc ddc = {ps->decim, T, taps, 15};
	rc = rxb200_power_mix_create(pp, window_coefs, NULL, ps->rate, offs, &ddc, 0, &ps->pm);
	free(offs); free(taps);
	if (rc == RXB200_OK && rs.taps) {
		rc = tiles ? rxb200_power_mix_set_burst_device_rate(ps->pm, &rs) : rxb200_power_mix_set_device_rate(ps->pm, &rs);
		if (!tiles) { ps->rs_up = rs.up; ps->rs_down = rs.down; }
	}
	free((void *)rs.taps);
	if (rc == RXB200_OK && g_in_fmt != RXB200_IN_CS16) { rc = rxb200_power_mix_set_input_format(ps->pm, g_in_fmt); }
	if (rc != RXB200_OK) { fprintf(stderr, "rxb200: %s\n", rxb200_last_error()); return 1; }
	return 0;
}

/* The mode's sample rate on the device: R, or at a device rate R_dev the rate the device reports, planning again (a
 * new handle in *ps) when that is not R_dev.  The centres do not depend on the rate, so a tuning stands.  Nonzero,
 * reported on stderr, when the device reports no valid rate or the new plan is refused. */
static int device_side_rate(SoapySDRDevice *dev, size_t channel, int tiles, const rxb200_power_plan *plan,
                            const int *window_coefs, const char *limit, long long dev_rate, struct power_setup *ps)
{
	if (!dev_rate) { SoapySDRDevice_setSampleRate(dev, SOAPY_SDR_RX, channel, (double)ps->rate); return 0; }
	const long long got = sdr_device_rate(dev, channel, dev_rate);
	if (got < 0) { return 1; }
	if (got == dev_rate) { return 0; }
	fprintf(stderr, "The device reports %lld Hz, not RXB200_DEVICE_RATE=%lld Hz: planning again.\n", got, dev_rate);
	rxb200_power_mix_destroy(ps->pm);
	return power_setup(tiles, plan, window_coefs, limit, got, ps);
}

/* Tile mode's device side and report loop.  Per sweep, each tile retunes to its centre when the device is elsewhere,
 * then gathers one burst of rxb200_power_mix_burst_in_len int16 (G + M * buf_len / 2 complex samples, or at a device
 * rate the device samples that emit E more) from reads of whatever length the device returns and accumulates it for
 * the tile's hops.  A failed read drops the burst, so the tile's hops get no pass this sweep; the
 * stream has run dry when no tile got its burst in a sweep. */
static int tile_mode(struct power_setup *ps, const rxb200_power_plan *plan, const int *window_coefs, const char *limit,
                     long long dev_rate, const char *dev_query, size_t channel, const char *gain_str, const char *antenna,
                     const char *filename, int ppm, int direct_sampling, int offset_tuning, int tuner_sleep_usec,
                     int tuner_retry_max, int interval, int single, time_t exit_after)
{
	const rxb200_power_params *pp = &plan->params;
	const int n_hops = pp->n_hops, N = 1 << pp->bin_e;
	SoapySDRDevice *dev = NULL; SoapySDRStream *stream = NULL;
	FILE *out = open_radio(dev_query, channel, antenna, gain_str, ppm, direct_sampling, offset_tuning, filename, &dev, &stream);
	if (!out) { return 1; }
	if (device_side_rate(dev, channel, 1, plan, window_coefs, limit, dev_rate, ps) != 0) {
		if (out != stdout) { fclose(out); }
		sdr_close(dev, stream);
		return 1;
	}
	rxb200_power_mix *pm = ps->pm;
	const rxb200_power_tiling *tl = &ps->tl;
	rxb200_power *pw = rxb200_power_mix_member(pm);
	size_t burst16 = 0;                                  /* the lead plus one pass, device int16 at a device rate */
	rxb200_power_mix_burst_in_len(pm, 1, &burst16);
	int16_t *burst = (int16_t *)malloc(burst16 * sizeof(int16_t));
	int16_t *dump = (int16_t *)malloc((size_t)BUFFER_DUMP * 4);
	const int row_len = rxb200_power_row_len(pp->bin_e, plan->crop);
	double *db = (double *)malloc((size_t)n_hops * (size_t)row_len * sizeof(double));
	int *samples = (int *)malloc((size_t)n_hops * sizeof(int));
	char *row = (char *)malloc(64 + 16 * ((size_t)N + 8));
	const char *hook = getenv("RXB200_MAX_SWEEPS");       /* test hook: report after this many sweeps and exit */
	const long max_sweeps = hook ? atol(hook) : 0;
	long sweeps = 0;
	time_t next_tick = time(NULL) + interval, exit_time = exit_after ? time(NULL) + exit_after : 0;
	int done = 0, rc = 0;
	while (!done && !g_stop) {
		/* ---- one sweep: one burst per tile */
		int n_ok = 0;
		for (int t = 0; t < tl->n_tiles && !g_stop && !rc; t++) {
			int hb = 0, he = 0; int64_t fc = 0;
			rxb200_power_tile(plan, tl, t, &hb, &he, &fc);
			if ((int64_t)SoapySDRDevice_getFrequency(dev, SOAPY_SDR_RX, channel) != fc) {
				retune(dev, stream, channel, fc, dump, tuner_sleep_usec, tuner_retry_max);
			}
			size_t have = 0;
			while (have < burst16 && !g_stop) {
				void *bp[] = {(unsigned char *)burst + have / 2 * device_format_bytes(g_in_fmt)};   /* have: int16 */
				int flags = 0; long long tn = 0;
				const int r = SoapySDRDevice_readStream(dev, stream, bp, (burst16 - have) / 2, &flags, &tn, 1000000);
				if (r < 0) { fprintf(stderr, "Error: reading stream %d\n", r); break; }    /* the burst is dropped */
				have += 2 * (size_t)r;
			}
			if (have < burst16) { continue; }
			if (rxb200_power_mix_accumulate_burst(pm, hb, he, burst, burst16) != RXB200_OK) { fprintf(stderr, "rxb200: %s\n", rxb200_last_error()); rc = 1; break; }
			n_ok++;
		}
		if (rc) { break; }
		sweeps++;
		const int dry = n_ok == 0;
		time_t now = time(NULL);
		const int hooked = max_sweeps && sweeps >= max_sweeps;
		if (now < next_tick && !hooked && !dry) { continue; }
		char tstr[50];
		time_string(tstr, sizeof tstr, now);
		if (report(out, pw, plan, db, row_len, samples, row, 64 + 16 * ((size_t)N + 8), tstr) != 0) { rc = 1; break; }
		rxb200_power_reset(pw);
		while (time(NULL) >= next_tick) { next_tick += interval; }
		if (single || hooked || dry) { done = 1; }
		if (exit_time && time(NULL) >= exit_time) { done = 1; }
	}
	fprintf(stderr, g_stop ? "\nUser cancel, exiting...\n" : "\nDone, exiting...\n");
	if (out != stdout) { fclose(out); }
	free(burst); free(dump); free(db); free(samples); free(row);
	sdr_close(dev, stream);
	return rc;
}

/* Capture mode's device side and report loop: one tune to fc at R, one flush read, then passes of M * buf_len int16
 * collected from reads of whatever length the device returns; a failed read discards the partial pass, and
 * tuner_retry_max failed reads in a row mean the stream has run dry. */
static int capture_mode(struct power_setup *ps, const rxb200_power_plan *plan, const int *window_coefs,
                        const char *limit, long long dev_rate, const char *dev_query, size_t channel, const char *gain_str,
                        const char *antenna, const char *filename, int ppm, int direct_sampling, int offset_tuning,
                        int tuner_sleep_usec, int tuner_retry_max, int interval, int single, time_t exit_after)
{
	const rxb200_power_params *pp = &plan->params;
	const int n_hops = pp->n_hops, N = 1 << pp->bin_e;
	SoapySDRDevice *dev = NULL; SoapySDRStream *stream = NULL;
	FILE *out = open_radio(dev_query, channel, antenna, gain_str, ppm, direct_sampling, offset_tuning, filename, &dev, &stream);
	if (!out) { return 1; }
	if (device_side_rate(dev, channel, 0, plan, window_coefs, limit, dev_rate, ps) != 0) {
		if (out != stdout) { fclose(out); }
		sdr_close(dev, stream);
		return 1;
	}
	rxb200_power_mix *pm = ps->pm;
	rxb200_power *pw = rxb200_power_mix_member(pm);
	int16_t *dump = (int16_t *)malloc((size_t)BUFFER_DUMP * 4);
	retune(dev, stream, channel, ps->fc, dump, tuner_sleep_usec, tuner_retry_max);
	free(dump);
	/* a pass: M * buf_len capture int16; at a device rate, the device samples that emit them from the count so far */
	const size_t cap16 = (size_t)ps->decim * (size_t)pp->buf_len;
	const size_t max16 = ps->rs_up ? 2 * ((cap16 / 2 * (size_t)ps->rs_down + (size_t)ps->rs_up - 1) / (size_t)ps->rs_up + 1) : cap16;
	unsigned long long dev_pos = 0;                       /* device samples of the passes taken */
	int16_t *pass = (int16_t *)malloc(max16 * sizeof(int16_t));
	const int row_len = rxb200_power_row_len(pp->bin_e, plan->crop);
	double *db = (double *)malloc((size_t)n_hops * (size_t)row_len * sizeof(double));
	int *samples = (int *)malloc((size_t)n_hops * sizeof(int));
	char *row = (char *)malloc(64 + 16 * ((size_t)N + 8));
	const char *hook = getenv("RXB200_MAX_SWEEPS");       /* test hook: report after this many sweeps and exit */
	const long max_sweeps = hook ? atol(hook) : 0;
	long sweeps = 0;
	time_t next_tick = time(NULL) + interval, exit_time = exit_after ? time(NULL) + exit_after : 0;
	int done = 0, rc = 0;
	while (!done && !g_stop) {
		/* ---- one pass: M * buf_len int16 (or the device int16 that emit them) from as many reads as it takes */
		size_t pass16 = cap16;
		if (ps->rs_up) {
			size_t c = 0;
			rxb200_resample_in_len(ps->rs_up, ps->rs_down, dev_pos, cap16 / 2, &c);
			pass16 = 2 * c;
		}
		size_t have = 0;
		int fails = 0, dry = 0;
		while (have < pass16 && !g_stop) {
			void *bp[] = {(unsigned char *)pass + have / 2 * device_format_bytes(g_in_fmt)};   /* have: int16 */
			int flags = 0; long long tn = 0;
			const int r = SoapySDRDevice_readStream(dev, stream, bp, (pass16 - have) / 2, &flags, &tn, 1000000);
			if (r < 0) {
				fprintf(stderr, "Error: reading stream %d\n", r);
				have = 0;                                         /* the partial pass is not continuous with the next read */
				if (++fails >= tuner_retry_max) { dry = 1; break; }
				continue;
			}
			fails = 0;
			have += 2 * (size_t)r;
		}
		if (have == pass16) {
			if (rxb200_power_mix_accumulate(pm, pass, pass16) != RXB200_OK) { fprintf(stderr, "rxb200: %s\n", rxb200_last_error()); rc = 1; break; }
			dev_pos += pass16 / 2;
			sweeps++;
		}
		time_t now = time(NULL);
		const int hooked = max_sweeps && sweeps >= max_sweeps;
		if (now < next_tick && !hooked && !dry) { continue; }
		char tstr[50];
		time_string(tstr, sizeof tstr, now);
		if (report(out, pw, plan, db, row_len, samples, row, 64 + 16 * ((size_t)N + 8), tstr) != 0) { rc = 1; break; }
		rxb200_power_reset(pw);                               /* the accumulators only: the capture stream goes on */
		while (time(NULL) >= next_tick) { next_tick += interval; }
		if (single || hooked || dry) { done = 1; }
		if (exit_time && time(NULL) >= exit_time) { done = 1; }
	}
	fprintf(stderr, g_stop ? "\nUser cancel, exiting...\n" : "\nDone, exiting...\n");
	if (out != stdout) { fclose(out); }
	free(pass); free(db); free(samples); free(row);
	sdr_close(dev, stream);
	return rc;
}

int main(int argc, char **argv)
{
	const char *dev_query = "", *gain_str = NULL, *antenna = NULL, *filename = "-", *freq_arg = NULL;
	int opt, interval = 10, single = 0, ppm = 0, direct_sampling = 0, offset_tuning = 0, window = RXB200_WIN_RECTANGLE;
	int boxcar = 1, comp_fir_size = 0, peak_hold = 0, tuner_sleep_usec = 5000, tuner_retry_max = 3;
	size_t channel = 0;
	double crop = 0.0;
	time_t exit_after = 0;
	while ((opt = getopt(argc, argv, "a:C:f:i:s:t:d:g:p:e:w:c:F:1PD:OS:R:h")) != -1) {
		switch (opt) {
		case 'a': antenna = optarg; break;
		case 'C': channel = (size_t)atoi(optarg); break;
		case 'f': freq_arg = optarg; break;
		case 'd': dev_query = optarg; break;
		case 'g': gain_str = optarg; break;
		case 'c': crop = parse_fraction(optarg); break;
		case 'i': interval = (int)round(parse_seconds(optarg)); break;
		case 'e': exit_after = (time_t)((int)round(parse_seconds(optarg))); break;
		case 's': case 't': break;                    /* parsed but unused by the reference as well (:875-880, :899-901) */
		case 'w': { int w = window_id(optarg); if (w >= 0) { window = w; } } break;
		case 'p': ppm = atoi(optarg); break;
		case '1': single = 1; break;
		case 'P': peak_hold = 1; break;
		case 'D': direct_sampling = atoi(optarg); break;
		case 'O': offset_tuning = 1; break;
		case 'F': boxcar = 0; comp_fir_size = atoi(optarg); break;
		case 'S': tuner_sleep_usec = atoi(optarg); break;
		case 'R': tuner_retry_max = atoi(optarg); break;
		default: usage();
		}
	}
	if (!freq_arg) { fprintf(stderr, "No frequency range provided.\n"); usage(); }
	if (crop < 0.0 || crop > 1.0) { fprintf(stderr, "Crop value outside of 0 to 1.\n"); return 1; }
	if (argc > optind) { filename = argv[optind]; }
	if (interval < 1) { interval = 1; }

	/* -f lower:upper:bin */
	char *fa = strdup(freq_arg), *c1 = strchr(fa, ':'), *c2 = c1 ? strchr(c1 + 1, ':') : NULL;
	if (!c1 || !c2) { fprintf(stderr, "Bad frequency range.\n"); return 1; }
	*c1++ = 0; *c2++ = 0;
	rxb200_power_plan plan;
	if (rxb200_power_plan_range((int64_t)parse_scaled(fa), (int64_t)parse_scaled(c1), (int64_t)parse_scaled(c2), crop,
	                            boxcar, comp_fir_size, peak_hold, &plan) != RXB200_OK) {
		fprintf(stderr, "rxb200: %s\n", rxb200_last_error());
		return 1;
	}
	free(fa);
	const rxb200_power_params *pp = &plan.params;
	const int n_hops = pp->n_hops, N = 1 << pp->bin_e, buf_len = pp->buf_len;
	fprintf(stderr, "Number of frequency hops: %i\n", n_hops);
	fprintf(stderr, "Dongle bandwidth: %iHz\n", plan.rate);
	fprintf(stderr, "Downsampling by: %ix\n", pp->downsample);
	fprintf(stderr, "Cropping by: %0.2f%%\n", plan.crop * 100);
	fprintf(stderr, "Total FFT bins: %i\n", n_hops * N);
	fprintf(stderr, "Logged FFT bins: %i\n", (int)((double)(n_hops * N) * (1.0 - plan.crop)));
	fprintf(stderr, "FFT bin size: %0.2fHz\n", plan.bin_size_hz);
	fprintf(stderr, "Buffer size: %i bytes (%0.2fms)\n", buf_len, 1000 * 0.5 * (float)buf_len / (float)plan.rate);
	fprintf(stderr, "Reporting every %i seconds\n", interval);

	int *window_coefs = (int *)malloc(sizeof(int) * (size_t)N);
	rxb200_window_table(window, N, window_coefs);
	int n_gpus = getenv("RXB200_GPUS") ? atoi(getenv("RXB200_GPUS")) : 1;
	if (n_gpus < 1) { n_gpus = 1; }
	if (n_gpus > n_hops) { n_gpus = n_hops; }
	const char *cap_env = getenv("RXB200_CAPTURE_RATE"), *tile_env = getenv("RXB200_TILE_RATE");
	const long long dev_rate = device_rate_env(cap_env || tile_env, "capture or tile mode (RXB200_CAPTURE_RATE or RXB200_TILE_RATE)");
	if (dev_rate < 0) { return 1; }
	g_in_fmt = device_format_env(cap_env || tile_env, "capture or tile mode (RXB200_CAPTURE_RATE or RXB200_TILE_RATE)",
	                             &g_in_name);
	if (g_in_fmt < 0) { return 1; }
	if (tile_env) {
		/* tile mode: the planner's tiles, each hop's offset from its tile's centre, one filter for every tile */
		if (cap_env) { fprintf(stderr, "Tile mode (RXB200_TILE_RATE) and capture mode (RXB200_CAPTURE_RATE) exclude each other.\n"); return 1; }
		if (n_gpus > 1) { fprintf(stderr, "Tile mode (RXB200_TILE_RATE) runs on one GPU: unset RXB200_GPUS.\n"); return 1; }
		struct power_setup ps;
		if (power_setup(1, &plan, window_coefs, tile_env, dev_rate, &ps) != 0) { return 1; }
		const int rc = tile_mode(&ps, &plan, window_coefs, tile_env, dev_rate, dev_query, channel, gain_str, antenna, filename,
		                         ppm, direct_sampling, offset_tuning, tuner_sleep_usec, tuner_retry_max, interval, single,
		                         exit_after);
		rxb200_power_mix_destroy(ps.pm);
		return rc;
	}
	if (cap_env) {
		/* capture mode: centre of the hops, each hop's offset from it, the smallest M whose capture holds them all */
		if (n_gpus > 1) { fprintf(stderr, "Capture mode (RXB200_CAPTURE_RATE) runs on one GPU: unset RXB200_GPUS.\n"); return 1; }
		struct power_setup ps;
		if (power_setup(0, &plan, window_coefs, cap_env, dev_rate, &ps) != 0) { return 1; }
		const int rc = capture_mode(&ps, &plan, window_coefs, cap_env, dev_rate, dev_query, channel, gain_str, antenna,
		                            filename, ppm, direct_sampling, offset_tuning, tuner_sleep_usec, tuner_retry_max,
		                            interval, single, exit_after);
		rxb200_power_mix_destroy(ps.pm);
		return rc;
	}
	rxb200_power_group *grp = NULL;
	if (rxb200_power_group_create(pp, window_coefs, NULL, n_gpus, NULL, &grp) != RXB200_OK) { fprintf(stderr, "rxb200: %s\n", rxb200_last_error()); return 1; }
	rxb200_power *pw = rxb200_power_group_member(grp, 0);     /* after the gather member 0 holds every row */
	if (n_gpus > 1) { fprintf(stderr, "Hops sharded over %d GPUs\n", n_gpus); }

	SoapySDRDevice *dev = NULL; SoapySDRStream *stream = NULL;
	FILE *out = open_radio(dev_query, channel, antenna, gain_str, ppm, direct_sampling, offset_tuning, filename, &dev, &stream);
	if (!out) { return 1; }
	SoapySDRDevice_setSampleRate(dev, SOAPY_SDR_RX, channel, (double)plan.rate);

	/* buffers: one read of buf_len COMPLEX elements per hop (the reference asks for that many, src/rtl_power.c:694),
	 * of which the first buf_len int16 are the hop buffer (:715-720, SURVEY F10) */
	int16_t *rd = (int16_t *)malloc((size_t)buf_len * 4);
	int16_t *dump = (int16_t *)malloc((size_t)BUFFER_DUMP * 4);
	int16_t *stage = (int16_t *)malloc((size_t)n_hops * (size_t)buf_len * 2);
	const int row_len = rxb200_power_row_len(pp->bin_e, plan.crop);
	double *db = (double *)malloc((size_t)n_hops * (size_t)row_len * sizeof(double));
	int *samples = (int *)malloc((size_t)n_hops * sizeof(int));
	char *row = (char *)malloc(64 + 16 * ((size_t)N + 8));
	const char *hook = getenv("RXB200_MAX_SWEEPS");       /* test hook: report after this many sweeps and exit */
	const long max_sweeps = hook ? atol(hook) : 0;
	long sweeps = 0;
	time_t next_tick = time(NULL) + interval, exit_time = exit_after ? time(NULL) + exit_after : 0;
	int done = 0;
	while (!done && !g_stop) {
		/* ---- one sweep: scanner()'s device side (:679-708) */
		int first_ok = -1, n_ok = 0;
		for (int i = 0; i < n_hops && g_stop < 2; i++) {
			const int64_t f = plan.first_freq + (int64_t)i * plan.freq_step;
			if ((int64_t)SoapySDRDevice_getFrequency(dev, SOAPY_SDR_RX, channel) != f) {
				retune(dev, stream, channel, f, dump, tuner_sleep_usec, tuner_retry_max);
			}
			void *buffs[] = {rd};
			int flags = 0; long long tn = 0;
			int r = SoapySDRDevice_readStream(dev, stream, buffs, (size_t)buf_len, &flags, &tn, 1000000);
			if (r < 0) { fprintf(stderr, "Error: reading stream %d\n", r); continue; }           /* :700-703 */
			if (first_ok < 0) { first_ok = i; }
			if (i != first_ok + n_ok) {
				/* a hop in the middle failed: flush the contiguous run gathered so far, start a new one */
				rxb200_power_group_accumulate(grp, stage + (size_t)first_ok * buf_len, 1, first_ok, first_ok + n_ok);
				first_ok = i; n_ok = 0;
			}
			memcpy(stage + (size_t)i * buf_len, rd, (size_t)buf_len * 2);
			n_ok++;
		}
		if (n_ok > 0) {
			if (rxb200_power_group_accumulate(grp, stage + (size_t)first_ok * buf_len, 1, first_ok, first_ok + n_ok) != RXB200_OK) {
				fprintf(stderr, "rxb200: %s\n", rxb200_last_error());
				break;
			}
		}
		sweeps++;
		const int stream_dry = (first_ok < 0);              /* replay device ran out of samples */
		time_t now = time(NULL);
		const int hooked = max_sweeps && sweeps >= max_sweeps;
		if (now < next_tick && !hooked && !stream_dry) { continue; }
		/* ---- report (:1044-1058) */
		char tstr[50];
		time_string(tstr, sizeof tstr, now);
		if (rxb200_power_group_gather(grp) != RXB200_OK) { fprintf(stderr, "rxb200: %s\n", rxb200_last_error()); break; }
		if (report(out, pw, &plan, db, row_len, samples, row, 64 + 16 * ((size_t)N + 8), tstr) != 0) { break; }
		rxb200_power_group_reset(grp);
		while (time(NULL) >= next_tick) { next_tick += interval; }
		if (single || hooked || stream_dry) { done = 1; }
		if (exit_time && time(NULL) >= exit_time) { done = 1; }
	}
	fprintf(stderr, g_stop ? "\nUser cancel, exiting...\n" : "\nDone, exiting...\n");
	if (out != stdout) { fclose(out); }
	rxb200_power_group_destroy(grp);
	sdr_close(dev, stream);
	return 0;
}
