/* rx_sdr_b200 — drop-in rx_sdr: records I/Q from a SoapySDR device, the format conversions on the GPU (librxb200).
 *
 * Plain mode: rx_sdr's command line (-d -f -g -c -a -s -b -n -p -D -S -I -F -t filename) and its output bytes.  Input
 * and output formats: the same format in and out (written as read), CS16 in and CS8 / CU8 / CF32 out
 * (rxb200_sdr_convert), or CS12 in and CS16 out; any other pair exits 1.  Every read of any length is converted and
 * written.  -n N keeps rx_sdr's rule: a read longer than the count still to record is cut to it and ends the run; the
 * count then drops by each read's length, and once it reaches 0 exactly it no longer limits the run.  The run ends when
 * the device reports an error other than an overflow (a replay device at the end of its data).
 *
 * Capture mode: RXB200_CAPTURE_RATE=<max Hz> with one or more -f records every -f channel from ONE wideband capture.
 * The plan is rxb200_sdr_plan_capture's for the channels and -s (RXB200_CAPTURE_STAGES=2: the two-stage plan of
 * rxb200_fm_plan_capture_two_stage with chain rate -s; RXB200_CAPTURE_STAGES=raster: the raster plan of
 * rxb200_fm_plan_capture_raster, for channels on a common grid); the device is tuned once to the centre at the plan's rate R
 * and read as CS16 in reads of any length, and one rx_sdr I/Q down-converter handle (rxb200_sdr_mix_*) writes channel
 * f's -F samples to <filename>.<f>, f the tuned frequency in Hz.  With -n N every file gets exactly N samples and the
 * run stops; without it every output is written until the stream ends.  '-' as the filename, -I other than CS16, a
 * frequency given twice and a plan above the cap (the message names the rate needed) or, for the raster, above 4096 bins
 * exit 1 before the device is opened, and no file is created.
 *
 * RXB200_DEVICE_RATE=<Hz> with capture mode: the device runs at that rate instead of R.  The plan is the _at planner's
 * (its decimation leaves the resampler's guard band, and a plan above the device rate exits 1 before the device is
 * opened); the device is asked for R_dev, and the rate it reports is what the plan and the resampler
 * (rxb200_plan_resample, rxb200_sdr_mix_set_device_rate) start from, so every read goes to the handle at the device's
 * rate and the files hold the same channels, resampled to R on the GPU.
 *
 * RXB200_DEVICE_FORMAT=CS16|CS8|CU8|CS12 with capture mode: the stream is opened in that format, the read buffer holds
 * -b elements of it, and the handle widens each read to CS16 on the GPU (rxb200_sdr_mix_set_input_format), so the
 * files are those of the same run on the widened CS16 stream.  -I may be left out or name the same format; any other -I
 * exits 1.  An unknown value, or the variable without capture mode, exits 1 before the device is opened.  Without the
 * variable, -I other than CS16 keeps capture mode's refusal.
 */
#include <limits.h>
#include <signal.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <strings.h>
#include <unistd.h>
#include <SoapySDR/Device.h>
#include <SoapySDR/Formats.h>
#include "rxb200.h"
#include "sdr_util.h"

#define BLOCK_DEFAULT (16 * 16384)
#define BLOCK_MIN 512
#define BLOCK_MAX (256 * 16384)
#define MAX_FREQS 1024

static volatile sig_atomic_t g_stop = 0;
static void on_signal(int s) { (void)s; g_stop = 1; }

static void usage(void)
{
	fprintf(stderr,
		"rx_sdr_b200, an I/Q recorder for SoapySDR devices (format conversions on the GPU)\n\n"
		"Usage:\t -f frequency_to_tune_to [Hz]\n"
		"\t[-s samplerate (default: 2048000 Hz)]\n"
		"\t[-d device key/value query (ex: 0, 1, driver=rtlsdr, driver=hackrf)]\n"
		"\t[-g tuner gain(s) (ex: 20, 40, LNA=40,VGA=20,AMP=0)]\n"
		"\t[-c channel number (ex: 0)]\n"
		"\t[-a antenna (ex: 'Tuner 1 50 ohm')]\n"
		"\t[-p ppm_error (default: 0)]\n"
		"\t[-b output_block_size (default: 16 * 16384)]\n"
		"\t[-n number of samples to read (default: 0, infinite)]\n"
		"\t[-I input format, CU8|CS8|CS12|CS16|CF32 (default: CS16)]\n"
		"\t[-F output format, CU8|CS8|CS12|CS16|CF32 (default: CU8)]\n"
		"\t[-S force sync output (default: async)]\n"
		"\t[-D direct_sampling_mode, 0 (default/off), 1 (I), 2 (Q), 3 (no-mod)]\n"
		"\t[-t SDR settings (ex: rfnotch_ctrl=false,dabnotch_ctrlb=true)]\n"
		"\tfilename (a '-' dumps samples to stdout)\n\n"
		"environment: RXB200_CAPTURE_RATE=max_Hz records every -f channel from one capture of at most max_Hz samples/s,\n"
		"each to filename.<frequency>; RXB200_CAPTURE_STAGES=2 plans that capture in two stages, and\n"
		"RXB200_CAPTURE_STAGES=raster as one raster of bins (channels on a common grid, at most 4096 bins);\n"
		"RXB200_DEVICE_RATE=Hz (with capture mode) runs the device at that rate and resamples its stream to the\n"
		"capture's rate on the GPU; RXB200_DEVICE_FORMAT=CS16|CS8|CU8|CS12 (with capture mode) reads the device in\n"
		"that format and widens it to CS16 on the GPU.\n");
	exit(1);
}

static const char *format_of(const char *s)
{
	static const char *names[] = {SOAPY_SDR_CU8, SOAPY_SDR_CS8, SOAPY_SDR_CS12, SOAPY_SDR_CS16, SOAPY_SDR_CF32};
	for (size_t i = 0; i < sizeof names / sizeof names[0]; i++) {
		if (s && !strcasecmp(s, names[i])) { return names[i]; }
	}
	return NULL;
}

static int same(const char *a, const char *b) { return !strcmp(a, b); }

/* the rxb200 output format of -F (input CS16) */
static int out_kind(const char *fmt)
{
	return same(fmt, SOAPY_SDR_CS8) ? RXB200_CVT_CS16_CS8 : same(fmt, SOAPY_SDR_CU8) ? RXB200_CVT_CS16_CU8
	     : same(fmt, SOAPY_SDR_CF32) ? RXB200_CVT_CS16_CF32 : RXB200_SDR_OUT_CS16;
}

static size_t out_bytes(const char *fmt) { return same(fmt, SOAPY_SDR_CF32) ? 8 : same(fmt, SOAPY_SDR_CS16) ? 4 : 2; }

/* "key=value,key=value" to the device's settings */
static void write_settings(SoapySDRDevice *dev, const char *s)
{
	char *c = strdup(s), *save = NULL;
	for (char *kv = strtok_r(c, ",", &save); kv; kv = strtok_r(NULL, ",", &save)) {
		char *eq = strchr(kv, '=');
		if (!eq) { fprintf(stderr, "Ignoring setting '%s' (no '=')\n", kv); continue; }
		*eq = 0;
		if (SoapySDRDevice_writeSetting(dev, kv, eq + 1) != 0) { fprintf(stderr, "Failed to set %s\n", kv); }
	}
	free(c);
}

struct opts {
	const char *query, *gain, *antenna, *settings, *filename, *in_fmt, *out_fmt;
	int in_given;          /* -I was on the command line */
	size_t channel;
	int ppm, direct;
	uint32_t rate, block, n_samples;
	uint32_t freqs[MAX_FREQS];
	int n_freqs;
};

/* device bring-up as rx_sdr does it: rate, frequency, gain, antenna, ppm, then a stream of `fmt` on the channel */
static int open_device(const struct opts *o, const char *fmt, double rate, double freq, SoapySDRDevice **dev,
                       SoapySDRStream **stream)
{
	SoapySDRKwargs none = {0, NULL, NULL};
	size_t ch = o->channel;
	*dev = SoapySDRDevice_makeStrArgs(o->query);
	if (!*dev) { fprintf(stderr, "Failed to open sdr device matching '%s'.\n", o->query); return -1; }
	if (o->direct) {
		char v[16];
		snprintf(v, sizeof v, "%d", o->direct);
		SoapySDRDevice_writeSetting(*dev, "direct_samp", v);
	}
	SoapySDRDevice_setSampleRate(*dev, SOAPY_SDR_RX, ch, rate);
	fprintf(stderr, "Sampling at %.0f S/s.\n", rate);
	SoapySDRDevice_setFrequency(*dev, SOAPY_SDR_RX, ch, freq, NULL);
	fprintf(stderr, "Tuned to %.0f Hz.\n", freq);
	sdr_set_gain(*dev, ch, o->gain);
	if (o->antenna && SoapySDRDevice_setAntenna(*dev, SOAPY_SDR_RX, ch, o->antenna) != 0) {
		fprintf(stderr, "Failed to set antenna");
	}
	if (o->ppm) { SoapySDRDevice_setFrequencyCorrection(*dev, SOAPY_SDR_RX, ch, (double)o->ppm); }
	*stream = SoapySDRDevice_setupStream(*dev, SOAPY_SDR_RX, fmt, &ch, 1, &none);
	if (!*stream) { fprintf(stderr, "Failed to setup stream\n"); return -1; }
	if (o->settings) { write_settings(*dev, o->settings); }
	if (SoapySDRDevice_activateStream(*dev, *stream, 0, 0, 0) != 0) { fprintf(stderr, "Failed to activate stream\n"); return -1; }
	return 0;
}

/* one read of at most `elems` complex elements; < 0 when the stream has ended (overflows are skipped) */
static int read_some(SoapySDRDevice *dev, SoapySDRStream *stream, void *buf, size_t elems)
{
	while (!g_stop) {
		void *buffs[] = {buf};
		int flags = 0;
		long long t_ns = 0;
		const int r = SoapySDRDevice_readStream(dev, stream, buffs, elems, &flags, &t_ns, 1000000);
		if (r >= 0) { return r; }
		if (r != SOAPY_SDR_OVERFLOW) { return r; }
		fprintf(stderr, "O");
	}
	return -1;
}

static int plain_mode(const struct opts *o)
{
	const size_t in_size = SoapySDR_formatToSize(o->in_fmt), cvt = !same(o->in_fmt, o->out_fmt);
	void *buf = malloc((size_t)o->block * 4 > (size_t)o->block * in_size ? (size_t)o->block * 4 : (size_t)o->block * in_size);
	void *out = malloc((size_t)o->block * 8);
	SoapySDRDevice *dev = NULL;
	SoapySDRStream *stream = NULL;
	if (open_device(o, o->in_fmt, o->rate, o->n_freqs ? o->freqs[o->n_freqs - 1] : 100000000, &dev, &stream) != 0) { return 1; }
	FILE *f = same(o->filename, "-") ? stdout : fopen(o->filename, "wb");
	if (!f) { fprintf(stderr, "Failed to open %s\n", o->filename); return 1; }
	fprintf(stderr, "Using output format: %s (input format %s, %d bytes per element)\n", o->out_fmt, o->in_fmt, (int)in_size);
	uint32_t left = o->n_samples;
	int rc = 0;
	while (!g_stop) {
		const int r = read_some(dev, stream, buf, o->block);
		if (r < 0) { break; }
		size_t n = (size_t)r;
		int last = 0;
		if (left > 0 && left < (uint32_t)r) { n = left; last = 1; }
		const void *w = buf;
		size_t bytes = n * in_size;
		if (cvt && n) {
			const int kind = same(o->in_fmt, SOAPY_SDR_CS12) ? RXB200_CVT_CS12_CS16 : out_kind(o->out_fmt);
			if (rxb200_sdr_convert(kind, buf, n, out, 0) != RXB200_OK) {
				fprintf(stderr, "rxb200_sdr_convert: %s\n", rxb200_last_error());
				rc = 1;
				break;
			}
			w = out;
			bytes = n * (kind == RXB200_CVT_CS12_CS16 ? 4 : out_bytes(o->out_fmt));
		}
		if (fwrite(w, 1, bytes, f) != bytes) { fprintf(stderr, "Short write, samples lost, exiting!\n"); rc = 1; break; }
		if (last) { break; }
		if (left > 0) { left -= (uint32_t)r; }
	}
	if (f != stdout) { fclose(f); }
	SoapySDRDevice_deactivateStream(dev, stream, 0, 0);
	sdr_close(dev, stream);
	free(buf);
	free(out);
	return rc;
}

static int capture_mode(const struct opts *o, const char *cap_env, long long dev_rate, int dev_fmt, const char *dev_fmt_name)
{
	const int K = o->n_freqs;
	if (same(o->filename, "-")) { fprintf(stderr, "Capture mode (RXB200_CAPTURE_RATE) writes one file per channel, not to '-'.\n"); return 1; }
	if (!getenv("RXB200_DEVICE_FORMAT")) {
		if (!same(o->in_fmt, SOAPY_SDR_CS16)) { fprintf(stderr, "Capture mode (RXB200_CAPTURE_RATE) reads CS16, not %s.\n", o->in_fmt); return 1; }
	} else if (o->in_given && !same(o->in_fmt, dev_fmt_name)) {
		fprintf(stderr, "Capture mode reads the device in RXB200_DEVICE_FORMAT=%s, not -I %s.\n", dev_fmt_name, o->in_fmt);
		return 1;
	}
	for (int i = 0; i < K; i++) {
		for (int j = 0; j < i; j++) {
			if (o->freqs[i] == o->freqs[j]) { fprintf(stderr, "Capture mode (RXB200_CAPTURE_RATE): %u Hz is given twice.\n", o->freqs[i]); return 1; }
		}
	}
	const char *stages = getenv("RXB200_CAPTURE_STAGES");
	const enum capture_kind kind = stages && !strcmp(stages, "raster") ? CAPTURE_RASTER
	                             : stages && atoi(stages) == 2         ? CAPTURE_TWO_STAGE
	                                                                   : CAPTURE_SINGLE;
	int64_t tuned[MAX_FREQS];
	int chans[MAX_FREQS];
	for (int i = 0; i < K; i++) { tuned[i] = o->freqs[i]; }
	struct capture_plan pl;
	rxb200_resampler rs = {1, 1, 0, NULL, 15};
	if (capture_plan(kind, tuned, K, (int)o->rate, cap_env, 1, dev_rate, &pl, chans) != 0) { return 1; }
	fputs(pl.banner, stderr);
	if (dev_rate && device_resampler(dev_rate, pl.capture_rate, pl.span, &rs) != 0) { return 1; }
	SoapySDRDevice *dev = NULL;
	SoapySDRStream *stream = NULL;
	if (open_device(o, dev_fmt_name, dev_rate ? dev_rate : pl.capture_rate, (double)pl.centre_hz, &dev, &stream) != 0) { return 1; }
	const long long got = dev_rate ? sdr_device_rate(dev, o->channel, dev_rate) : 0;
	if (got < 0) { sdr_close(dev, stream); return 1; }
	if (got != dev_rate) {
		/* the device runs at another rate than it was asked for: plan and resample from the rate it reports */
		fprintf(stderr, "The device reports %lld Hz, not RXB200_DEVICE_RATE=%lld Hz: planning again.\n", got, dev_rate);
		capture_plan_release(&pl);
		free((void *)rs.taps);
		rs.taps = NULL;
		if (capture_plan(kind, tuned, K, (int)o->rate, cap_env, 1, got, &pl, chans) != 0) { sdr_close(dev, stream); return 1; }
		fputs(pl.banner, stderr);
		if (device_resampler(got, pl.capture_rate, pl.span, &rs) != 0) { sdr_close(dev, stream); return 1; }
	}
	rxb200_sdr_mix *h = NULL;
	const int rc0 = kind == CAPTURE_RASTER ? rxb200_sdr_mix_create_raster(pl.n_bins, chans, K, &pl.ddc, 0, &h)
	              : kind == CAPTURE_TWO_STAGE
	                  ? rxb200_sdr_mix_create_two_stage(pl.capture_rate, pl.n_bins, chans, K, &pl.ddc, &pl.fine, 0, &h)
	                  : rxb200_sdr_mix_create(pl.capture_rate, chans, K, &pl.ddc, 0, &h);
	if (rc0 != RXB200_OK) { fprintf(stderr, "rxb200_sdr_mix_create: %s\n", rxb200_last_error()); return 1; }
	if (rs.taps && rxb200_sdr_mix_set_device_rate(h, &rs) != RXB200_OK) { fprintf(stderr, "rxb200: %s\n", rxb200_last_error()); return 1; }
	if (dev_fmt != RXB200_IN_CS16 && rxb200_sdr_mix_set_input_format(h, dev_fmt) != RXB200_OK) { fprintf(stderr, "rxb200: %s\n", rxb200_last_error()); return 1; }
	free((void *)rs.taps);
	FILE *files[MAX_FREQS];
	for (int k = 0; k < K; k++) {
		char name[4096];
		snprintf(name, sizeof name, "%s.%u", o->filename, o->freqs[k]);
		if (!(files[k] = fopen(name, "wb"))) { fprintf(stderr, "Failed to open %s\n", name); return 1; }
	}
	const int fmt = out_kind(o->out_fmt);
	/* each read's outputs per channel come from the handle (rxb200_sdr_mix_decimated_len counts device int16 once a
	 * resampler is attached), and the output buffer grows to hold them */
	const size_t E = out_bytes(o->out_fmt);
	size_t stride = o->block / (size_t)pl.decim + 2;
	int16_t *buf = malloc((size_t)o->block * device_format_bytes(dev_fmt));   /* -b elements of the device's format */
	unsigned char *out = malloc((size_t)K * stride * E);
	unsigned long long written = 0;
	int rc = 0;
	while (!g_stop && !(o->n_samples && written >= o->n_samples)) {
		const int r = read_some(dev, stream, buf, o->block);
		if (r < 0) { break; }
		size_t n = 0, need = 0;
		rxb200_sdr_mix_decimated_len(h, 2 * (size_t)r, &need);
		if (need > stride) {
			unsigned char *grown = realloc(out, (size_t)K * need * E);
			if (!grown) { fprintf(stderr, "Out of memory for %zu outputs per channel\n", need); rc = 1; break; }
			out = grown;
			stride = need;
		}
		if (rxb200_sdr_mix_process(h, buf, 2 * (size_t)r, fmt, out, (size_t)K * stride, stride, &n) != RXB200_OK) {
			fprintf(stderr, "rxb200_sdr_mix_process: %s\n", rxb200_last_error());
			rc = 1;
			break;
		}
		if (o->n_samples && written + n > o->n_samples) { n = (size_t)(o->n_samples - written); }
		for (int k = 0; k < K && n; k++) {
			if (fwrite(out + (size_t)k * stride * E, E, n, files[k]) != n) { fprintf(stderr, "Short write, samples lost, exiting!\n"); rc = 1; }
		}
		written += n;
		if (rc) { break; }
	}
	for (int k = 0; k < K; k++) { fclose(files[k]); }
	rxb200_sdr_mix_destroy(h);
	SoapySDRDevice_deactivateStream(dev, stream, 0, 0);
	sdr_close(dev, stream);
	free(buf); free(out);
	capture_plan_release(&pl);
	return rc;
}

int main(int argc, char **argv)
{
	struct opts o;
	memset(&o, 0, sizeof o);
	o.query = "";
	o.rate = 2048000;
	o.block = BLOCK_DEFAULT;
	o.in_fmt = SOAPY_SDR_CS16;
	o.out_fmt = SOAPY_SDR_CU8;
	int opt;
	while ((opt = getopt(argc, argv, "d:f:g:c:a:s:b:n:p:D:SI:F:t:")) != -1) {
		switch (opt) {
		case 'd': o.query = optarg; break;
		case 'f':
			if (o.n_freqs == MAX_FREQS) { fprintf(stderr, "Too many frequencies (at most %d)\n", MAX_FREQS); return 1; }
			o.freqs[o.n_freqs++] = (uint32_t)parse_scaled(optarg);
			break;
		case 'g': o.gain = optarg; break;
		case 'c': o.channel = (size_t)atoi(optarg); break;
		case 'a': o.antenna = optarg; break;
		case 's': o.rate = (uint32_t)parse_scaled(optarg); break;
		case 'p': o.ppm = atoi(optarg); break;
		case 'b': o.block = (uint32_t)atof(optarg); break;
		case 'n': o.n_samples = (uint32_t)parse_scaled(optarg); break;
		case 'S': break;                            /* reads are synchronous either way */
		case 'I':
			if (!(o.in_fmt = format_of(optarg))) { fprintf(stderr, "Unsupported input format: %s\n", optarg); return 1; }
			o.in_given = 1;
			break;
		case 'F':
			if (!(o.out_fmt = format_of(optarg))) { fprintf(stderr, "Unsupported output format: %s\n", optarg); return 1; }
			break;
		case 'D': o.direct = atoi(optarg); break;
		case 't': o.settings = optarg; break;
		default: usage();
		}
	}
	/* capture mode with RXB200_DEVICE_FORMAT widens any -I on the GPU and checks -I against the variable itself */
	const char *cap_env = getenv("RXB200_CAPTURE_RATE");
	const int capture = cap_env && *cap_env && o.n_freqs >= 1;
	if (!(capture && getenv("RXB200_DEVICE_FORMAT")) && !same(o.in_fmt, o.out_fmt) && !same(o.in_fmt, SOAPY_SDR_CS16) &&
	    !(same(o.in_fmt, SOAPY_SDR_CS12) && same(o.out_fmt, SOAPY_SDR_CS16))) {
		fprintf(stderr, "Unsupported input/output conversion: %s to %s\n", o.in_fmt, o.out_fmt);
		return 1;
	}
	if (argc <= optind) { usage(); }
	o.filename = argv[optind];
	if (o.block < BLOCK_MIN || o.block > BLOCK_MAX) {
		fprintf(stderr, "Output block size wrong value, falling back to default\n");
		fprintf(stderr, "Minimal length: %u\nMaximal length: %u\n", BLOCK_MIN, BLOCK_MAX);
		o.block = BLOCK_DEFAULT;
	}
	signal(SIGINT, on_signal);
	signal(SIGTERM, on_signal);
	signal(SIGPIPE, on_signal);
	const long long dev_rate = device_rate_env(capture, "capture mode (RXB200_CAPTURE_RATE with -f)");
	if (dev_rate < 0) { return 1; }
	const char *dev_fmt_name = NULL;
	const int dev_fmt = device_format_env(capture, "capture mode (RXB200_CAPTURE_RATE with -f)", &dev_fmt_name);
	if (dev_fmt < 0) { return 1; }
	if (capture) { return capture_mode(&o, cap_env, dev_rate, dev_fmt, dev_fmt_name); }
	return plain_mode(&o);
}
