/* rx_fm_b200 — drop-in for rx_tools' rx_fm whose DSP runs on an H100 through librxb200.so.
 *
 * Same command line (option string of src/rtl_fm.c:1224), same raw int16 / WAV output, same
 * SoapySDR CS16 stream surface.  The host side is our own code: three threads (stream reader ->
 * demodulator -> writer) joined by small bounded queues, so — unlike the reference's lock/signal
 * hand-off (src/rtl_fm.c:858-862, SURVEY F12) — no chunk is ever overwritten before it was consumed
 * and a file replay is deterministic.  Every DSP stage of rtlsdr_callback()+full_demod() is one call:
 * rxb200_fm_process_read(), one stream read (<= 131072 complex) per call, like the reference's chunks
 * (a read re-blocked to the library's chunk granularity with -o N).
 */
#include <errno.h>
#include <math.h>
#include <pthread.h>
#include <signal.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>
#include "sdr_util.h"
#include "rxb200.h"

#define CHUNK_COMPLEX 131072          /* MAXIMUM_BUF_LENGTH / 2, src/rtl_fm.c:80-82, :871 */
#define MUTE_AFTER_HOP 4096           /* BUFFER_DUMP, src/rtl_fm.c:83, :1047 */
#define MAX_FREQS 1000
#define QDEPTH 4

static volatile sig_atomic_t g_stop = 0;
static void on_signal(int s) { (void)s; g_stop = 1; }

/* ---- bounded queue of buffers ---- */
typedef struct { int16_t *data; size_t n; int eof; } Slot;
typedef struct {
	Slot slot[QDEPTH];
	int head, tail, count;
	pthread_mutex_t m; pthread_cond_t not_empty, not_full;
} Queue;
static void q_init(Queue *q, size_t cap_int16)
{
	memset(q, 0, sizeof *q);
	for (int i = 0; i < QDEPTH; i++) { q->slot[i].data = (int16_t *)malloc(cap_int16 * sizeof(int16_t)); }
	pthread_mutex_init(&q->m, NULL); pthread_cond_init(&q->not_empty, NULL); pthread_cond_init(&q->not_full, NULL);
}
static Slot *q_begin_put(Queue *q)
{
	pthread_mutex_lock(&q->m);
	while (q->count == QDEPTH) { pthread_cond_wait(&q->not_full, &q->m); }
	Slot *s = &q->slot[q->tail];
	pthread_mutex_unlock(&q->m);
	return s;
}
static void q_end_put(Queue *q)
{
	pthread_mutex_lock(&q->m);
	q->tail = (q->tail + 1) % QDEPTH; q->count++;
	pthread_cond_signal(&q->not_empty);
	pthread_mutex_unlock(&q->m);
}
static Slot *q_begin_get(Queue *q)
{
	pthread_mutex_lock(&q->m);
	while (q->count == 0) { pthread_cond_wait(&q->not_empty, &q->m); }
	Slot *s = &q->slot[q->head];
	pthread_mutex_unlock(&q->m);
	return s;
}
static void q_end_get(Queue *q)
{
	pthread_mutex_lock(&q->m);
	q->head = (q->head + 1) % QDEPTH; q->count--;
	pthread_cond_signal(&q->not_full);
	pthread_mutex_unlock(&q->m);
}

/* ---- program state ---- */
static struct {
	SoapySDRDevice *dev; SoapySDRStream *stream; size_t channel;
	const char *dev_query, *gain_str, *antenna, *filename;
	uint32_t freqs[MAX_FREQS]; int freq_len, freq_now;
	rxb200_fm_cli cli; rxb200_fm_derived der;
	int conseq_squelch, terminate_on_squelch, squelch_zero, wav, edge, ppm, custom_ppm, bandwidth, verbosity;
	int direct_sampling, rtlagc;
	int print_levels, level_no, level_max, level_max_max; double level_sum;   /* -L (src/rtl_fm.c:96-100) */
	volatile int mute;                 /* int16 to zero at the start of the next read */
	size_t multiple;                   /* chunk granularity librxb200 accepts, int16 */
	size_t min_chunk;                  /* shortest chunk handed on, int16 */
	int failed;                        /* a library call failed: exit status 1 */
	rxb200_fm *fm;
	FILE *out;
	Queue q_raw, q_pcm;
	pthread_mutex_t hop_m;
} G;

static void usage(void)
{
	fprintf(stderr,
		"rx_fm_b200, rx_fm with the demodulator on an H100 GPU\n\n"
		"Use:\trx_fm_b200 -f freq [-options] [filename]\n"
		"\t-f frequency_to_tune_to [Hz] (repeat for scanning, ranges a:b:step)\n"
		"\t[-M modulation (default: fm)] fm|nbfm|nfm, wbfm|wfm, raw|iq, am, usb, lsb\n"
		"\t[-s sample_rate (default: 24k)] [-r resample_rate] [-d device] [-C channel] [-a antenna]\n"
		"\t[-g gain] [-w bandwidth] [-l squelch_level] [-t squelch_delay] [-p ppm] [-o oversampling]\n"
		"\t[-E edge|dc|adc|rdc|deemp|direct|no-mod|offset|agc|zero|wav] [-q rdc_block_const]\n"
		"\t[-F fir_size] [-A std|fast|lut|ale] [-c us|eu|N] [-L N] [-v]\n"
		"\tfilename ('-' means stdout)\n");
	exit(1);
}

static void add_range(char *arg)
{
	/* -f start:stop:step (src/rtl_fm.c:1052-1070) */
	char *stop = strchr(arg, ':'), *step = stop ? strchr(stop + 1, ':') : NULL;
	if (!stop || !step) { return; }
	*stop++ = 0; *step++ = 0;
	for (int f = (int)parse_scaled(arg); f <= (int)parse_scaled(stop) && G.freq_len < MAX_FREQS; f += (int)parse_scaled(step)) {
		G.freqs[G.freq_len++] = (uint32_t)f;
	}
}

static uint32_t capture_freq(int idx)
{
	/* optimal_settings(): capture_freq = freq + capture_rate/4 (+ edge*rate_in/2) (src/rtl_fm.c:976-993);
	 * wbfm adds 16 kHz to every tuned frequency (:1006-1011) */
	int64_t f = (int64_t)G.freqs[idx] + (G.cli.wbfm ? 16000 : 0) + G.der.capture_freq_offset;
	if (G.edge) { f += (int64_t)(G.der.params.rate_out * G.der.params.post_downsample) / 2; }
	return (uint32_t)f;
}

static void write_wav_header(void)
{
	/* generate_header(), src/rtl_fm.c:1174-1206: sizes unknown (0xFFFFFFFF), PCM 16 bit */
	const int raw = (G.der.params.mode == RXB200_MODE_RAW);
	uint32_t rate = (uint32_t)G.der.output_rate, brate = rate * 2u * (raw ? 2u : 1u);
	unsigned char h[44] = {'R','I','F','F',0xFF,0xFF,0xFF,0xFF,'W','A','V','E','f','m','t',' ',16,0,0,0,1,0,
	                       (unsigned char)(raw ? 2 : 1),0, 0,0,0,0, 0,0,0,0, (unsigned char)(raw ? 4 : 2),0,16,0,
	                       'd','a','t','a',0xFF,0xFF,0xFF,0xFF};
	for (int i = 0; i < 4; i++) { h[24 + i] = (unsigned char)(rate >> (8 * i)); h[28 + i] = (unsigned char)(brate >> (8 * i)); }
	fwrite(h, 1, sizeof h, G.out);
}

/* ---- threads ---- */
static void *reader_thread(void *arg)
{
	(void)arg;
	/* what a read left over past the library's chunk granularity is carried into the next slot, never dropped: the
	 * stream stays continuous whatever lengths the device returns (the reference hands any length on, :894-899).
	 * Where every length is accepted (see main) nothing is carried but a read below min_chunk */
	static int16_t rem[8192];
	size_t rem_n = 0;
	SoapySDRDevice_activateStream(G.dev, G.stream, 0, 0, 0);
	for (;;) {
		Slot *s = q_begin_put(&G.q_raw);
		memcpy(s->data, rem, rem_n * sizeof(int16_t));
		void *buffs[] = {s->data + rem_n};
		int flags = 0; long long t_ns = 0;
		int r = g_stop ? -1 : SoapySDRDevice_readStream(G.dev, G.stream, buffs, CHUNK_COMPLEX - (rem_n + 1) / 2, &flags, &t_ns, 1000000);
		if (r == SOAPY_SDR_OVERFLOW) { fprintf(stderr, "O"); fflush(stderr); continue; }      /* :901-905 */
		if (r <= 0) {
			if (!g_stop) { fprintf(stderr, "readStream read failed: %d\n", r); }
			s->n = 0; s->eof = 1; q_end_put(&G.q_raw);
			break;
		}
		size_t n16 = rem_n + (size_t)r * 2;
		/* librxb200 chunk granularity: the excess opens the next slot; so does all of a read shorter than the minimum */
		const size_t over = n16 < G.min_chunk ? n16 : n16 % G.multiple;
		n16 -= over;
		memcpy(rem, s->data + n16, over * sizeof(int16_t));
		rem_n = over;
		if (n16 == 0) { continue; }                      /* less than one granule so far: same slot again */
		pthread_mutex_lock(&G.hop_m);
		if (G.mute) {                                  /* zero the first samples after a hop (:839-843) */
			size_t z = (size_t)G.mute < n16 ? (size_t)G.mute : n16;
			memset(s->data, 0, z * sizeof(int16_t));
			G.mute = 0;
		}
		pthread_mutex_unlock(&G.hop_m);
		s->n = n16; s->eof = 0;
		q_end_put(&G.q_raw);
	}
	return NULL;
}

static void hop_to_next(void)
{
	/* controller_thread_fn's hop (src/rtl_fm.c:1039-1048) */
	if (G.freq_len <= 1) { return; }
	SoapySDRKwargs none = {0, NULL, NULL};
	pthread_mutex_lock(&G.hop_m);
	G.freq_now = (G.freq_now + 1) % G.freq_len;
	SoapySDRDevice_setFrequency(G.dev, SOAPY_SDR_RX, 0, (double)capture_freq(G.freq_now), &none);
	G.mute = MUTE_AFTER_HOP;
	pthread_mutex_unlock(&G.hop_m);
}

static void *demod_thread(void *arg)
{
	(void)arg;
	const int squelch = G.der.params.squelch_level;
	for (;;) {
		Slot *in = q_begin_get(&G.q_raw);
		if (in->eof) { q_end_get(&G.q_raw); break; }
		Slot *out = q_begin_put(&G.q_pcm);
		size_t n_pcm = 0;
		/* a slot re-blocked for -o N is a read rxb200_fm_process(h, x, n, n) takes, and runs exactly as that call */
		int rc = rxb200_fm_process_read(G.fm, in->data, in->n, out->data, 2 * CHUNK_COMPLEX, &n_pcm);
		q_end_get(&G.q_raw);
		if (rc != RXB200_OK) { fprintf(stderr, "rxb200: %s\n", rxb200_last_error()); g_stop = 1; G.failed = 1; n_pcm = 0; }
		if (G.print_levels && rc == RXB200_OK) {                                  /* :792-806, one chunk per call */
			int sr = 0; size_t nl = 0;
			if (rxb200_fm_levels(G.fm, &sr, 1, &nl) == RXB200_OK && nl == 1) {
				--G.level_no;
				G.level_sum += sr;
				if (G.level_max < sr) { G.level_max = sr; }
				if (G.level_max_max < sr) { G.level_max_max = sr; }
				if (!G.level_no) {
					G.level_no = G.print_levels;
					fprintf(stderr, "%f, %d, %d, %d\n", G.level_sum / G.print_levels, G.level_max, G.level_max_max, squelch);
					G.level_max = 0; G.level_sum = 0;
				}
			}
		}
		int hits = 0;
		if (squelch) { rxb200_fm_squelch_hits(G.fm, &hits); }
		const int squelch_active = squelch && hits > G.conseq_squelch;            /* :928 */
		if (squelch_active && !G.squelch_zero) {                                  /* :929-933: nothing is written, hop */
			/* -t <negative> sets terminate_on_squelch in the reference too (:1270-1275), but nothing there ever reads
			 * it (exit_flag is never set, :925): the stream keeps running, and so does this one */
			hop_to_next();
			out->n = 0; out->eof = 0; q_end_put(&G.q_pcm);
			continue;
		}
		if (squelch_active && G.squelch_zero) { memset(out->data, 0, n_pcm * sizeof(int16_t)); }   /* :935-936 */
		out->n = n_pcm; out->eof = 0;
		q_end_put(&G.q_pcm);
	}
	Slot *out = q_begin_put(&G.q_pcm);
	out->n = 0; out->eof = 1;
	q_end_put(&G.q_pcm);
	return NULL;
}

static void *writer_thread(void *arg)
{
	(void)arg;
	for (;;) {
		Slot *s = q_begin_get(&G.q_pcm);
		if (s->eof) { q_end_get(&G.q_pcm); break; }
		if (s->n && fwrite(s->data, 2, s->n, G.out) != s->n) { g_stop = 1; }
		q_end_get(&G.q_pcm);
	}
	fflush(G.out);
	return NULL;
}

int main(int argc, char **argv)
{
	int opt;
	memset(&G, 0, sizeof G);
	G.dev_query = ""; G.conseq_squelch = 10;
	G.cli.mode = RXB200_MODE_FM; G.cli.custom_atan = -1; G.cli.deemph = -1; G.cli.post_downsample = 1; G.cli.time_constant_us = 75;
	pthread_mutex_init(&G.hop_m, NULL);
	while ((opt = getopt(argc, argv, "a:C:d:f:g:s:b:l:L:o:t:r:p:E:q:F:A:M:c:h:w:v")) != -1) {
		switch (opt) {
		case 'a': G.antenna = optarg; break;
		case 'C': G.channel = (size_t)atoi(optarg); break;
		case 'd': G.dev_query = optarg; break;
		case 'f':
			if (strchr(optarg, ':')) { char *c = strdup(optarg); add_range(c); free(c); }
			else if (G.freq_len < MAX_FREQS) { G.freqs[G.freq_len++] = (uint32_t)parse_scaled(optarg); }
			break;
		case 'g': G.gain_str = optarg; break;
		case 'l': G.cli.squelch_level = (int)atof(optarg); break;
		case 'L': G.print_levels = (int)atof(optarg); break;     /* src/rtl_fm.c:1253 */
		case 's': G.cli.rate_s = (int)(uint32_t)parse_scaled(optarg); break;
		case 'r': G.cli.rate_r = (int)parse_scaled(optarg); break;
		case 'o': fprintf(stderr, "Warning: -o is very buggy\n"); G.cli.post_downsample = (int)atof(optarg); break;
		case 't':
			G.conseq_squelch = (int)atof(optarg);
			if (G.conseq_squelch < 0) { G.conseq_squelch = -G.conseq_squelch; G.terminate_on_squelch = 1; }
			break;
		case 'p': G.ppm = atoi(optarg); G.custom_ppm = 1; break;
		case 'E':
			if (!strcmp(optarg, "edge")) { G.edge = 1; }
			if (!strcmp(optarg, "dc") || !strcmp(optarg, "adc")) { G.cli.dc_block_audio = 1; }
			if (!strcmp(optarg, "rdc")) { G.cli.dc_block_raw = 1; }
			if (!strcmp(optarg, "deemp")) { G.cli.deemph = 1; }
			if (!strcmp(optarg, "direct")) { G.direct_sampling = 1; }
			if (!strcmp(optarg, "no-mod")) { G.direct_sampling = 3; }
			if (!strcmp(optarg, "offset")) { G.cli.offset_tuning = 1; }
			if (!strcmp(optarg, "rtlagc") || !strcmp(optarg, "agc")) { G.rtlagc = 1; }
			if (!strcmp(optarg, "zero")) { G.squelch_zero = 1; }
			if (!strcmp(optarg, "wav")) { G.wav = 1; }
			break;
		case 'q': G.cli.rdc_block_const = atoi(optarg); break;
		case 'F': G.cli.use_F = 1; G.cli.comp_fir_size = atoi(optarg); break;
		case 'A':
			if (!strcmp(optarg, "std")) { G.cli.custom_atan = RXB200_ATAN_STD; }
			if (!strcmp(optarg, "fast")) { G.cli.custom_atan = RXB200_ATAN_FAST; }
			if (!strcmp(optarg, "lut")) { G.cli.custom_atan = RXB200_ATAN_LUT; }
			if (!strcmp(optarg, "ale")) { G.cli.custom_atan = RXB200_ATAN_ALE; }
			break;
		case 'M':
			if (!strcmp(optarg, "nbfm") || !strcmp(optarg, "nfm") || !strcmp(optarg, "fm")) { G.cli.mode = RXB200_MODE_FM; }
			if (!strcmp(optarg, "raw") || !strcmp(optarg, "iq")) { G.cli.mode = RXB200_MODE_RAW; }
			if (!strcmp(optarg, "am")) { G.cli.mode = RXB200_MODE_AM; }
			if (!strcmp(optarg, "usb")) { G.cli.mode = RXB200_MODE_USB; }
			if (!strcmp(optarg, "lsb")) { G.cli.mode = RXB200_MODE_LSB; }
			if (!strcmp(optarg, "wbfm") || !strcmp(optarg, "wfm")) {
				/* the preset also resets -s/-r/-A/-E deemp given earlier on the command line (src/rtl_fm.c:1331-1341) */
				G.cli.wbfm = 1; G.cli.mode = RXB200_MODE_FM; G.cli.rate_s = 0; G.cli.rate_r = 0;
				G.cli.custom_atan = -1; G.cli.deemph = -1; G.cli.squelch_level = 0;
			}
			break;
		case 'c':
			if (!strcmp(optarg, "us")) { G.cli.time_constant_us = 75; }
			else if (!strcmp(optarg, "eu")) { G.cli.time_constant_us = 50; }
			else { G.cli.time_constant_us = (int)atof(optarg); }
			break;
		case 'v': G.verbosity++; break;
		case 'w':
			G.bandwidth = (int)parse_scaled(optarg);
			if (G.bandwidth) { G.cli.offset_tuning = 1; }
			break;
		default: usage();
		}
	}
	if (G.freq_len == 0) { fprintf(stderr, "Please specify a frequency.\n"); usage(); }
	if (G.freq_len > 1 && G.cli.squelch_level == 0) {
		fprintf(stderr, "Please specify a squelch level.  Required for scanning multiple frequencies.\n");
		return 1;
	}
	if (G.freq_len > 1) { G.terminate_on_squelch = 0; }
	G.filename = (argc <= optind) ? "-" : argv[optind];
	if (rxb200_fm_derive(&G.cli, &G.der) != RXB200_OK) { fprintf(stderr, "rxb200: %s\n", rxb200_last_error()); return 1; }
	if (G.der.params.post_downsample <= 1) {
		/* no -o: every read is handed on as it was read, one rxb200_fm_process_read per read, like the reference's
		 * full_demod per read, reads too short to complete a boxcar included.  Only a read with fifth_order passes
		 * shorter than 2^P complex samples (for which the reference reads before its buffer), or one too short to
		 * complete a boxcar when a per-chunk stage is on (the reference divides by its empty length), waits for the next */
		const rxb200_fm_params *q = &G.der.params;
		const int P = q->downsample_passes;
		const int per_chunk = q->squelch_level || q->dc_block_audio || q->dc_block_raw || G.print_levels;
		G.multiple = 2;
		G.min_chunk = P ? (size_t)2 << P : (per_chunk ? 2 * (size_t)q->downsample : 2);
	} else {   /* -o N: chunk granularity accepted by the library: 16 int16 and 2*2^P int16 */
		size_t m = (size_t)2 << G.der.params.downsample_passes;
		G.multiple = m > 16 ? m : 16;
		G.min_chunk = 0;
	}
	G.der.params.report_levels = G.print_levels ? 1 : 0;
	G.level_no = 1;
	if (rxb200_fm_create(&G.der.params, 0, 1, &G.fm) != RXB200_OK) { fprintf(stderr, "rxb200: %s\n", rxb200_last_error()); return 1; }

	if (sdr_open(G.dev_query, G.channel, &G.dev, &G.stream) != 0) {
		fprintf(stderr, "Failed to open sdr device matching '%s'.\n", G.dev_query);
		return 1;
	}
	struct sigaction sa; memset(&sa, 0, sizeof sa); sa.sa_handler = on_signal;
	sigaction(SIGINT, &sa, NULL); sigaction(SIGTERM, &sa, NULL); sigaction(SIGQUIT, &sa, NULL);
	signal(SIGPIPE, SIG_IGN);
	if (G.antenna && SoapySDRDevice_setAntenna(G.dev, SOAPY_SDR_RX, G.channel, G.antenna) != 0) { fprintf(stderr, "Failed to set antenna"); }
	sdr_set_gain(G.dev, G.channel, G.gain_str);
	SoapySDRDevice_setGainMode(G.dev, SOAPY_SDR_RX, G.channel, G.rtlagc);
	if (G.custom_ppm) { SoapySDRDevice_setFrequencyCorrection(G.dev, SOAPY_SDR_RX, G.channel, (double)G.ppm); }
	if (G.bandwidth) { SoapySDRDevice_setBandwidth(G.dev, SOAPY_SDR_RX, G.channel, (double)G.bandwidth); }
	if (G.direct_sampling) { SoapySDRDevice_writeSetting(G.dev, "direct_samp", G.direct_sampling == 1 ? "1" : "3"); }
	if (G.cli.offset_tuning) { SoapySDRDevice_writeSetting(G.dev, "offset_tune", "true"); }
	{
		SoapySDRKwargs none = {0, NULL, NULL};
		SoapySDRDevice_setFrequency(G.dev, SOAPY_SDR_RX, G.channel, (double)capture_freq(0), &none);
		SoapySDRDevice_setSampleRate(G.dev, SOAPY_SDR_RX, G.channel, (double)G.der.capture_rate);
	}
	fprintf(stderr, "Oversampling input by: %ix.\n", G.der.params.downsample);
	fprintf(stderr, "Oversampling output by: %ix.\n", G.der.params.post_downsample);
	fprintf(stderr, "Output at %u Hz.\n", (unsigned)G.der.params.rate_out);

	if (!strcmp(G.filename, "-")) { G.out = stdout; }
	else if (!(G.out = fopen(G.filename, "wb"))) { fprintf(stderr, "Failed to open %s\n", G.filename); return 1; }
	if (G.wav) { write_wav_header(); }

	q_init(&G.q_raw, 2 * CHUNK_COMPLEX);
	q_init(&G.q_pcm, 2 * CHUNK_COMPLEX);
	pthread_t tr, td, tw;
	pthread_create(&tw, NULL, writer_thread, NULL);
	pthread_create(&td, NULL, demod_thread, NULL);
	pthread_create(&tr, NULL, reader_thread, NULL);
	pthread_join(tr, NULL); pthread_join(td, NULL); pthread_join(tw, NULL);
	if (G.out != stdout) { fclose(G.out); }
	rxb200_fm_destroy(G.fm);
	sdr_close(G.dev, G.stream);
	return G.failed ? 1 : 0;
}
