/* soapy_fake.c — a replay-only fake of the 32 SoapySDR C entry points rx_tools calls.
 *
 * A REPLAY DEVICE, no DSP: it only hands stored samples to readStream.  SoapySDR is not installed in this image and the
 * reference (rxseger/rx_tools) has no fake device of its own (SURVEY.md §4, §8c), so this
 * file supplies one.  Two uses:
 *   1. oracle/_ref/libref_fm.so / libref_power.so: the unmodified reference sources are
 *      compiled against host/soapy_replay and linked with this file so every symbol
 *      resolves; the harness feeds samples from memory (soapy_fake_set_memory).
 *   2. the drop-in host shells (host/rx_fm_b200, host/rx_power_b200) run hardware-free
 *      with `-d driver=file,path=capture.cs16[,loop=1][,reads=a:b:c][,rate=Hz]`; reads= caps successive reads at a, b, c, a, ...
 *      complex elements, the way a device that reads in packets returns them; rate=<Hz> models a device that runs only
 *      at that rate: setSampleRate records the request, getSampleRate returns rate and listSampleRates {rate}.  Without
 *      it getSampleRate returns the last request (a device that honours any rate).
 *
 * Behaviour that matters: readStream (copies the next numElems complex elements of the stream's format,
 * returns the count, SOAPY_SDR_TIMEOUT... never; returns -2 STREAM_ERROR at end of data so
 * the reference's dongle thread terminates), set/getFrequency (remembers the last value so
 * rx_power's retune() logic runs as on hardware), set/getSampleRate, formatToSize, getNumChannels.
 * Everything else is a successful no-op.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>
#include <SoapySDR/Device.h>
#include <SoapySDR/Formats.h>

struct SoapySDRDevice {
	const int16_t *mem;     /* the capture: interleaved CS16 (or raw bytes of another element format, see elem_size) */
	size_t n_complex;       /* total complex elements available */
	size_t n_bytes;         /* the same capture in bytes (file replay) */
	size_t elem_size;       /* bytes per complex element of the stream format: 4 (CS16), 3 (CS12), 2 (CS8, CU8) */
	size_t pos;             /* next complex element */
	int loop;
	int owns_mem;
	double freq;
	double rate;            /* the last setSampleRate request */
	double fixed_rate;      /* rate=: the only rate the device runs at; 0: any rate it is asked for */
	double bw;
	long long reads;        /* number of readStream calls served */
	size_t read_len[64];    /* reads=a:b:c: a read returns at most these many complex elements, in turn (a device reading in packets) */
	int n_read_len;         /* 0: a read returns whatever was asked for, as far as the capture goes */
	int read_idx;
};
struct SoapySDRStream { int active; };

static struct SoapySDRDevice g_dev;
static struct SoapySDRStream g_stream;
static const char *g_err = "";
static int (*g_read_hook)(void * const *buffs, size_t numElems) = NULL;

/* ---- harness-side controls (not part of SoapySDR) ---- */
void soapy_fake_set_memory(const int16_t *cs16, size_t n_complex, int loop)
{
	if (g_dev.owns_mem) { free((void *)g_dev.mem); }
	g_dev.mem = cs16; g_dev.n_complex = n_complex; g_dev.n_bytes = n_complex * 4; g_dev.elem_size = 4; g_dev.pos = 0;
	g_dev.loop = loop; g_dev.owns_mem = 0; g_dev.reads = 0;
}
void soapy_fake_set_read_hook(int (*hook)(void * const *buffs, size_t numElems)) { g_read_hook = hook; }
size_t soapy_fake_position(void) { return g_dev.pos; }
long long soapy_fake_reads(void) { return g_dev.reads; }

static const char *kw_find(const char *args, const char *key, char *out, size_t outsz)
{
	/* args is "k=v,k=v"; returns out or NULL */
	size_t klen = strlen(key);
	const char *p = args;
	while (p && *p) {
		while (*p == ' ' || *p == ',') { p++; }
		if (strncmp(p, key, klen) == 0 && p[klen] == '=') {
			const char *v = p + klen + 1;
			const char *e = strchr(v, ',');
			size_t n = e ? (size_t)(e - v) : strlen(v);
			if (n >= outsz) { n = outsz - 1; }
			memcpy(out, v, n); out[n] = 0;
			return out;
		}
		p = strchr(p, ',');
	}
	return NULL;
}

static int load_file(const char *path)
{
	FILE *f = fopen(path, "rb");
	long sz;
	int16_t *buf;
	if (!f) { g_err = "fake: cannot open path"; return -1; }
	fseek(f, 0, SEEK_END); sz = ftell(f); fseek(f, 0, SEEK_SET);
	buf = (int16_t *)malloc(sz > 0 ? (size_t)sz : 4);
	if (!buf) { fclose(f); g_err = "fake: malloc"; return -1; }
	if (sz > 0 && fread(buf, 1, (size_t)sz, f) != (size_t)sz) { fclose(f); free(buf); g_err = "fake: short read"; return -1; }
	fclose(f);
	if (g_dev.owns_mem) { free((void *)g_dev.mem); }
	g_dev.mem = buf; g_dev.n_bytes = (size_t)sz; g_dev.elem_size = 4; g_dev.n_complex = (size_t)sz / 4; g_dev.pos = 0; g_dev.owns_mem = 1; g_dev.reads = 0;
	return 0;
}

/* ---- SoapySDR C API subset ---- */
size_t SoapySDR_formatToSize(const char *format)
{
	if (!format) { return 0; }
	if (!strcmp(format, SOAPY_SDR_CS16) || !strcmp(format, SOAPY_SDR_CU16)) { return 4; }
	if (!strcmp(format, SOAPY_SDR_CS8) || !strcmp(format, SOAPY_SDR_CU8)) { return 2; }
	if (!strcmp(format, SOAPY_SDR_CF32) || !strcmp(format, SOAPY_SDR_CS32)) { return 8; }
	if (!strcmp(format, SOAPY_SDR_CF64)) { return 16; }
	if (!strcmp(format, SOAPY_SDR_CS12)) { return 3; }
	return 0;
}

SoapySDRKwargs SoapySDRKwargs_fromString(const char *markup)
{
	SoapySDRKwargs k = {0, NULL, NULL};
	const char *p = markup;
	while (p && *p) {
		const char *e = strchr(p, ',');
		size_t n = e ? (size_t)(e - p) : strlen(p);
		const char *eq = memchr(p, '=', n);
		if (eq) {
			size_t kl = (size_t)(eq - p), vl = n - kl - 1;
			k.keys = (char **)realloc(k.keys, (k.size + 1) * sizeof(char *));
			k.vals = (char **)realloc(k.vals, (k.size + 1) * sizeof(char *));
			k.keys[k.size] = (char *)calloc(kl + 1, 1); memcpy(k.keys[k.size], p, kl);
			k.vals[k.size] = (char *)calloc(vl + 1, 1); memcpy(k.vals[k.size], eq + 1, vl);
			k.size++;
		}
		p = e ? e + 1 : NULL;
	}
	return k;
}

void SoapySDRKwargs_clear(SoapySDRKwargs *args)
{
	size_t i;
	if (!args) { return; }
	for (i = 0; i < args->size; i++) { free(args->keys[i]); free(args->vals[i]); }
	free(args->keys); free(args->vals);
	args->keys = args->vals = NULL; args->size = 0;
}

const char *SoapySDRDevice_lastError(void) { return g_err; }

SoapySDRDevice *SoapySDRDevice_makeStrArgs(const char *args)
{
	char v[1024];
	g_dev.freq = 0; g_dev.rate = 0; g_dev.bw = 0;
	g_dev.fixed_rate = 0.0;
	if (args && kw_find(args, "rate", v, sizeof v)) {
		char *e = NULL;
		g_dev.fixed_rate = strtod(v, &e);
		if (e == v || *e || !(g_dev.fixed_rate > 0)) { g_err = "fake: rate= takes a positive rate in Hz"; return NULL; }
	}
	if (args && kw_find(args, "path", v, sizeof v)) {
		if (load_file(v) != 0) { return NULL; }
	}
	g_dev.loop = (args && kw_find(args, "loop", v, sizeof v)) ? atoi(v) : g_dev.loop;
	g_dev.n_read_len = 0; g_dev.read_idx = 0;
	if (args && kw_find(args, "reads", v, sizeof v)) {
		char *p = v;
		while (*p && g_dev.n_read_len < 64) {
			char *e;
			long n = strtol(p, &e, 10);
			if (e == p || n < 1) { g_err = "fake: reads=a:b:c takes positive element counts"; return NULL; }
			g_dev.read_len[g_dev.n_read_len++] = (size_t)n;
			p = (*e == ':') ? e + 1 : e;
			if (*e != ':' && *e) { g_err = "fake: reads=a:b:c takes positive element counts"; return NULL; }
		}
	}
	return &g_dev;
}
int SoapySDRDevice_unmake(SoapySDRDevice *d) { (void)d; return 0; }

static char *dupstr(const char *s) { char *r = (char *)malloc(strlen(s) + 1); strcpy(r, s); return r; }
char *SoapySDRDevice_getDriverKey(const SoapySDRDevice *d) { (void)d; return dupstr("file"); }
char *SoapySDRDevice_getHardwareKey(const SoapySDRDevice *d) { (void)d; return dupstr("replay"); }
SoapySDRKwargs SoapySDRDevice_getHardwareInfo(const SoapySDRDevice *d) { SoapySDRKwargs k = {0, NULL, NULL}; (void)d; return k; }
size_t SoapySDRDevice_getNumChannels(const SoapySDRDevice *d, const int dir) { (void)d; (void)dir; return 1; }

SoapySDRStream *SoapySDRDevice_setupStream(SoapySDRDevice *d, const int dir, const char *format,
	const size_t *channels, const size_t numChans, const SoapySDRKwargs *args)
{
	(void)d; (void)dir; (void)channels; (void)numChans; (void)args;
	/* CS16 is what rx_fm / rx_power ask for; rx_sdr may also ask for the packed 12-bit format (-I CS12,
	 * src/rtl_sdr.c:352-362), and any shell for a device's own CS8, CU8 or CS12 (RXB200_DEVICE_FORMAT): the capture
	 * file is then taken as raw 3-byte (CS12) or 2-byte (CS8, CU8) elements */
	if (format && strcmp(format, SOAPY_SDR_CS12) == 0) { g_dev.elem_size = 3; }
	else if (format && strcmp(format, SOAPY_SDR_CS16) == 0) { g_dev.elem_size = 4; }
	else if (format && (strcmp(format, SOAPY_SDR_CS8) == 0 || strcmp(format, SOAPY_SDR_CU8) == 0)) { g_dev.elem_size = 2; }
	else { g_err = "fake: only CS16, CS12, CS8 and CU8"; return NULL; }
	if (g_dev.n_bytes) { g_dev.n_complex = g_dev.n_bytes / g_dev.elem_size; }
	return &g_stream;
}
int SoapySDRDevice_closeStream(SoapySDRDevice *d, SoapySDRStream *s) { (void)d; (void)s; return 0; }
int SoapySDRDevice_activateStream(SoapySDRDevice *d, SoapySDRStream *s, const int flags, const long long t, const size_t n)
{ (void)d; (void)flags; (void)t; (void)n; if (s) { s->active = 1; } return 0; }
int SoapySDRDevice_deactivateStream(SoapySDRDevice *d, SoapySDRStream *s, const int flags, const long long t)
{ (void)d; (void)flags; (void)t; if (s) { s->active = 0; } return 0; }

int SoapySDRDevice_readStream(SoapySDRDevice *d, SoapySDRStream *s, void * const *buffs, const size_t numElems,
	int *flags, long long *timeNs, const long timeoutUs)
{
	size_t avail, n;
	(void)s; (void)timeNs; (void)timeoutUs;
	if (flags) { *flags = 0; }
	if (g_read_hook) { if (d) { d->reads++; } return g_read_hook(buffs, numElems); }
	if (!d || !d->mem || d->n_complex == 0) { return SOAPY_SDR_STREAM_ERROR; }
	d->reads++;
	if (d->pos >= d->n_complex) {
		if (!d->loop) { return SOAPY_SDR_STREAM_ERROR; }
		d->pos = 0;
	}
	avail = d->n_complex - d->pos;
	n = numElems < avail ? numElems : avail;
	if (d->n_read_len) {
		const size_t cap = d->read_len[d->read_idx];
		d->read_idx = (d->read_idx + 1) % d->n_read_len;
		if (n > cap) { n = cap; }
	}
	memcpy(buffs[0], (const unsigned char *)d->mem + d->elem_size * d->pos, n * d->elem_size);
	d->pos += n;
	return (int)n;
}

int SoapySDRDevice_setAntenna(SoapySDRDevice *d, const int dir, const size_t ch, const char *name) { (void)d; (void)dir; (void)ch; (void)name; return 0; }
static char **empty_list(size_t *length) { if (length) { *length = 0; } return NULL; }
char **SoapySDRDevice_listAntennas(const SoapySDRDevice *d, const int dir, const size_t ch, size_t *length) { (void)d; (void)dir; (void)ch; return empty_list(length); }
char **SoapySDRDevice_listGains(const SoapySDRDevice *d, const int dir, const size_t ch, size_t *length) { (void)d; (void)dir; (void)ch; return empty_list(length); }
char **SoapySDRDevice_listFrequencies(const SoapySDRDevice *d, const int dir, const size_t ch, size_t *length) { (void)d; (void)dir; (void)ch; return empty_list(length); }
double *SoapySDRDevice_listSampleRates(const SoapySDRDevice *d, const int dir, const size_t ch, size_t *length)
{
	(void)dir; (void)ch;
	if (!d || d->fixed_rate <= 0) { if (length) { *length = 0; } return NULL; }
	double *r = (double *)malloc(sizeof(double));
	r[0] = d->fixed_rate;
	if (length) { *length = 1; }
	return r;
}
double *SoapySDRDevice_listBandwidths(const SoapySDRDevice *d, const int dir, const size_t ch, size_t *length) { (void)d; (void)dir; (void)ch; if (length) { *length = 0; } return NULL; }

int SoapySDRDevice_setGainMode(SoapySDRDevice *d, const int dir, const size_t ch, const bool a) { (void)d; (void)dir; (void)ch; (void)a; return 0; }
int SoapySDRDevice_setGain(SoapySDRDevice *d, const int dir, const size_t ch, const double v) { (void)d; (void)dir; (void)ch; (void)v; return 0; }
int SoapySDRDevice_setGainElement(SoapySDRDevice *d, const int dir, const size_t ch, const char *n, const double v) { (void)d; (void)dir; (void)ch; (void)n; (void)v; return 0; }

int SoapySDRDevice_setFrequency(SoapySDRDevice *d, const int dir, const size_t ch, const double f, const SoapySDRKwargs *a)
{ (void)dir; (void)ch; (void)a; if (d) { d->freq = f; } return 0; }
double SoapySDRDevice_getFrequency(const SoapySDRDevice *d, const int dir, const size_t ch) { (void)dir; (void)ch; return d ? d->freq : 0.0; }
int SoapySDRDevice_setFrequencyCorrection(SoapySDRDevice *d, const int dir, const size_t ch, const double v) { (void)d; (void)dir; (void)ch; (void)v; return 0; }
int SoapySDRDevice_setSampleRate(SoapySDRDevice *d, const int dir, const size_t ch, const double r) { (void)dir; (void)ch; if (d) { d->rate = r; } return 0; }
double SoapySDRDevice_getSampleRate(const SoapySDRDevice *d, const int dir, const size_t ch)
{ (void)dir; (void)ch; return !d ? 0.0 : d->fixed_rate > 0 ? d->fixed_rate : d->rate; }
int SoapySDRDevice_setBandwidth(SoapySDRDevice *d, const int dir, const size_t ch, const double bw) { (void)dir; (void)ch; if (d) { d->bw = bw; } return 0; }
double SoapySDRDevice_getBandwidth(const SoapySDRDevice *d, const int dir, const size_t ch) { (void)dir; (void)ch; return d ? d->bw : 0.0; }

int SoapySDRDevice_writeSetting(SoapySDRDevice *d, const char *k, const char *v) { (void)d; (void)k; (void)v; return 0; }
char *SoapySDRDevice_readSetting(const SoapySDRDevice *d, const char *k) { (void)d; (void)k; return dupstr("true"); }
