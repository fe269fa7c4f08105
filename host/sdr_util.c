#include "sdr_util.h"
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

static double with_suffix(const char *s, const char *units, const double *mult)
{
	size_t n = strlen(s);
	if (n == 0) { return 0.0; }
	const char *u = strchr(units, s[n - 1]);
	if (u && *u) {
		char tmp[64];
		if (n - 1 >= sizeof tmp) { return 0.0; }
		memcpy(tmp, s, n - 1); tmp[n - 1] = 0;
		return atof(tmp) * mult[u - units];
	}
	return atof(s);
}

double parse_scaled(const char *s)
{
	static const double m[] = {1e3, 1e3, 1e6, 1e6, 1e9, 1e9};
	return with_suffix(s, "kKmMgG", m);
}
double parse_seconds(const char *s)
{
	static const double m[] = {1, 1, 60, 60, 3600, 3600};
	return with_suffix(s, "sSmMhH", m);
}
double parse_fraction(const char *s)
{
	static const double m[] = {0.01};
	return with_suffix(s, "%", m);
}

int sdr_open(const char *query, size_t channel, const char *format, SoapySDRDevice **dev, SoapySDRStream **stream)
{
	SoapySDRKwargs none = {0, NULL, NULL};
	*dev = SoapySDRDevice_makeStrArgs(query ? query : "");
	if (!*dev) { fprintf(stderr, "SoapySDRDevice_make failed: %s\n", SoapySDRDevice_lastError()); return -1; }
	char *hw = SoapySDRDevice_getHardwareKey(*dev);
	fprintf(stderr, "Using device %s\n", hw ? hw : "?");
	free(hw);
	if (channel >= SoapySDRDevice_getNumChannels(*dev, SOAPY_SDR_RX)) {
		fprintf(stderr, "Invalid channel %d selected\n", (int)channel);
		return -3;
	}
	*stream = SoapySDRDevice_setupStream(*dev, SOAPY_SDR_RX, format, &channel, 1, &none);
	if (!*stream) { fprintf(stderr, "SoapySDRDevice_setupStream failed: %s\n", SoapySDRDevice_lastError()); return -3; }
	return 0;
}

void sdr_close(SoapySDRDevice *dev, SoapySDRStream *stream)
{
	if (dev && stream) { SoapySDRDevice_deactivateStream(dev, stream, 0, 0); SoapySDRDevice_closeStream(dev, stream); }
	if (dev) { SoapySDRDevice_unmake(dev); }
}

void sdr_set_gain(SoapySDRDevice *dev, size_t channel, const char *gain_str)
{
	if (!gain_str) {
		if (SoapySDRDevice_setGainMode(dev, SOAPY_SDR_RX, channel, true) != 0) { fprintf(stderr, "WARNING: Failed to enable automatic gain.\n"); }
		return;
	}
	if (strchr(gain_str, '=')) {
		SoapySDRKwargs kw = SoapySDRKwargs_fromString(gain_str);
		for (size_t i = 0; i < kw.size; i++) {
			if (SoapySDRDevice_setGainElement(dev, SOAPY_SDR_RX, channel, kw.keys[i], atof(kw.vals[i])) != 0) {
				fprintf(stderr, "WARNING: setGainElement(%s) failed: %s\n", kw.keys[i], SoapySDRDevice_lastError());
			}
		}
		SoapySDRKwargs_clear(&kw);
	} else if (SoapySDRDevice_setGain(dev, SOAPY_SDR_RX, channel, atof(gain_str)) != 0) {
		fprintf(stderr, "WARNING: Failed to set tuner gain: %s\n", SoapySDRDevice_lastError());
	}
}

/* rxb200_ddc_lowpass(M, T) as a filter at shift S, its taps on the heap */
static rxb200_ddc lowpass(int M, int T, int S)
{
	int32_t *taps = (int32_t *)malloc(sizeof(int32_t) * (size_t)T);
	rxb200_ddc_lowpass(M, T, 15, taps);
	return (rxb200_ddc){M, T, taps, S};
}

int capture_plan(enum capture_kind kind, const int64_t *tuned, int n, int chain_rate, const char *cap_env, int nco,
                 long long device_rate, struct capture_plan *p, int *chans)
{
	const long long cap = atoll(cap_env), R_dev = device_rate;
	int rc;
	memset(p, 0, sizeof *p);
	if (kind == CAPTURE_TWO_STAGE) {
		rxb200_fm_two_stage_plan t;
		rc = R_dev ? rxb200_fm_plan_capture_two_stage_at(tuned, n, chain_rate, cap, R_dev, &t, chans)
		           : rxb200_fm_plan_capture_two_stage(tuned, n, chain_rate, cap, &t, chans);
		if (rc == RXB200_OK) {
			p->centre_hz = t.centre_hz; p->capture_rate = t.capture_rate; p->decim = t.coarse_decim * t.fine_decim;
			p->n_bins = t.n_bins;
			p->ddc = lowpass(t.coarse_decim, t.coarse_taps, t.coarse_shift);
			p->fine = lowpass(t.fine_decim, t.fine_taps, t.fine_shift);
			snprintf(p->banner, sizeof p->banner, "Capture mode: %d Hz centred at %lld Hz in two stages: %d bins, coarse "
			         "decimation %d with %d taps, fine decimation %d with %d taps, %d channels\n", t.capture_rate,
			         (long long)t.centre_hz, t.n_bins, t.coarse_decim, t.coarse_taps, t.fine_decim, t.fine_taps, n);
		}
	} else if (kind == CAPTURE_RASTER) {
		rxb200_fm_raster_plan r;
		rc = R_dev ? rxb200_fm_plan_capture_raster_at(tuned, n, chain_rate, cap, R_dev, &r, chans)
		           : rxb200_fm_plan_capture_raster(tuned, n, chain_rate, cap, &r, chans);
		if (rc == RXB200_OK) {
			p->centre_hz = r.centre_hz; p->capture_rate = r.capture_rate; p->decim = r.decim; p->n_bins = r.n_bins;
			p->ddc = lowpass(r.decim, r.n_taps, r.shift);
			snprintf(p->banner, sizeof p->banner, "Capture mode: %d Hz centred at %lld Hz as a raster: %d bins, decimation "
			         "%d, %d taps, %d channels\n", r.capture_rate, (long long)r.centre_hz, r.n_bins, r.decim, r.n_taps, n);
		}
	} else {
		rxb200_fm_capture_plan s;
		rc = nco ? (R_dev ? rxb200_sdr_plan_capture_at(tuned, n, chain_rate, cap, R_dev, &s, chans)
		                  : rxb200_sdr_plan_capture(tuned, n, chain_rate, cap, &s, chans))
		         : (R_dev ? rxb200_fm_plan_capture_at(tuned, n, chain_rate, cap, R_dev, &s, chans)
		                  : rxb200_fm_plan_capture(tuned, n, chain_rate, cap, &s, chans));
		if (rc == RXB200_OK) {
			p->centre_hz = s.centre_hz; p->capture_rate = s.capture_rate; p->decim = s.decim;
			p->ddc = lowpass(s.decim, s.n_taps, 15);
			snprintf(p->banner, sizeof p->banner, "Capture mode: %d Hz centred at %lld Hz, decimation %d, %d taps, %d "
			         "channels\n", s.capture_rate, (long long)s.centre_hz, s.decim, s.n_taps, n);
		}
	}
	if (rc != RXB200_OK) {
		fprintf(stderr, "Capture mode: %s (RXB200_CAPTURE_RATE=%s).\n", rxb200_last_error(), cap_env);
		return 1;
	}
	long long A = 0;
	for (int k = 0; k < n; k++) {
		const long long o = (long long)(tuned[k] - p->centre_hz);
		if ((o < 0 ? -o : o) > A) { A = o < 0 ? -o : o; }
	}
	p->span = 2 * A + chain_rate;
	return 0;
}

void capture_plan_release(struct capture_plan *p)
{
	free((void *)p->ddc.taps);
	free((void *)p->fine.taps);
}

long long device_rate_env(int allowed, const char *needs)
{
	const char *v = getenv("RXB200_DEVICE_RATE");
	if (!v) { return 0; }
	if (!allowed) { fprintf(stderr, "RXB200_DEVICE_RATE needs %s.\n", needs); return -1; }
	char *e = NULL;
	const long long r = strtoll(v, &e, 10);
	if (e == v || *e || r < 1 || r > 2147483647LL) {
		fprintf(stderr, "RXB200_DEVICE_RATE=%s is not a rate in [1, 2^31 - 1] Hz.\n", v);
		return -1;
	}
	return r;
}

long long sdr_device_rate(SoapySDRDevice *dev, size_t channel, long long rate)
{
	SoapySDRDevice_setSampleRate(dev, SOAPY_SDR_RX, channel, (double)rate);
	const double got = SoapySDRDevice_getSampleRate(dev, SOAPY_SDR_RX, channel);
	if (!(got >= 0.5 && got < 2147483647.5)) {
		fprintf(stderr, "The device reports a sample rate of %.0f Hz after RXB200_DEVICE_RATE=%lld asked for it: not a "
		        "rate in [1, 2^31 - 1] Hz, so its samples cannot be resampled.\n", got, rate);
		return -1;
	}
	return llround(got);
}

int device_resampler(long long device_rate, long long rate, long long span, rxb200_resampler *rs)
{
	if (rxb200_plan_resample(device_rate, rate, span, rs) != RXB200_OK) {
		fprintf(stderr, "Device rate: %s (RXB200_DEVICE_RATE=%lld).\n", rxb200_last_error(), device_rate);
		return 1;
	}
	if (rs->up == 1 && rs->down == 1) {
		fprintf(stderr, "Device rate: %lld Hz, the capture rate: no resampling needed\n", device_rate);
		return 0;
	}
	int32_t *taps = (int32_t *)malloc(sizeof(int32_t) * (size_t)rs->up * (size_t)rs->taps_per_phase);
	rxb200_resample_lowpass(rs->up, rs->down, rs->taps_per_phase, taps);
	rs->taps = taps;
	fprintf(stderr, "Device rate: %lld Hz, resampled by %d/%d with %d taps per phase to %lld Hz\n", device_rate, rs->up,
	        rs->down, rs->taps_per_phase, rate);
	return 0;
}

size_t resample_out_count(int up, int down, unsigned long long n0, size_t c)
{
	typedef unsigned __int128 u128;
	const u128 L = (u128)up, N = (u128)down;
	return (size_t)((((u128)n0 + c) * L + N - 1) / N - ((u128)n0 * L + N - 1) / N);
}

int device_format_env(int allowed, const char *needs, const char **name)
{
	static const char *names[] = {SOAPY_SDR_CS16, SOAPY_SDR_CS8, SOAPY_SDR_CU8, SOAPY_SDR_CS12};   /* RXB200_IN_* order */
	const char *v = getenv("RXB200_DEVICE_FORMAT");
	*name = SOAPY_SDR_CS16;
	if (!v) { return RXB200_IN_CS16; }
	if (!allowed) { fprintf(stderr, "RXB200_DEVICE_FORMAT needs %s.\n", needs); return -1; }
	for (int f = RXB200_IN_CS16; f <= RXB200_IN_CS12; f++) {
		if (!strcmp(v, names[f])) { *name = names[f]; return f; }
	}
	fprintf(stderr, "RXB200_DEVICE_FORMAT=%s is not one of CS16, CS8, CU8, CS12.\n", v);
	return -1;
}

size_t device_format_bytes(int in_fmt) { return in_fmt == RXB200_IN_CS16 ? 4 : in_fmt == RXB200_IN_CS12 ? 3 : 2; }
