// host_plan.cpp — the host-side arithmetic that surrounds the kernels: parameter derivation
// (rx_fm main() + optimal_settings()), the rx_power hop planner (frequency_range()), the window /
// sine tables and the CSV row formatter (csv_dbm()).  Pure C++, no CUDA, no reference code: each
// function restates what the cited reference lines compute so the drop-in host shells and the
// Python mirror get identical numbers (checked against the reference in tests/test_oracle_pin.py
// and tests/test_host_logic.py).
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include <cuda_runtime.h>
#include "../../include/rxb200.h"

namespace rxb {
static thread_local char g_err[512] = "";
void set_error(const char *fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof g_err, fmt, ap);
	va_end(ap);
}
}  // namespace rxb
using rxb::set_error;

extern "C" const char *rxb200_last_error(void) { return rxb::g_err; }
extern "C" int rxb200_abi_version(void) { return RXB200_ABI_VERSION; }
extern "C" int rxb200_device_count(void)
{
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
	return n;
}

// ---------------------------------------------------------------------------------- rx_fm
// main(): defaults (demod_init, src/rtl_fm.c:1084-1115), the -M wbfm preset (:1331-1341), -s/-r/-F/-A
// (:1255-1262, :1305-1319), rate_in *= post_downsample (:1371), output.rate default (:1373),
// optimal_settings() (:960-997) and deemph_a (:1410-1412).
extern "C" int rxb200_fm_derive(const rxb200_fm_cli *cli, rxb200_fm_derived *out)
{
	if (!cli || !out) { set_error("null argument"); return RXB200_EINVAL; }
	memset(out, 0, sizeof *out);
	rxb200_fm_params &p = out->params;
	int rate_in = 24000, rate_out = 24000, rate_out2 = -1, output_rate = 0;
	int custom_atan = RXB200_ATAN_STD, deemph = 0, squelch = cli->squelch_level;
	int mode = cli->mode;
	if (cli->wbfm) {
		mode = RXB200_MODE_FM;
		rate_in = 170000; rate_out = 170000; rate_out2 = 32000; output_rate = 32000;
		// the preset zeroes squelch_level WHEN -M is parsed (:1339), so a later -l survives: the caller applies that
		// parse-order rule to cli->squelch_level (host/rx_fm_b200.c does), derive keeps what it is given
		custom_atan = RXB200_ATAN_FAST; deemph = 1;
	}
	if (cli->rate_s > 0) { rate_in = cli->rate_s; rate_out = cli->rate_s; }
	if (cli->rate_r > 0) { output_rate = cli->rate_r; rate_out2 = cli->rate_r; }
	if (cli->custom_atan >= 0) { custom_atan = cli->custom_atan; }
	if (cli->deemph >= 0) { deemph = cli->deemph; }
	int post = cli->post_downsample > 0 ? cli->post_downsample : 1;
	int passes = cli->use_F ? 1 : 0;
	rate_in *= post;
	if (!output_rate) { output_rate = rate_out; }
	if (rate_in <= 0) { set_error("rate_in %d", rate_in); return RXB200_EINVAL; }
	int downsample = (1000000 / rate_in) + 1;
	if (passes) {
		passes = (int)log2((double)downsample) + 1;
		downsample = 1 << passes;
	}
	int capture_rate = downsample * rate_in;
	int capture_off = cli->offset_tuning ? 0 : capture_rate / 4;
	int output_scale = (1 << 15) / (128 * downsample);
	if (output_scale < 1) { output_scale = 1; }
	if (mode == RXB200_MODE_FM) { output_scale = 1; }
	int deemph_a = 0;
	if (deemph) {
		double tc = (double)(cli->time_constant_us > 0 ? cli->time_constant_us : 75) * 1e-6;
		deemph_a = (int)round(1.0 / ((1.0 - exp(-1.0 / (rate_out * tc)))));
	}
	p.mode = mode; p.downsample = downsample; p.downsample_passes = passes;
	p.comp_fir_size = cli->use_F ? cli->comp_fir_size : 0;
	p.custom_atan = custom_atan; p.output_scale = output_scale; p.post_downsample = post;
	p.deemph = deemph; p.deemph_a = deemph_a; p.rate_out = rate_out; p.rate_out2 = rate_out2;
	p.squelch_level = squelch; p.dc_block_audio = cli->dc_block_audio; p.adc_block_const = 9;
	p.dc_block_raw = cli->dc_block_raw; p.rdc_block_const = cli->rdc_block_const > 0 ? cli->rdc_block_const : 9;
	p.offset_tuning = cli->offset_tuning;
	out->capture_rate = capture_rate;
	out->capture_freq_offset = capture_off;
	out->output_rate = output_rate;
	return RXB200_OK;
}

// The mixer table of a channel f Hz away from the centre of a capture at R Hz (include/rxb200.h, "rx_fm channels of one
// capture"): Q15 with unity 2^15, one entry per complex sample of the period R / gcd(R, |f|).  The angle's residue is
// exact (64-bit integers); only cos / sin of it are fp64, and its symmetric representative makes f and -f conjugates.
#define RXB_MIX_MAX_PERIOD (1 << 20)
extern "C" int rxb200_fm_mix_table(int capture_rate, int offset_hz, int32_t *table, size_t cap, size_t *period)
{
	if (!period) { set_error("null argument"); return RXB200_EINVAL; }
	const long long R = capture_rate, f = offset_hz;
	if (R <= 0 || 2 * (f < 0 ? -f : f) >= R) { set_error("mixer needs capture_rate > 0 and |offset| < capture_rate/2 (%d, %d)", capture_rate, offset_hz); return RXB200_EINVAL; }
	long long a = R, b = f < 0 ? -f : f;
	while (b) { const long long t = a % b; a = b; b = t; }
	const long long L = R / a;
	if (L > RXB_MIX_MAX_PERIOD) { set_error("mixer period %lld > 2^20 samples (capture_rate %d, offset %d)", L, capture_rate, offset_hz); return RXB200_EUNSUPPORTED; }
	*period = (size_t)L;
	if (!table || cap < 2 * (size_t)L) { set_error("mixer table capacity %zu < %lld", cap, 2 * L); return RXB200_ECAPACITY; }
	for (long long m = 0; m < L; m++) {
		long long r = ((m * f) % R + R) % R;          // |m f| < 2^20 * 2^31: no overflow
		if (2 * r > R) { r -= R; }                      // (-R/2, R/2]
		const double t = -2.0 * M_PI * (double)r / (double)R;
		table[2 * m] = (int32_t)round(32768.0 * cos(t));
		table[2 * m + 1] = (int32_t)round(32768.0 * sin(t));
	}
	return RXB200_OK;
}

// The capture plan of the rx_fm shell's capture mode (include/rxb200.h, "rx_fm channels of one capture in the shell").
// The centre fc, the decimation M and the channel grid g of rxb200_fm_plan_capture's rule, with its refusals of the
// arguments (g_out may be NULL).  G: the guard band a resampler from a device rate needs (rxb200_plan_resample), which
// the decimation floor leaves, M = ceil((2 A + c + G) / c); 0 without a device rate, today's rule.
static int capture_centre(const int64_t *tuned_hz, int n_channels, int chain_rate, long long G, long long *fc_out,
                          long long *M_out, long long *g_out = NULL)
{
	if (n_channels < 1 || chain_rate < 1) {
		set_error("capture plan of %d channels at a chain capture rate of %d Hz (need >= 1 of each)", n_channels, chain_rate);
		return RXB200_EINVAL;
	}
	const long long fmax = 1ll << 61;                   // keeps 2 A + 2 c below 2^63
	long long tmin = tuned_hz[0], tmax = tuned_hz[0];
	for (int k = 0; k < n_channels; k++) {
		if (tuned_hz[k] < 0 || tuned_hz[k] >= fmax) { set_error("tuned frequency %lld Hz outside [0, 2^61)", (long long)tuned_hz[k]); return RXB200_EINVAL; }
		tmin = std::min(tmin, (long long)tuned_hz[k]);
		tmax = std::max(tmax, (long long)tuned_hz[k]);
	}
	long long g = 0;                                      // gcd of every t_k - tmin; 0 when all are equal
	for (int k = 0; k < n_channels; k++) {
		long long a = tuned_hz[k] - tmin, b = g;
		while (b) { const long long t = a % b; a = b; b = t; }
		g = a;
	}
	const long long fc = g ? tmin + g * ((tmax - tmin) / (2 * g)) : tmin;
	const long long A = std::max(fc - tmin, tmax - fc), c = chain_rate;
	*fc_out = fc;
	*M_out = (2 * A + c + G + c - 1) / c;
	if (g_out) { *g_out = g; }
	return RXB200_OK;
}

// the single-stage plan's refusal of its capture rate R = M c
static int rate_check(long long R, long long M, long long max_capture_rate)
{
	if (R > max_capture_rate || R > 2147483647ll || M > 256) {
		set_error("the channels need a capture rate of %lld Hz (decimation %lld), above the cap of %lld Hz, 2^31 - 1 or "
		          "decimation 256", R, M, max_capture_rate);
		return RXB200_EINVAL;
	}
	return RXB200_OK;
}

// The guard band G = ceil(R_dev / 32) of the _at planners' device rate (rxb200_plan_resample's), with its refusal
static int device_guard(long long device_rate, long long *G)
{
	if (device_rate < 1 || device_rate > 2147483647ll) {
		set_error("device rate %lld Hz outside [1, 2^31 - 1]", device_rate);
		return RXB200_EINVAL;
	}
	*G = (device_rate + 31) / 32;
	return RXB200_OK;
}

// the _at planners' refusal of a capture rate R above the device rate (device_rate 0: no device rate): the shells only
// resample down
static int device_check(long long R, long long device_rate)
{
	if (device_rate && R > device_rate) {
		set_error("the channels need a capture rate of %lld Hz, above the device rate of %lld Hz", R, device_rate);
		return RXB200_EUNSUPPORTED;
	}
	return RXB200_OK;
}

// rxb200_fm_plan_capture's rule; table: refuse offsets whose mixer table rxb200_fm_mix_table refuses (the rx_fm shell's
// table mixer), else take any offset (the rx_sdr shell's NCO, rxb200_sdr_plan_capture).  device_rate: 0, or the _at
// planners' checked device rate, whose guard band G the decimation floor leaves
static int capture_plan(const int64_t *tuned_hz, int n_channels, int chain_rate, long long max_capture_rate,
                        long long device_rate, long long G, rxb200_fm_capture_plan *out, int *offsets_hz, bool table)
{
	if (!tuned_hz || !out || !offsets_hz) { set_error("null argument"); return RXB200_EINVAL; }
	long long fc = 0, M = 0;
	int rc = capture_centre(tuned_hz, n_channels, chain_rate, G, &fc, &M);
	if (rc != RXB200_OK) { return rc; }
	const long long R = M * chain_rate;
	rc = rate_check(R, M, max_capture_rate);
	if (rc == RXB200_OK) { rc = device_check(R, device_rate); }
	if (rc != RXB200_OK) { return rc; }
	for (int k = 0; k < n_channels; k++) {
		size_t L = 0;
		rc = table ? rxb200_fm_mix_table((int)R, (int)(tuned_hz[k] - fc), NULL, 0, &L) : RXB200_ECAPACITY;
		if (rc != RXB200_ECAPACITY) { return rc; }        // the table's own refusal and message
		offsets_hz[k] = (int)(tuned_hz[k] - fc);
	}
	out->centre_hz = fc;
	out->decim = (int)M;
	out->capture_rate = (int)R;
	out->n_taps = (int)std::min(8191ll, 32 * M + 1);
	return RXB200_OK;
}

extern "C" int rxb200_fm_plan_capture(const int64_t *tuned_hz, int n_channels, int chain_rate, long long max_capture_rate,
                                      rxb200_fm_capture_plan *out, int *offsets_hz)
{
	return capture_plan(tuned_hz, n_channels, chain_rate, max_capture_rate, 0, 0, out, offsets_hz, true);
}

extern "C" int rxb200_fm_plan_capture_at(const int64_t *tuned_hz, int n_channels, int chain_rate,
                                         long long max_capture_rate, long long device_rate, rxb200_fm_capture_plan *out,
                                         int *offsets_hz)
{
	long long G = 0;
	const int rc = device_guard(device_rate, &G);
	if (rc != RXB200_OK) { return rc; }
	return capture_plan(tuned_hz, n_channels, chain_rate, max_capture_rate, device_rate, G, out, offsets_hz, true);
}

extern "C" int rxb200_sdr_plan_capture(const int64_t *tuned_hz, int n_channels, int sample_rate,
                                       long long max_capture_rate, rxb200_fm_capture_plan *out, int *offsets_hz)
{
	return capture_plan(tuned_hz, n_channels, sample_rate, max_capture_rate, 0, 0, out, offsets_hz, false);
}

extern "C" int rxb200_sdr_plan_capture_at(const int64_t *tuned_hz, int n_channels, int sample_rate,
                                          long long max_capture_rate, long long device_rate, rxb200_fm_capture_plan *out,
                                          int *offsets_hz)
{
	long long G = 0;
	const int rc = device_guard(device_rate, &G);
	if (rc != RXB200_OK) { return rc; }
	return capture_plan(tuned_hz, n_channels, sample_rate, max_capture_rate, device_rate, G, out, offsets_hz, false);
}

// rxb200_fm_plan_capture_two_stage's rule; device_rate and G as for capture_plan
static int two_stage_plan(const int64_t *tuned_hz, int n_channels, int chain_rate, long long max_capture_rate,
                          long long device_rate, long long G, rxb200_fm_two_stage_plan *out, int *offsets_hz)
{
	if (!tuned_hz || !out || !offsets_hz) { set_error("null argument"); return RXB200_EINVAL; }
	long long fc = 0, M = 0;
	int rc = capture_centre(tuned_hz, n_channels, chain_rate, G, &fc, &M);
	if (rc != RXB200_OK) { return rc; }
	const long long Mp = 4 * ((M + 3) / 4), R = Mp * chain_rate;
	if (Mp < 8) {
		set_error("two-stage capture plan: decimation %lld (from %lld) is below 8; the single-stage plan fits", Mp, M);
		return RXB200_EINVAL;
	}
	if (R > max_capture_rate || R > 2147483647ll || Mp > 256) {
		set_error("the channels need a capture rate of %lld Hz (two-stage decimation %lld), above the cap of %lld Hz, "
		          "2^31 - 1 or decimation 256", R, Mp, max_capture_rate);
		return RXB200_EINVAL;
	}
	rc = device_check(R, device_rate);
	if (rc != RXB200_OK) { return rc; }
	for (int k = 0; k < n_channels; k++) { offsets_hz[k] = (int)(tuned_hz[k] - fc); }
	const int M1 = (int)(Mp / 4);
	out->centre_hz = fc;
	out->capture_rate = (int)R;
	out->n_bins = 2 * M1;
	out->coarse_decim = M1;
	out->coarse_taps = std::min(8191, 24 * M1 + 1);
	out->coarse_shift = 30;
	out->fine_decim = 4;
	out->fine_taps = 129;
	out->fine_shift = 15;
	return RXB200_OK;
}

extern "C" int rxb200_fm_plan_capture_two_stage(const int64_t *tuned_hz, int n_channels, int chain_rate,
                                                long long max_capture_rate, rxb200_fm_two_stage_plan *out, int *offsets_hz)
{
	return two_stage_plan(tuned_hz, n_channels, chain_rate, max_capture_rate, 0, 0, out, offsets_hz);
}

extern "C" int rxb200_fm_plan_capture_two_stage_at(const int64_t *tuned_hz, int n_channels, int chain_rate,
                                                   long long max_capture_rate, long long device_rate,
                                                   rxb200_fm_two_stage_plan *out, int *offsets_hz)
{
	long long G = 0;
	const int rc = device_guard(device_rate, &G);
	if (rc != RXB200_OK) { return rc; }
	return two_stage_plan(tuned_hz, n_channels, chain_rate, max_capture_rate, device_rate, G, out, offsets_hz);
}

// rxb200_fm_plan_capture_raster's rule; device_rate and G as for capture_plan
static int raster_plan(const int64_t *tuned_hz, int n_channels, int chain_rate, long long max_capture_rate,
                       long long device_rate, long long G, rxb200_fm_raster_plan *out, int *bins)
{
	if (!tuned_hz || !out || !bins) { set_error("null argument"); return RXB200_EINVAL; }
	long long fc = 0, M = 0, g = 0;
	int rc = capture_centre(tuned_hz, n_channels, chain_rate, G, &fc, &M, &g);
	if (rc != RXB200_OK) { return rc; }
	const long long R = M * chain_rate;
	rc = rate_check(R, M, max_capture_rate);
	if (rc == RXB200_OK) { rc = device_check(R, device_rate); }
	if (rc != RXB200_OK) { return rc; }
	long long a = R, b = g;                              // K0 = R / gcd(R, g), 1 for g = 0
	while (b) { const long long t = a % b; a = b; b = t; }
	const long long K = std::max(3ll, R / a);
	if (K > 4096) {
		set_error("raster capture plan: the channels' %lld Hz grid at a capture rate of %lld Hz needs %lld bins, above "
		          "4096; RXB200_CAPTURE_STAGES=2 takes channels off a grid", g, R, K);
		return RXB200_EINVAL;
	}
	for (int k = 0; k < n_channels; k++) {
		const long long o = tuned_hz[k] - fc;             // a multiple of R / K: o K / R is exact
		bins[k] = (int)((o * K / R % K + K) % K);
	}
	out->centre_hz = fc;
	out->capture_rate = (int)R;
	out->n_bins = (int)K;
	out->decim = (int)M;
	out->n_taps = (int)std::min(8191ll, 32 * M + 1);
	out->shift = 30;
	return RXB200_OK;
}

extern "C" int rxb200_fm_plan_capture_raster(const int64_t *tuned_hz, int n_channels, int chain_rate,
                                             long long max_capture_rate, rxb200_fm_raster_plan *out, int *bins)
{
	return raster_plan(tuned_hz, n_channels, chain_rate, max_capture_rate, 0, 0, out, bins);
}

extern "C" int rxb200_fm_plan_capture_raster_at(const int64_t *tuned_hz, int n_channels, int chain_rate,
                                                long long max_capture_rate, long long device_rate,
                                                rxb200_fm_raster_plan *out, int *bins)
{
	long long G = 0;
	const int rc = device_guard(device_rate, &G);
	if (rc != RXB200_OK) { return rc; }
	return raster_plan(tuned_hz, n_channels, chain_rate, max_capture_rate, device_rate, G, out, bins);
}

// The channel filter of rx_power's capture mode (include/rxb200.h, "rx_power hops of one capture"): a Blackman-windowed
// sinc with its cutoff at 1/(2M) cycles per sample, quantised to 2^shift / sum(g) and the rounding error put on the
// centre tap, so that the DC gain is 2^shift exactly.
extern "C" int rxb200_ddc_lowpass(int decim, int n_taps, int shift, int32_t *taps)
{
	if (!taps) { set_error("null argument"); return RXB200_EINVAL; }
	if (decim < 1 || decim > 4096 || n_taps < 1 || n_taps > 8191 || n_taps % 2 == 0 || shift < 0 || shift > 30) {
		set_error("lowpass decim %d, n_taps %d, shift %d: need 1 <= decim <= 4096, odd 1 <= n_taps <= 8191, 0 <= shift <= 30",
		          decim, n_taps, shift);
		return RXB200_EINVAL;
	}
	const int c = (n_taps - 1) / 2;
	double sum = 0.0;
	std::vector<double> g((size_t)n_taps);
	for (int j = 0; j < n_taps; j++) {
		const double x = (double)(j - c) / (double)decim;           // 2 * cutoff * (j - c)
		const double s = j == c ? 1.0 : sin(M_PI * x) / (M_PI * x);
		const double a = n_taps == 1 ? 0.0 : 2.0 * M_PI * (double)j / (double)(n_taps - 1);
		g[j] = s * (n_taps == 1 ? 1.0 : 0.42 - 0.5 * cos(a) + 0.08 * cos(2.0 * a));
		sum += g[j];
	}
	const double unity = (double)(1ll << shift);
	long long q = 0;
	for (int j = 0; j < n_taps; j++) {
		taps[j] = (int32_t)llround(unity * g[j] / sum);
		q += taps[j];
	}
	taps[c] += (int32_t)((1ll << shift) - q);
	return RXB200_OK;
}

// The resampler's prototype filter (include/rxb200.h, "capture from a device at its own rate"): a Blackman-windowed
// sinc over J L taps with its cutoff at 1/(2 max(L, N)) cycles per prototype sample, scaled so that each of the L
// phases sums to about 2^15, rounded, then each phase's sum made exactly 2^15 on its largest-magnitude tap.
extern "C" int rxb200_resample_lowpass(int up, int down, int taps_per_phase, int32_t *taps)
{
	if (!taps) { set_error("null argument"); return RXB200_EINVAL; }
	if (up < 1 || down < 1 || taps_per_phase < 1 || taps_per_phase > 1024 || (long long)taps_per_phase * up > (1ll << 22)) {
		set_error("resampler lowpass up %d, down %d, taps_per_phase %d: need up, down >= 1, 1 <= taps_per_phase <= 1024 "
		          "and taps_per_phase * up <= 2^22", up, down, taps_per_phase);
		return RXB200_EINVAL;
	}
	const long long L = up, J = taps_per_phase, n = J * L;
	const double c = (double)(n - 1) / 2.0, fc = 1.0 / (2.0 * (double)std::max(up, down));
	std::vector<double> g((size_t)n);
	double sum = 0.0;
	for (long long i = 0; i < n; i++) {
		const double x = 2.0 * fc * ((double)i - c);
		const double s = x == 0.0 ? 1.0 : sin(M_PI * x) / (M_PI * x);
		const double a = 2.0 * M_PI * (double)(i + 1) / (double)(n + 1);
		g[i] = s * (0.42 - 0.5 * cos(a) + 0.08 * cos(2.0 * a));
		sum += g[i];
	}
	const double scale = 32768.0 * (double)L / sum;
	for (long long i = 0; i < n; i++) { taps[i] = (int32_t)llround(g[i] * scale); }
	for (long long p = 0; p < L; p++) {
		long long s = 0, k = p;
		for (long long i = p; i < n; i += L) {
			s += taps[i];
			if (std::llabs(taps[i]) > std::llabs(taps[k])) { k = i; }
		}
		taps[k] += (int32_t)(32768 - s);
	}
	return RXB200_OK;
}

extern "C" int rxb200_plan_resample(long long device_rate, long long rate, long long span, rxb200_resampler *out)
{
	if (!out) { set_error("null argument"); return RXB200_EINVAL; }
	if (device_rate < 1 || device_rate > 2147483647ll || rate < 1 || rate > 2147483647ll || span < 0) {
		set_error("resampler plan: device rate %lld Hz, rate %lld Hz, span %lld Hz (need rates in [1, 2^31 - 1] and a "
		          "span >= 0)", device_rate, rate, span);
		return RXB200_EINVAL;
	}
	const long long G = (device_rate + 31) / 32, D = std::min(rate, device_rate) - span;
	if (D < G) {
		set_error("the channels span %lld Hz, too wide for a device at %lld Hz resampled to %lld Hz: the largest span "
		          "that fits is %lld Hz", span, device_rate, rate, std::min(rate, device_rate) - G);
		return RXB200_EINVAL;
	}
	long long a = rate, b = device_rate;
	while (b) { const long long t = a % b; a = b; b = t; }
	const long long L = rate / a, N = device_rate / a, J = 8 * (((6 * device_rate + D - 1) / D + 7) / 8);
	if (J * L > (1ll << 22)) {
		set_error("resampling by %lld/%lld needs %lld taps (%lld per phase), above 2^22", L, N, J * L, J);
		return RXB200_EUNSUPPORTED;
	}
	out->up = (int)L;
	out->down = (int)N;
	out->taps_per_phase = (int)J;
	out->taps = NULL;
	out->shift = 15;
	return RXB200_OK;
}

extern "C" int rxb200_resample_in_len(int up, int down, unsigned long long n0, size_t n_out, size_t *n_in)
{
	if (!n_in || up < 1 || down < 1) { set_error("resample_in_len: need up, down >= 1 and n_in"); return RXB200_EINVAL; }
	typedef unsigned __int128 u128;
	if (n_out == 0) { *n_in = 0; return RXB200_OK; }
	// output m is emitted by device sample floor(m N / L): the call must reach the last output's, m0 + n_out - 1
	const u128 L = (u128)up, N = (u128)down, m0 = ((u128)n0 * L + N - 1) / N;
	const u128 c = ((m0 + (u128)n_out - 1) * N) / L + 1 - (u128)n0;
	if (c > (u128)SIZE_MAX) { set_error("resample_in_len: %zu outputs need more than 2^64 device samples", n_out); return RXB200_EINVAL; }
	*n_in = (size_t)c;
	return RXB200_OK;
}

// The tiling of a sweep wider than one capture (include/rxb200.h, "wide sweeps in tiles"): c(k) is the centre of a run
// of k hops from its first hop, Mreq(k) the decimation a capture centred there needs.
static long long tile_centre(long long k, long long s) { return (k - 1) * s / 2; }
// G: the guard band of a device rate (0 without one), which the decimation floor leaves
static long long tile_decim(long long k, long long s, long long r, long long G)
{
	const long long c = tile_centre(k, s), half = std::max(c, (k - 1) * s - c);
	return (2 * half + r + G + r - 1) / r;
}

// a plan the rx_power planners take
static int power_plan_check(const rxb200_power_plan *plan, const char *what)
{
	const long long n = plan->params.n_hops, r = plan->rate, s = plan->freq_step;
	if (n < 1 || r < 1 || s < 0) {
		set_error("%s: plan with n_hops %lld, rate %lld, freq_step %lld (need n_hops, rate >= 1, freq_step >= 0)", what, n, r, s);
		return RXB200_EINVAL;
	}
	return RXB200_OK;
}

// rxb200_power_plan_tiles's rule; device_rate: 0, or the _at planner's checked device rate with its guard band G
static int power_tiles(const rxb200_power_plan *plan, long long max_capture_rate, long long device_rate, long long G,
                       rxb200_power_tiling *out, int *offsets_hz)
{
	if (!plan || !out) { set_error("null argument"); return RXB200_EINVAL; }
	int rc = power_plan_check(plan, "tiling");
	if (rc != RXB200_OK) { return rc; }
	const long long n = plan->params.n_hops, r = plan->rate, s = plan->freq_step;
	const long long top = device_rate ? std::min(max_capture_rate, device_rate) : max_capture_rate;
	const long long mcap = std::min(4096ll, std::min(top, 2147483647ll) / r);
	if (mcap < 1) {
		set_error("tiling: a capture rate of at most %lld Hz is below the hop rate %lld Hz", top, r);
		return RXB200_EINVAL;
	}
	if (tile_decim(1, s, r, G) > mcap) {
		set_error("tiling: one hop at %lld Hz with the guard band of a device at %lld Hz needs %lld Hz, above %lld Hz", r,
		          device_rate, tile_decim(1, s, r, G) * r, mcap * r);
		return RXB200_EINVAL;
	}
	long long hmax = 1;                                  // Mreq is non-decreasing in k
	while (hmax < n && tile_decim(hmax + 1, s, r, G) <= mcap) { hmax++; }
	const long long n_tiles = (n + hmax - 1) / hmax, h = (n + n_tiles - 1) / n_tiles, M = tile_decim(h, s, r, G);
	out->n_tiles = (int)n_tiles;
	out->hops_per_tile = (int)h;
	out->decim = (int)M;
	out->n_taps = (int)std::min(8191ll, 32 * M + 1);
	out->capture_rate = (int)(M * r);
	if (offsets_hz) {
		for (long long i = 0; i < n; i++) {
			const long long t = i / h, len = std::min(h, n - t * h);
			offsets_hz[i] = (int)((i - t * h) * s - tile_centre(len, s));
		}
	}
	return RXB200_OK;
}

extern "C" int rxb200_power_plan_tiles(const rxb200_power_plan *plan, long long max_capture_rate,
                                       rxb200_power_tiling *out, int *offsets_hz)
{
	return power_tiles(plan, max_capture_rate, 0, 0, out, offsets_hz);
}

extern "C" int rxb200_power_plan_tiles_at(const rxb200_power_plan *plan, long long max_capture_rate,
                                          long long device_rate, rxb200_power_tiling *out, int *offsets_hz)
{
	long long G = 0;
	const int rc = device_guard(device_rate, &G);
	if (rc != RXB200_OK) { return rc; }
	return power_tiles(plan, max_capture_rate, device_rate, G, out, offsets_hz);
}

// The rx_power shell's capture mode (include/rxb200.h, "rx_power plans at a device rate"): the centre of the hops, each
// hop's offset from it and the smallest M whose capture holds them all, with the guard band G of a device rate
static int power_capture(const rxb200_power_plan *plan, long long max_capture_rate, long long device_rate, long long G,
                         rxb200_fm_capture_plan *out, int *offsets_hz)
{
	if (!plan || !out) { set_error("null argument"); return RXB200_EINVAL; }
	int rc = power_plan_check(plan, "capture plan");
	if (rc != RXB200_OK) { return rc; }
	const long long n = plan->params.n_hops, r = plan->rate, s = plan->freq_step;
	const long long fc = plan->first_freq + (n - 1) * s / 2;
	long long span = 0;
	for (long long i = 0; i < n; i++) {
		const long long f = plan->first_freq + i * s - fc;
		span = std::max(span, 2 * std::llabs(f));
	}
	const long long M = (span + r + G + r - 1) / r, R = M * r;
	if (R > max_capture_rate || R > 2147483647ll || M > 4096) {
		// the rx_power shell appends ", above RXB200_CAPTURE_RATE=<cap>", its refusal since before this planner
		set_error("the span needs a capture rate of %lld Hz", R);
		return RXB200_EINVAL;
	}
	if (device_rate && R > device_rate) {
		set_error("the hops need a capture rate of %lld Hz, above the device rate of %lld Hz", R, device_rate);
		return RXB200_EUNSUPPORTED;
	}
	if (offsets_hz) {
		for (long long i = 0; i < n; i++) { offsets_hz[i] = (int)(plan->first_freq + i * s - fc); }
	}
	out->centre_hz = fc;
	out->decim = (int)M;
	out->capture_rate = (int)R;
	out->n_taps = (int)std::min(8191ll, 32 * M + 1);
	return RXB200_OK;
}

extern "C" int rxb200_power_plan_capture(const rxb200_power_plan *plan, long long max_capture_rate,
                                         rxb200_fm_capture_plan *out, int *offsets_hz)
{
	return power_capture(plan, max_capture_rate, 0, 0, out, offsets_hz);
}

extern "C" int rxb200_power_plan_capture_at(const rxb200_power_plan *plan, long long max_capture_rate,
                                            long long device_rate, rxb200_fm_capture_plan *out, int *offsets_hz)
{
	long long G = 0;
	const int rc = device_guard(device_rate, &G);
	if (rc != RXB200_OK) { return rc; }
	return power_capture(plan, max_capture_rate, device_rate, G, out, offsets_hz);
}

extern "C" int rxb200_power_tile(const rxb200_power_plan *plan, const rxb200_power_tiling *tl, int t,
                                 int *hop_begin, int *hop_end, int64_t *centre_hz)
{
	if (!plan || !tl || !hop_begin || !hop_end || !centre_hz) { set_error("null argument"); return RXB200_EINVAL; }
	if (t < 0 || t >= tl->n_tiles || tl->hops_per_tile < 1) {
		set_error("tile %d outside [0, %d)", t, tl->n_tiles);
		return RXB200_EINVAL;
	}
	const long long h = tl->hops_per_tile, b = (long long)t * h, e = std::min(b + h, (long long)plan->params.n_hops);
	if (b >= e) { set_error("tile %d of %d hops is empty", t, plan->params.n_hops); return RXB200_EINVAL; }
	*hop_begin = (int)b;
	*hop_end = (int)e;
	*centre_hz = plan->first_freq + (int64_t)b * plan->freq_step + (int64_t)tile_centre(e - b, plan->freq_step);
	return RXB200_OK;
}

// ---------------------------------------------------------------------------------- rx_power
#define RXB_MAXIMUM_RATE 2800000      /* src/rtl_power.c:74 */
#define RXB_MINIMUM_RATE 1000000      /* :75 */
#define RXB_DEFAULT_BUF  16384        /* :71 */
#define RXB_MAX_TUNES    10000        /* :111 */

// frequency_range() (src/rtl_power.c:431-543) on already-parsed numbers.
extern "C" int rxb200_power_plan_range(int64_t lower, int64_t upper, int64_t max_size, double crop,
                                       int boxcar, int comp_fir_size, int peak_hold, rxb200_power_plan *out)
{
	if (!out) { set_error("null argument"); return RXB200_EINVAL; }
	if (crop < 0.0 || crop >= 1.0 || upper <= lower || max_size <= 0) { set_error("bad range/crop"); return RXB200_EINVAL; }
	memset(out, 0, sizeof *out);
	int64_t bw_seen = 0, bw_used = 0, downsample = 1, passes = 0;
	int tune_count = 0, bin_e = 0;
	for (int i = 1; i < 1500; i++) {
		bw_seen = (upper - lower) / i;
		bw_used = (int64_t)((double)bw_seen / (1.0 - crop));
		if (bw_used > RXB_MAXIMUM_RATE) { continue; }
		tune_count = i;
		break;
	}
	if (bw_used <= 0) { set_error("unsupported bandwidth"); return RXB200_EINVAL; }
	if (bw_used < RXB_MINIMUM_RATE) {
		tune_count = 1;
		downsample = RXB_MAXIMUM_RATE / bw_used;
		if (downsample <= 0) { set_error("unsupported bandwidth"); return RXB200_EINVAL; }
		bw_used = bw_used * downsample;
	}
	if (!boxcar && downsample > 1) {
		passes = (int)log2((double)downsample);
		downsample = (int64_t)1 << passes;
		bw_used = (int)((double)(bw_seen * downsample) / (1.0 - crop));
	}
	double bin_size = 0.0;
	for (int i = 1; i <= 21; i++) {
		bin_e = i;
		bin_size = (double)bw_used / (double)(((int64_t)1 << i) * downsample);
		if (bin_size <= (double)max_size) { break; }
	}
	if (max_size >= RXB_MINIMUM_RATE) {
		bw_seen = max_size; bw_used = max_size;
		tune_count = (int)((upper - lower) / bw_seen);
		bin_e = 0; crop = 0;
	}
	if (tune_count <= 0) { set_error("no tuning ranges"); return RXB200_EINVAL; }
	if (tune_count > RXB_MAX_TUNES) { set_error("bandwidth too wide"); return RXB200_EINVAL; }
	int64_t buf_len = 2 * ((int64_t)1 << bin_e) * downsample;
	if (buf_len < RXB_DEFAULT_BUF) { buf_len = RXB_DEFAULT_BUF; }
	out->params.n_hops = tune_count; out->params.bin_e = bin_e; out->params.buf_len = (int)buf_len;
	out->params.downsample = (int)downsample; out->params.downsample_passes = (int)passes;
	out->params.comp_fir_size = comp_fir_size; out->params.boxcar = boxcar; out->params.peak_hold = peak_hold;
	out->rate = (int)bw_used; out->crop = crop;
	out->first_freq = lower + bw_seen / 2; out->freq_step = bw_seen;
	out->bin_size_hz = bin_size;
	return RXB200_OK;
}

// window shapes, src/rtl_power.c:322-401
static double window_value(int id, int i, int length)
{
	const double n1 = (double)(length - 1);
	double w;
	switch (id) {
	case RXB200_WIN_HAMMING:
		return 25.0 / 46.0 - (21.0 / 46.0) * cos(2 * i * M_PI / n1);
	case RXB200_WIN_BLACKMAN:
		return 7938.0 / 18608.0 - (9240.0 / 18608.0) * cos(2 * i * M_PI / n1) + (1430.0 / 18608.0) * cos(4 * i * M_PI / n1);
	case RXB200_WIN_BLACKMAN_HARRIS:
		return 0.35875 - 0.48829 * cos(2 * i * M_PI / n1) + 0.14128 * cos(4 * i * M_PI / n1) - 0.01168 * cos(6 * i * M_PI / n1);
	case RXB200_WIN_HANN_POISSON:
		return 0.5 * (1 - cos(2 * M_PI * i / n1)) * pow(M_E, (-2.0 * (double)abs((int)(n1 - 1 - 2 * i))) / n1);
	case RXB200_WIN_YOUSSEF:
		w = 0.35875 - 0.48829 * cos(2 * i * M_PI / n1) + 0.14128 * cos(4 * i * M_PI / n1) - 0.01168 * cos(6 * i * M_PI / n1);
		return w * pow(M_E, (-0.0025 * (double)abs((int)(n1 - 1 - 2 * i))) / n1);
	case RXB200_WIN_BARTLETT:
		w = (i - n1 / 2) / ((double)length / 2);
		return 1 - (w < 0 ? -w : w);
	case RXB200_WIN_HANN:
		return 0.5 * (1 - cos(2 * M_PI * i / n1));
	default:
		return 1.0;   // rectangle, kaiser (src/rtl_power.c:322, :385)
	}
}

extern "C" int rxb200_window_table(int window, int length, int *coefs)
{
	if (!coefs || length < 1 || window < 0 || window > RXB200_WIN_HANN) { set_error("bad window request"); return RXB200_EINVAL; }
	for (int i = 0; i < length; i++) { coefs[i] = (int)(256 * window_value(window, i, length)); }   // :1036
	return RXB200_OK;
}

extern "C" int rxb200_sine_table(int log2_n, int16_t *sine)
{
	if (!sine || log2_n < 0 || log2_n > 21) { set_error("bad sine table request"); return RXB200_EINVAL; }
	const int n = 1 << log2_n;
	for (int i = 0; i < n * 3 / 4; i++) {
		double d = (double)i * 2.0 * M_PI / n;
		sine[i] = (int16_t)(int)round(32767 * sin(d));   // src/rtl_power.c:250-251
	}
	return RXB200_OK;
}

// csv_dbm() (src/rtl_power.c:774-817) for one row, without the date/time prefix and without the
// zeroing (the device accumulators are cleared by rxb200_power_reset).
extern "C" int rxb200_power_row_len(int bin_e, double crop)
{
	if (bin_e < 0 || bin_e > 30) { return RXB200_EINVAL; }
	const int len = 1 << bin_e;
	const int i1 = 0 + (int)((double)len * crop * 0.5);
	const int i2 = (len - 1) - (int)((double)len * crop * 0.5);
	return (i2 >= i1 ? i2 - i1 + 1 : 0) + 1;
}

extern "C" int rxb200_power_format_db_row(const double *db, int bin_e, int64_t freq, int rate, int downsample,
                                          double crop, int samples, char *dst, size_t cap)
{
	if (!db || !dst) { set_error("null argument"); return RXB200_EINVAL; }
	const int len = 1 << bin_e, ds = downsample;
	const int n = rxb200_power_row_len(bin_e, crop);
	size_t w = 0;
#define RXB_EMIT(...)                                                        \
	do {                                                                     \
		int n__ = snprintf(dst + w, w < cap ? cap - w : 0, __VA_ARGS__);     \
		if (n__ < 0 || w + (size_t)n__ >= cap) { return RXB200_ECAPACITY; }  \
		w += (size_t)n__;                                                    \
	} while (0)
	int bin_count = (int)((double)len * (1.0 - crop));
	int bw2 = (int)(((double)rate * (double)bin_count) / (len * 2 * ds));
	RXB_EMIT("%lli, %lli, %.2f, %i, ", (long long)freq - bw2, (long long)freq + bw2,
	         (double)rate / (double)(len * ds), samples);
	for (int i = 0; i < n - 1; i++) { RXB_EMIT("%.2f, ", db[i]); }
	RXB_EMIT("%.2f\n", db[n - 1]);
#undef RXB_EMIT
	return (int)w;
}

extern "C" int rxb200_power_format_row(int64_t *avg, int bin_e, int64_t freq, int rate, int downsample,
                                       double crop, int samples, char *dst, size_t cap)
{
	if (!avg || !dst) { set_error("null argument"); return RXB200_EINVAL; }
	const int len = 1 << bin_e, ds = downsample;
	size_t w = 0;
#define RXB_EMIT(...)                                                        \
	do {                                                                     \
		int n__ = snprintf(dst + w, w < cap ? cap - w : 0, __VA_ARGS__);     \
		if (n__ < 0 || w + (size_t)n__ >= cap) { return RXB200_ECAPACITY; }  \
		w += (size_t)n__;                                                    \
	} while (0)
	if (bin_e > 0) {
		avg[0] = avg[1];                       // DC bin copied from its neighbour (:784)
		for (int i = 0; i < len / 2; i++) {    // half-swap (:786-790)
			int64_t t = avg[i]; avg[i] = avg[i + len / 2]; avg[i + len / 2] = t;
		}
	}
	int bin_count = (int)((double)len * (1.0 - crop));
	int bw2 = (int)(((double)rate * (double)bin_count) / (len * 2 * ds));
	RXB_EMIT("%lli, %lli, %.2f, %i, ", (long long)freq - bw2, (long long)freq + bw2,
	         (double)rate / (double)(len * ds), samples);
	int i1 = 0 + (int)((double)len * crop * 0.5);
	int i2 = (len - 1) - (int)((double)len * crop * 0.5);
	double dbm;
	for (int i = i1; i <= i2; i++) {
		dbm = (double)avg[i];
		dbm /= (double)rate;
		dbm /= (double)samples;
		dbm = 10 * log10(dbm);
		RXB_EMIT("%.2f, ", dbm);
	}
	dbm = (double)avg[i2] / ((double)rate * (double)samples);   // last bin once more (:807)
	if (bin_e == 0) { dbm = ((double)avg[0] / ((double)rate * (double)samples)); }
	dbm = 10 * log10(dbm);
	RXB_EMIT("%.2f\n", dbm);
#undef RXB_EMIT
	return (int)w;
}
