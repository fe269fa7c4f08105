// capture_front.cuh — the front stage of the handles that take channels from one wideband capture (fm_mix.cu's
// rxb200_fm_mix, sdr_mix.cu's rxb200_sdr_mix): one of three kinds of down-converter from the capture to the channels'
// decimated streams, with the state it carries between calls.  A single stage is ddc.cuh's down-converter with the
// handle's own mixer (the handle launches it); a raster is fm_raster.cu's polyphase channelizer (raster_front); two
// stages are fm_two_stage.cu's coarse raster then per-channel NCO stage (TwoStage::front).  The front owns the capture
// count, and so the rule that makes a recording's bytes independent of how the capture is cut into calls: each call's
// kernels start at the count's phases, and commit advances the count and the histories.  A front with a resampler
// attached (resample_stage.cuh) takes device-rate samples: each call resamples them to the capture first, and every
// count below that takes a call's length counts device samples.  A front whose input format is not CS16
// (input_stage.cuh) widens each call's elements to CS16 first, ahead of the resampler.  Its host code is in ddc.cu.
#pragma once
#include <algorithm>
#include "ddc.cuh"
#include "input_stage.cuh"
#include "raster.cuh"
#include "resample_stage.cuh"
#include "two_stage.cuh"

namespace rxb {

struct CaptureFront {
	enum Kind { SINGLE, RASTER, TWO_STAGE };
	Kind kind = SINGLE;
	DdcFilter f;                                 // the single stage's or the raster's filter, the coarse one for two stages
	unsigned long long pos = 0;                  // capture samples since create or reset
	RasterPlan r;                                // raster: its shape, its twiddle matrix at d_wt
	double *d_wt = nullptr;
	double *d_v = nullptr; size_t v_cap = 0;     // raster, two stages: the (coarse) branch sums (doubles)
	TwoStage ts;                                 // two stages: the plan, the fine stage and the bins' histories
	uint32_t *d_y = nullptr; size_t y_cap = 0;   // two stages: the coarse rows (words)
	cudaEvent_t ev0 = nullptr, ev1 = nullptr;    // around the front's kernels of the last call
	ResampleStage rs;                            // from the device rate, once attached
	InputStage in;                               // the input format, widened to CS16 ahead of rs

	// The refusals of each kind, in the order the handles report them, then its host plan; no device work.  A single
	// stage is its filter's check alone.
	int plan_single(const rxb200_ddc *ddc) { return ddc_check(ddc, &f.wide); }
	int plan_raster(int n_bins, const int *bins, int n_channels, const rxb200_ddc *ddc);
	int plan_two_stage(int capture_rate, int n_bins, const int *offsets_hz, int n_channels, const rxb200_ddc *coarse,
	                   const rxb200_ddc *fine);
	// On the current device, after a plan: the events, the filter ddc (the coarse one for two stages; NULL: a single
	// stage without a filter, whose decimation is 1 and which carries no history) and the kind's device state (fine:
	// the two stages' fine filter), ordered on st.  The caller releases the front when it fails.
	int create(const rxb200_ddc *ddc, const rxb200_ddc *fine, cudaStream_t st);
	bool filtered() const { return f.taps != nullptr; }

	// M, or M1 M2 for two stages
	size_t decim() const { return (size_t)f.M * (size_t)(kind == TWO_STAGE ? ts.M2 : 1); }
	// the outputs per channel of c capture samples at the current count: those whose emission points m M + M - 1 fall
	// in them
	size_t dec_len(size_t c) const
	{
		const unsigned long long M = decim();
		return (size_t)((pos + c) / M - pos / M);
	}
	// the outputs per channel of a call of c device samples (capture samples without a resampler)
	size_t out_len(size_t c) const { return dec_len(rs.out_len(c)); }
	// Attaches the resampler, which only a front that has taken no sample since create or reset accepts (and only
	// once); its refusals precede any device work
	int set_device_rate(const rxb200_resampler *r);
	// The input format (RXB200_IN_*), which only a front that has taken no sample since create or reset accepts; its
	// refusals precede any device work
	int set_input_format(int fmt);

	// One call's front stage on the current device, ordered on st: the c device samples at src (a device pointer, in
	// the input format), widened to CS16 unless that is CS16, resampled to the capture when a resampler is attached, to the out_len(c) outputs per channel of the n_ch channels
	// at dst, channel k's output u at element k * stride + u in rx_sdr format fmt (RXB200_SDR_OUT_CS16: the int16
	// pair word); then the carry of the raw history.  ev0 and ev1 bracket the kernels.  Two stages run whenever the call has coarse outputs, since those advance the bins'
	// histories even when no fine output falls in the call; the other kinds run when the call has outputs.  single
	// launches a single stage from the DdcArgs<Mix> it is given, every field but mix filled (src, n_out and pos
	// describe the capture).  ev0 and ev1 also bracket the widening and the resampler.  Nothing becomes live before
	// commit(c).
	template <typename Mix, typename Single>
	int call(const int16_t *src, size_t c_dev, void *dst, long long stride, int fmt, int n_ch, cudaStream_t st,
	         Single single)
	{
		const size_t c = rs.out_len(c_dev);
		const long long n = (long long)dec_len(c);
		const long long r0 = (long long)(f.M - 1) - (long long)(pos % (unsigned long long)f.M);
		RXB_CUDA(cudaEventRecord(ev0, st));
		const uint32_t *w = nullptr, *x = nullptr;
		int rc = in.run(src, c_dev, st, &w);
		if (rc != RXB200_OK) { return rc; }
		rc = rs.run(w, c_dev, st, &x);
		if (rc != RXB200_OK) { return rc; }
		if (kind == TWO_STAGE) {
			const unsigned long long M1 = (unsigned long long)f.M, ma = pos / M1;
			const long long n1 = (long long)((pos + c) / M1 - ma);
			if (n1) {
				const long long F = std::min(ts.G, n1);
				RXB_CUDA(reserve(d_v, v_cap, (size_t)F * (size_t)ts.r.Kp));
				RXB_CUDA(reserve(d_y, y_cap, ts.y_words(F)));
				rc = ts.front(f, x, (long long)(ma * M1 + M1 - 1 - pos), (unsigned)(pos % (unsigned long long)ts.r.K), n1,
				              ma, (int)(ma % (unsigned long long)ts.M2), d_v, d_y, static_cast<uint32_t *>(dst), stride, st,
				              fmt);
			}
		} else if (n && kind == RASTER) {
			RXB_CUDA(reserve(d_v, v_cap, (size_t)std::min(n, r.group) * (size_t)r.Kp));
			rc = raster_front(r, d_wt, d_v, x, f.hist[f.cur], f.taps, f.M, f.T, f.S, r0,
			                  (unsigned)(pos % (unsigned long long)r.K), n, dst, stride, st, fmt);
		} else if (n) {
			DdcArgs<Mix> a{};
			a.src = x;
			a.hist = f.hist[f.cur];
			a.n_out = n;
			a.r0 = r0;
			a.pos = pos;
			a.dst = static_cast<uint32_t *>(dst);
			a.taps = f.taps;
			a.n_ch = n_ch; a.M = f.M; a.T = f.T; a.S = f.S;
			rc = single(a);
		}
		if (rc != RXB200_OK) { return rc; }
		RXB_CUDA(cudaEventRecord(ev1, st));
		return f.carry(x, c, st);
	}
	// the histories a call of c device samples wrote become live, and the counts advance past it
	void commit(size_t c)
	{
		pos += rs.out_len(c);
		rs.commit(c);
		f.commit();
		ts.commit();
	}
	// every history zeroed behind any call still running on st, and the counts cleared (a resampler stays attached)
	int reset(cudaStream_t st);
	// frees the device state, once no kernel of the front's is in flight: the caller has synchronised st, the stream
	// they ran on (or destroyed it, st = 0)
	void release(cudaStream_t st);
	// the time between ev0 and ev1 of the last call
	int kernel_ms(float *ms);
};

}  // namespace rxb
