// two_stage.cuh — the two-stage down-converter of two-stage mixing handles (include/rxb200.h, "two-stage mixing
// handles"): the host side the capture front (capture_front.cuh) needs from fm_two_stage.cu.  A two-stage handle, rx_fm's
// or rx_sdr's, is one whose CaptureFront's DdcFilter is the coarse stage's (M1, T1, h1, S1 and the raw capture history)
// and which runs TwoStage::front; rx_sdr's has it write a recorded format.
#pragma once
#include <vector>
#include "ddc.cuh"
#include "raster.cuh"

namespace rxb {

// The plan of a two-stage down-converter and the device state it carries between calls.  The coarse stage runs the
// raster kernels (raster_front) for the distinct bins of the channels, its slots in ascending bin order; the fine stage
// runs fine_ddc_kernel with the channels in bin order, each grid row a run of at most MIX_GROUP channels of one bin.
struct TwoStage {
	RasterPlan r;                         // the coarse stage: one raster channel per slot
	int M2 = 1, T2 = 1, S2 = 0;
	bool wide2 = false;                   // the fine kernel accumulates in 64 bits
	int n_ch = 0, n_rows = 0;
	long long G = 0;                      // coarse frames per group under RXB200_RASTER_SCRATCH_BYTES
	std::vector<unsigned char> blk;       // host image of the device block (the layout of plan())
	size_t o_nco = 0, o_rows = 0, o_w = 0, o_row = 0;   // its sections; the twiddle matrix is at 0
	unsigned char *d_blk = nullptr;       // the block, then the reversed fine taps (ddc_upload)
	const int32_t *d_taps2 = nullptr;
	// per slot, the last T2 - 1 coarse samples before the stream's coarse position, [slots][T2 - 1]: fh[cur] is live, a
	// call writes the next into fh[cur ^ 1] and commit makes it live (only a call that made coarse samples does)
	uint32_t *fh[2] = {nullptr, nullptr};
	int cur = 0;
	bool pending = false;

	// the refusals of the rule's K, coarse taps, R, offsets and M1 M2, then the plan; host only
	int plan(int capture_rate, int n_bins, const int *offsets_hz, int n_channels, const rxb200_ddc *coarse,
	         const rxb200_ddc *fine);
	// the device block and zeroed histories on the current device, ordered on st
	int upload(const rxb200_ddc *fine, cudaStream_t st);
	long long H() const { return (long long)T2 - 1; }
	size_t y_words(long long frames) const { return (size_t)r.C * (size_t)(H() + frames); }
	size_t hist_bytes() const { return std::max<size_t>(1, (size_t)r.C * (size_t)H()) * sizeof(uint32_t); }
	// One call's two stages: the n1 coarse outputs whose emission points fall in the call (the first at src index r0,
	// with coarse index nco0 for the fine mixer, and (ph2 + l) mod M2 = M2 - 1 marking a fine emission at local coarse
	// output l), in groups of at most G frames through d_v (G frames of branch sums) and d_y ([slots][T2 - 1 + G]);
	// fine output q of channel c to element c * stride + q of dst in format fmt (RXB200_SDR_OUT_CS16: the int16 pair
	// word).  f: the coarse filter; p0: the residue mod K of src[0]'s index.
	int front(const DdcFilter &f, const uint32_t *src, long long r0, unsigned p0, long long n1,
	          unsigned long long nco0, int ph2, double *d_v, uint32_t *d_y, uint32_t *dst, long long stride,
	          cudaStream_t st, int fmt = RXB200_SDR_OUT_CS16);
	void commit() { if (pending && T2 > 1) { cur ^= 1; } pending = false; }
	int reset(cudaStream_t st);
	void release(cudaStream_t st);
};

}  // namespace rxb
