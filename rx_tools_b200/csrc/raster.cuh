// raster.cuh — the raster down-converter of raster mixing handles (include/rxb200.h, "raster mixing handles"): the host
// side the capture front (capture_front.cuh) needs from fm_raster.cu.  A raster handle, rx_fm's or rx_sdr's, is one whose
// CaptureFront runs raster_front instead of a single-stage down-converter.
#pragma once
#include <vector>
#include "common.cuh"

namespace rxb {

// The refusals of K, bins and the taps' bound (the ddc itself is checked by ddc_check), before any device work.
int raster_check(int n_bins, const int *bins, int n_channels, const rxb200_ddc *ddc);

// The twiddle matrix of a raster and its shape: Wt[n][k] (Np rows of Kp doubles) is the transposed [2K][2C] matrix,
// zero-padded to Kp = 2K rounded up to 16 and Np = 2C rounded up to 64.
struct RasterPlan {
	int K = 0, C = 0, Kp = 0, Np = 0;
	long long group = 0;                  // frames per group of branch sums (RXB200_RASTER_SCRATCH_BYTES)
	std::vector<double> wt;               // host copy, built by plan()
	int plan(int n_bins, const int *bins, int n_channels);
	size_t w_bytes() const { return (size_t)Np * Kp * sizeof(double); }
	size_t v_bytes(long long frames) const { return (size_t)frames * Kp * sizeof(double); }
};

// One call's raster front stage on the current device: n_out outputs per channel from the capture at src (hist: the
// T - 1 samples before it; r0: src index of the first emission point; p0: the residue mod K of src[0]'s sample index)
// to dst, channel c's output u at complex element c * stride + u of rx_sdr format fmt (RXB200_SDR_OUT_CS16: the int16
// pair word), through V (room for min(n_out, plan.group) frames).
int raster_front(const RasterPlan &p, const double *d_wt, double *V, const uint32_t *src, const uint32_t *hist,
                 const int32_t *taps, int M, int T, int S, long long r0, unsigned p0, long long n_out, void *dst,
                 long long stride, cudaStream_t st, int fmt = RXB200_SDR_OUT_CS16);

}  // namespace rxb
