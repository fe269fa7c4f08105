// fm_two_stage.cu — the two-stage down-converter (include/rxb200.h, "two-stage mixing handles"): channels at any offset
// through a coarse polyphase stage on a K-bin grid, then a fine NCO stage per channel at the coarse rate.  The coarse
// stage is the raster down-converter (fm_raster.cu: raster_branch_kernel, raster_dft_kernel) run for the distinct bins
// of the channels, writing each bin's coarse stream to a scratch row after that bin's last T2 - 1 coarse samples.  The
// fine stage is ddc.cuh's down-converter with the rx_power NCO mixer (as power_ddc_kernel) whose grid rows each stage
// one bin's coarse stream (the ddc_row hook below) and whose channels write to their own rows of the output, as int16
// pair words or, for the rx_sdr two-stage handle (sdr_mix.cu), in a recorded format (SdrOut).
#include <algorithm>
#include <cstring>
#include <numeric>
#include "two_stage.cuh"

namespace rxb {

// ddc_body's mixer policy for the fine stage: channel k (in bin order) of the grid row mixes coarse sample m of its bin
// by NCO entry ((m w_k + 2^15) mod 2^32) >> 16, the phase taken per CTA as (uint32)g0 * w_k and stepped by off * w_k in
// uint32 arithmetic (as NcoMix), and writes its call output u to word u of its own row of dst.
struct BinMix {
	const int2 *nco;                 // NCO_ENTRIES (c, s) pairs
	const uint32_t *w;               // each channel's fine word, channels in bin order
	const int *row;                  // each channel's row of dst, channels in bin order
	const int4 *rows;                // each grid row: (its bin's slot, its first channel, its channel count, 0)
	long long src_stride;            // words between two slots' rows of the coarse scratch
	long long dst_stride;            // words (elements, for SdrOut) between two rows of dst
	template <typename Args>
	struct RowOf {
		const Args &a;
		int c0, c;
		uint32_t g0, w, th0;             // channel c's word and its phase at the CTA's first staged sample
		long long u0;
		__device__ RowOf(const Args &a, int c0, int, long long u0, long long g0)
		    : a(a), c0(c0), g0((uint32_t)(unsigned long long)g0), u0(u0) {}
		__device__ void chan(int k) { c = k; w = __ldg(a.mix.w + c0 + k); th0 = g0 * w; }
		__device__ const int2 *entry(int off) const { return a.mix.nco + ((th0 + (uint32_t)off * w + 32768u) >> 16); }
		__device__ uint32_t *out(int u) const
		{
			return a.dst + (long long)__ldg(a.mix.row + c0 + c) * a.mix.dst_stride + u0 + u;
		}
	};
	using Row = RowOf<DdcArgs<BinMix>>;
};

// the staging hook: grid row y stages its bin's row of the coarse scratch, whose T - 1 samples before a.src's column are
// that bin's fine history, so the history is contiguous with the stream
template <typename Args>
__device__ __forceinline__ DdcRow bin_row(const Args &a)
{
	const int4 g = a.mix.rows[blockIdx.y];
	const uint32_t *src = a.src + g.x * a.mix.src_stride;
	return DdcRow{g.y, g.z, src, src - (a.T - 1)};
}
template <>
__device__ __forceinline__ DdcRow ddc_row(const DdcArgs<BinMix> &a) { return bin_row(a); }
template <int F>
__device__ __forceinline__ DdcRow ddc_row(const DdcArgs<SdrOut<BinMix, F>> &a) { return bin_row(a); }

template <typename Acc>
__global__ void __launch_bounds__(DDC_THREADS) fine_ddc_kernel(const DdcArgs<BinMix> a) { ddc_body<Acc>(a); }
// the same writing rx_sdr format F (the rx_sdr two-stage handle; CS16 is the instance above)
template <typename Acc, int F>
__global__ void __launch_bounds__(DDC_THREADS) fine_ddc_kernel(const DdcArgs<SdrOut<BinMix, F>> a) { ddc_body<Acc>(a); }

namespace {

long long floor_div(long long a, long long b)
{
	const long long q = a / b;
	return (a % b != 0 && (a < 0) != (b < 0)) ? q - 1 : q;
}

__int128 floor_div(__int128 a, __int128 b)
{
	const __int128 q = a / b;
	return (a % b != 0 && (a < 0) != (b < 0)) ? q - 1 : q;
}

size_t align16(size_t n) { return (n + 15) / 16 * 16; }

template <int F>
int fine_launch(const DdcArgs<BinMix> &b, bool wide, cudaStream_t st, int rows)
{
	const DdcArgs<SdrOut<BinMix, F>> a = ddc_args_as<SdrOut<BinMix, F>>(b);
	return ddc_launch(a, wide ? fine_ddc_kernel<long long, F> : fine_ddc_kernel<int, F>, st, rows);
}

}  // namespace

int TwoStage::plan(int capture_rate, int n_bins, const int *offsets_hz, int n_channels, const rxb200_ddc *coarse,
                   const rxb200_ddc *fine)
{
	static const int bin0 = 0;
	int rc = raster_check(n_bins, &bin0, 1, coarse);        // K and sum |h1| < 2^22
	if (rc != RXB200_OK) { return rc; }
	if ((long long)coarse->decim * fine->decim > 4096) {
		set_error("two-stage decimation M1 M2 = %lld > 4096", (long long)coarse->decim * fine->decim);
		return RXB200_EINVAL;
	}
	std::vector<int> bins((size_t)std::max(n_channels, 0));
	std::vector<uint32_t> words(bins.size());
	rc = rxb200_two_stage_word(capture_rate, n_bins, coarse->decim, offsets_hz, n_channels, bins.data(), words.data());
	if (rc != RXB200_OK) { return rc; }
	M2 = fine->decim; T2 = fine->n_taps; S2 = fine->shift;
	n_ch = n_channels;
	std::vector<int> ord((size_t)n_ch), slot_bins, row_of((size_t)n_ch);
	std::iota(ord.begin(), ord.end(), 0);
	std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) { return bins[(size_t)a] < bins[(size_t)b]; });
	std::vector<uint32_t> w((size_t)n_ch);
	std::vector<int4> rows;
	for (int k = 0; k < n_ch; k++) {
		const int c = ord[(size_t)k], b = bins[(size_t)c];
		const bool new_bin = slot_bins.empty() || slot_bins.back() != b;
		if (new_bin) { slot_bins.push_back(b); }
		if (new_bin || rows.back().z == MIX_GROUP) { rows.push_back(make_int4((int)slot_bins.size() - 1, k, 0, 0)); }
		rows.back().z++;
		w[(size_t)k] = words[(size_t)c];
		row_of[(size_t)k] = c;
	}
	n_rows = (int)rows.size();
	rc = r.plan(n_bins, slot_bins.data(), (int)slot_bins.size());
	if (rc != RXB200_OK) { return rc; }
	// G frames of branch sums and coarse rows, with the rows' histories, under the scratch bound (at least one DFT tile)
	const long long fixed = (long long)r.C * H() * (long long)sizeof(uint32_t);
	const long long per = (long long)r.Kp * (long long)sizeof(double) + (long long)r.C * (long long)sizeof(uint32_t);
	G = std::max<long long>(64, ((long long)RXB200_RASTER_SCRATCH_BYTES - fixed) / per / 64 * 64);
	o_nco = align16(r.w_bytes());
	o_rows = o_nco + align16((size_t)NCO_ENTRIES * sizeof(int2));
	o_w = o_rows + align16((size_t)n_rows * sizeof(int4));
	o_row = o_w + align16((size_t)n_ch * sizeof(uint32_t));
	blk.assign(o_row + align16((size_t)n_ch * sizeof(int)), 0);
	memcpy(blk.data(), r.wt.data(), r.w_bytes());
	rxb200_nco_table(reinterpret_cast<int32_t *>(blk.data() + o_nco));
	memcpy(blk.data() + o_rows, rows.data(), rows.size() * sizeof(int4));
	memcpy(blk.data() + o_w, w.data(), w.size() * sizeof(uint32_t));
	memcpy(blk.data() + o_row, row_of.data(), row_of.size() * sizeof(int));
	r.wt.clear();
	return RXB200_OK;
}

int TwoStage::upload(const rxb200_ddc *fine, cudaStream_t st)
{
	ddc_check(fine, &wide2);
	DdcBlock b;
	const int rc = ddc_upload(blk, fine, st, &b);
	if (rc != RXB200_OK) { return rc; }
	d_blk = b.d;
	d_taps2 = b.taps;
	blk.clear();
	for (int i = 0; i < 2; i++) {
		RXB_CUDA(cudaMallocAsync((void **)&fh[i], hist_bytes(), st));
		RXB_CUDA(cudaMemsetAsync(fh[i], 0, hist_bytes(), st));
	}
	return RXB200_OK;
}

int TwoStage::front(const DdcFilter &f, const uint32_t *src, long long r0, unsigned p0, long long n1,
                    unsigned long long nco0, int ph2, double *d_v, uint32_t *d_y, uint32_t *dst, long long stride,
                    cudaStream_t st, int fmt)
{
	if (n1 <= 0) { return RXB200_OK; }
	const long long H = this->H(), F_max = std::min(G, n1), ys = H + F_max;
	const size_t hw = (size_t)H * sizeof(uint32_t), yw = (size_t)ys * sizeof(uint32_t);
	DdcArgs<BinMix> a{};
	a.taps = d_taps2;
	a.n_ch = n_ch; a.M = M2; a.T = T2; a.S = S2;
	a.mix = BinMix{reinterpret_cast<const int2 *>(d_blk + o_nco), reinterpret_cast<const uint32_t *>(d_blk + o_w),
	               reinterpret_cast<const int *>(d_blk + o_row), reinterpret_cast<const int4 *>(d_blk + o_rows), ys,
	               stride};
	for (long long l = 0; l < n1; l += F_max) {
		const long long F = std::min(F_max, n1 - l);
		if (H) { RXB_CUDA(cudaMemcpy2DAsync(d_y, yw, fh[l == 0 ? cur : cur ^ 1], hw, hw, r.C, cudaMemcpyDeviceToDevice, st)); }
		int rc = raster_front(r, reinterpret_cast<const double *>(d_blk), d_v, src, f.hist[f.cur], f.taps, f.M, f.T, f.S,
		                      r0 + l * f.M, p0, F, d_y + H, ys, st);
		if (rc != RXB200_OK) { return rc; }
		const long long qa = (ph2 + l) / M2, qb = (ph2 + l + F) / M2;
		if (qb > qa) {
			a.src = d_y + H;
			a.n_out = qb - qa;
			a.r0 = (M2 - 1) - (ph2 + l) % M2;
			a.pos = nco0 + (unsigned long long)l;
			a.dst = reinterpret_cast<uint32_t *>(reinterpret_cast<unsigned char *>(dst) + qa * sdr_elem_bytes(fmt));
			rc = fmt == RXB200_CVT_CS16_CS8  ? fine_launch<RXB200_CVT_CS16_CS8>(a, wide2, st, n_rows)
			   : fmt == RXB200_CVT_CS16_CU8  ? fine_launch<RXB200_CVT_CS16_CU8>(a, wide2, st, n_rows)
			   : fmt == RXB200_CVT_CS16_CF32 ? fine_launch<RXB200_CVT_CS16_CF32>(a, wide2, st, n_rows)
			                                 : ddc_launch(a, wide2 ? fine_ddc_kernel<long long> : fine_ddc_kernel<int>, st, n_rows);
			if (rc != RXB200_OK) { return rc; }
		}
		// each slot's last H coarse samples: the row's words [F, F + H) of (history, the group's outputs)
		if (H) { RXB_CUDA(cudaMemcpy2DAsync(fh[cur ^ 1], hw, d_y + F, yw, hw, r.C, cudaMemcpyDeviceToDevice, st)); }
	}
	pending = true;
	return RXB200_OK;
}

int TwoStage::reset(cudaStream_t st)
{
	RXB_CUDA(cudaMemsetAsync(fh[0], 0, hist_bytes(), st));
	RXB_CUDA(cudaMemsetAsync(fh[1], 0, hist_bytes(), st));
	cur = 0;
	pending = false;
	return RXB200_OK;
}

void TwoStage::release(cudaStream_t st)
{
	for (void *p : {(void *)d_blk, (void *)fh[0], (void *)fh[1]}) {
		if (p) { cudaFreeAsync(p, st); }
	}
	d_blk = nullptr; fh[0] = fh[1] = nullptr;
}

}  // namespace rxb

using namespace rxb;

extern "C" int rxb200_two_stage_word(int capture_rate, int n_bins, int coarse_decim, const int *offsets_hz,
                                     int n_channels, int *bins, uint32_t *words)
{
	if (!offsets_hz || !bins || !words || n_channels < 1) { set_error("bad two-stage arguments (NULL, or n_channels < 1)"); return RXB200_EINVAL; }
	const long long R = capture_rate, K = n_bins, M1 = coarse_decim;
	if (R <= 0) { set_error("capture_rate %d must be > 0", capture_rate); return RXB200_EINVAL; }
	if (K < 3 || K > 4096) { set_error("two-stage n_bins %d: need 3 <= n_bins <= 4096", n_bins); return RXB200_EINVAL; }
	if (M1 < 1 || M1 > 4096) { set_error("coarse decim %d: need 1 <= decim <= 4096", coarse_decim); return RXB200_EINVAL; }
	const __int128 D = (__int128)K * R;
	for (int c = 0; c < n_channels; c++) {
		const long long f = offsets_hz[c];
		if (2 * (f < 0 ? -f : f) >= R) {
			set_error("channel %d: offset %lld needs |offset| < capture_rate/2 (%lld)", c, f, R);
			return RXB200_EINVAL;
		}
	}
	for (int c = 0; c < n_channels; c++) {
		const long long f = offsets_hz[c];
		long long b = floor_div(f * K + R / 2, R) % K;
		if (b < 0) { b += K; }
		const long long bp = 2 * b > K ? b - K : b;                 // b in (-K/2, K/2]
		const __int128 N = (__int128)(f * K - bp * R) * M1;
		const __int128 q = floor_div(N * ((__int128)1 << 32) + D / 2, D);
		bins[c] = (int)b;
		words[c] = (uint32_t)(unsigned __int128)q;
	}
	return RXB200_OK;
}

extern "C" int rxb200_two_stage_device(int capture_rate, int n_bins, const int *offsets_hz, int n_channels,
                                       unsigned long long n0, const rxb200_ddc *coarse, const rxb200_ddc *fine,
                                       const int16_t *d_src, size_t n_complex, int16_t *d_dst, void *stream)
{
	if (!d_src || !d_dst) { set_error("bad two-stage request (null pointer)"); return RXB200_EINVAL; }
	if (((uintptr_t)d_src & 3u) || ((uintptr_t)d_dst & 3u)) { set_error("pointers must be 4-byte aligned"); return RXB200_EINVAL; }
	int rc = ddc_check(fine, nullptr);
	if (rc != RXB200_OK) { return rc; }
	rc = ddc_check(coarse, nullptr);
	if (rc != RXB200_OK) { return rc; }
	TwoStage t;
	rc = t.plan(capture_rate, n_bins, offsets_hz, n_channels, coarse, fine);
	if (rc != RXB200_OK) { return rc; }
	const long long M1 = coarse->decim, n_out = (long long)(n_complex / (size_t)(M1 * fine->decim));
	if (n_out == 0) { return RXB200_OK; }
	const long long n1 = n_out * fine->decim, F = std::min(t.G, n1);   // the coarse outputs the fine ones need
	const cudaStream_t st = (cudaStream_t)stream;
	std::vector<unsigned char> none;
	DdcBlock cb;
	rc = ddc_upload(none, coarse, st, &cb);
	if (rc != RXB200_OK) { return rc; }
	DdcFilter f;
	f.M = coarse->decim; f.T = coarse->n_taps; f.S = coarse->shift;
	f.taps = const_cast<int32_t *>(cb.taps);
	f.hist[0] = const_cast<uint32_t *>(cb.hist);
	double *v = nullptr;
	uint32_t *y = nullptr;
	rc = t.upload(fine, st);
	if (rc == RXB200_OK && (cudaMallocAsync((void **)&v, t.r.v_bytes(F), st) != cudaSuccess ||
	                        cudaMallocAsync((void **)&y, t.y_words(F) * sizeof(uint32_t), st) != cudaSuccess)) {
		set_error("two-stage scratch allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
		rc = RXB200_ECUDA;
	}
	if (rc == RXB200_OK) {
		rc = t.front(f, reinterpret_cast<const uint32_t *>(d_src), M1 - 1, (unsigned)(n0 % (unsigned long long)n_bins), n1,
		             n0 / (unsigned long long)M1, 0, v, y, reinterpret_cast<uint32_t *>(d_dst), n_out, st);
	}
	if (v) { cudaFreeAsync(v, st); }
	if (y) { cudaFreeAsync(y, st); }
	t.release(st);
	cudaFreeAsync(cb.d, st);
	return rc;
}
