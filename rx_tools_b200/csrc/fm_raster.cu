// fm_raster.cu — the raster down-converter (include/rxb200.h, "raster mixing handles"): the channels of a K-bin raster
// over one capture through a polyphase channelizer.  The rule's sum over taps regroups exactly by the residue
// rho = (e_m - j) mod K of each sample's index, since the twiddle of a sample depends on its index only through rho:
//     v_rho[m] = sum_{j<T, (e_m - j) mod K = rho} h[j] x[e_m - j],     A_k[m] = sum_rho tw[(k rho) mod K] v_rho[m].
// raster_branch_kernel makes the rows v[m] (2K doubles) of a group of frames, shared by every channel; raster_dft_kernel
// multiplies them by the handle's constant real [2K][2C] twiddle matrix with DMMA (mma.sync m8n8k4 f64) and rounds,
// saturates and writes each channel's outputs, as int16 pair words or in an rx_sdr format (sdr_mix.cu's raster kind).
// Every value is an integer: |v| <= sum |h| 2^15 < 2^37, every product |v| 2^15 < 2^52 and every partial sum at most
// sum |h| 2^31 < 2^53, so fp64 holds them all exactly and the result does not depend on the order the tensor cores sum
// in.
#include <algorithm>
#include <cstring>
#include "ddc.cuh"
#include "raster.cuh"

namespace rxb {

#define RAS_THREADS 256
#define RAS_SPAN 8192                 // capture samples a branch CTA stages at most (T <= 8192: one frame always fits)
#define RAS_BM 64                     // DFT tile: frames
#define RAS_BN 64                     // DFT tile: output columns (32 channels)
#define RAS_BK 16                     // DFT tile: input columns per stage
#define RAS_LD (RAS_BK + 4)           // shared row stride in doubles: the fragment loads of a warp hit distinct banks

struct BranchArgs {
	const uint32_t *src;              // the call's capture, one word per complex sample
	const uint32_t *hist;             // the T - 1 raw capture samples before src
	const int32_t *taps;              // reversed: taps[t] = h[T - 1 - t]
	double *V;                        // [F][Kp]: (Re, Im) of v_rho at 2 rho, zeros past 2K
	long long F;                      // frames of this group
	long long b0;                     // src index of the group's first window's first sample
	int K, Kp, M, T;
	unsigned p0;                      // the residue mod K of src[0]'s sample index
	int ws;                           // staged samples between two frames' windows: M when T >= M, else T
	unsigned ws_m;                    // floor((2^32 - 1) / ws)
	int U;                            // frames per CTA
};

// One CTA: U consecutive frames.  It stages the capture samples their windows cover once (the history before the
// call's first sample), as ddc_body does, then one thread per (frame, rho) sums the taps t = t0, t0 + K, ... of its
// residue class in fp64 (exact: every product and sum is an integer below 2^37).
__global__ void __launch_bounds__(RAS_THREADS) raster_branch_kernel(const BranchArgs a)
{
	extern __shared__ int4 ras_smem[];
	const int T = a.T, K = a.K, half = a.Kp / 2;
	const int room = (a.U - 1) * a.ws + T;
	int32_t *s_h = reinterpret_cast<int32_t *>(ras_smem);
	uint32_t *s_x = reinterpret_cast<uint32_t *>(s_h + T);
	int *s_q = reinterpret_cast<int *>(s_x + room);                    // each frame's window start, mod K
	const long long u0 = (long long)blockIdx.x * a.U;
	const int U = (int)min((long long)a.U, a.F - u0);
	const int n = (U - 1) * a.ws + T;
	const long long b0 = a.b0 + u0 * a.M;                              // >= -(T - 1)
	for (int j = threadIdx.x; j < T; j += blockDim.x) { s_h[j] = a.taps[j]; }
	for (int s = threadIdx.x; s < n; s += blockDim.x) {
		const long long i = b0 + ddc_off(s, a);
		s_x[s] = i >= 0 ? __ldg(a.src + i) : a.hist[(T - 1) + i];
	}
	for (int u = threadIdx.x; u < U; u += blockDim.x) {
		const long long q = ((long long)a.p0 + b0 + (long long)u * a.M) % K;
		s_q[u] = (int)(q < 0 ? q + K : q);
	}
	__syncthreads();
	for (int e = threadIdx.x; e < U * half; e += blockDim.x) {
		const int u = e / half, rho = e - u * half;
		double vr = 0.0, vi = 0.0;
		if (rho < K) {
			int t = rho - s_q[u];
			if (t < 0) { t += K; }
			const uint32_t *z = s_x + u * a.ws;
			for (; t < T; t += K) {
				const uint32_t w = z[t];
				const double h = (double)s_h[t];
				vr = fma(h, (double)(int16_t)(w & 0xffffu), vr);
				vi = fma(h, (double)(int16_t)(w >> 16), vi);
			}
		}
		reinterpret_cast<double2 *>(a.V + (u0 + u) * a.Kp)[rho] = make_double2(vr, vi);
	}
}

struct DftArgs {
	const double *V;                  // [F][Kp]
	const double *Wt;                 // [Np][Kp]
	long long F;
	int Kp, n_col, S;                 // n_col = 2C
	void *dst;                        // channel c's output u is complex element c * stride + u of the format's row at dst
	long long stride;
};

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem, int bytes)
{
	const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
	asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(bytes));
}

// Y = V Wt^T for one 64 x 64 tile (64 frames, 32 channels): eight warps of 32 x 16, each a 4 x 2 grid of DMMA 8 x 8
// tiles over k steps of 4; the operands stream through shared memory in stages of 16 input columns with cp.async,
// two stages in flight.  Frames past F load as zeros and store nothing.  The epilogue converts each (I, Q) pair to
// int64 (exact), rounds by S and saturates with ddc_out, and writes one element per channel and frame in rx_sdr format
// F (sdr_put): the int16 pair word for RXB200_SDR_OUT_CS16 (rx_fm's raster and two-stage handles), a CS16 conversion
// for the rx_sdr raster handle.
template <int F>
__global__ void __launch_bounds__(RAS_THREADS) raster_dft_kernel(const DftArgs a)
{
	__shared__ __align__(16) double s_a[2][RAS_BM][RAS_LD];
	__shared__ __align__(16) double s_b[2][RAS_BN][RAS_LD];
	const int tid = (int)threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int g = lane >> 2, t4 = lane & 3;
	const int wm = (warp & 1) * 32, wn = (warp >> 1) * 16;
	const long long m0 = (long long)blockIdx.x * RAS_BM;
	const int n0 = (int)blockIdx.y * RAS_BN;
	double acc[4][2][2];
#pragma unroll
	for (int i = 0; i < 4; i++) {
#pragma unroll
		for (int j = 0; j < 2; j++) { acc[i][j][0] = 0.0; acc[i][j][1] = 0.0; }
	}
	auto load = [&](int buf, int k0) {
#pragma unroll
		for (int r = 0; r < 2; r++) {
			const int q = tid + r * RAS_THREADS, row = q >> 3, c2 = (q & 7) * 2;   // 64 rows x 8 16-byte pieces
			const bool ok = m0 + row < a.F;
			cp_async16(&s_a[buf][row][c2], ok ? a.V + (m0 + row) * a.Kp + k0 + c2 : a.V, ok ? 16 : 0);
			cp_async16(&s_b[buf][row][c2], a.Wt + (long long)(n0 + row) * a.Kp + k0 + c2, 16);
		}
		asm volatile("cp.async.commit_group;\n" ::);
	};
	const int nk = a.Kp / RAS_BK;
	load(0, 0);
	for (int kt = 0; kt < nk; kt++) {
		if (kt + 1 < nk) {
			load((kt + 1) & 1, (kt + 1) * RAS_BK);
			asm volatile("cp.async.wait_group 1;\n" ::);
		} else {
			asm volatile("cp.async.wait_group 0;\n" ::);
		}
		__syncthreads();
		const int buf = kt & 1;
#pragma unroll
		for (int kk = 0; kk < RAS_BK; kk += 4) {
			double fa[4], fb[2];
#pragma unroll
			for (int i = 0; i < 4; i++) { fa[i] = s_a[buf][wm + i * 8 + g][kk + t4]; }    // A: row g, column t4
#pragma unroll
			for (int j = 0; j < 2; j++) { fb[j] = s_b[buf][wn + j * 8 + g][kk + t4]; }    // B: row t4, column g
#pragma unroll
			for (int i = 0; i < 4; i++) {
#pragma unroll
				for (int j = 0; j < 2; j++) {
					asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n"
					             : "+d"(acc[i][j][0]), "+d"(acc[i][j][1])
					             : "d"(fa[i]), "d"(fb[j]));
				}
			}
		}
		__syncthreads();                    // the stage is read before the next iteration's load overwrites it
	}
	// C: row g, columns 2 t4 and 2 t4 + 1 of each 8 x 8 tile, which are I and Q of one channel
#pragma unroll
	for (int i = 0; i < 4; i++) {
		const long long f = m0 + wm + i * 8 + g;
#pragma unroll
		for (int j = 0; j < 2; j++) {
			const int col = n0 + wn + j * 8 + 2 * t4;
			if (f < a.F && col < a.n_col) {
				const int yi = ddc_out((long long)acc[i][j][0], a.S), yq = ddc_out((long long)acc[i][j][1], a.S);
				sdr_put<F>(a.dst, (long long)(col >> 1) * a.stride + f, ((uint32_t)yi & 0xffffu) | ((uint32_t)yq << 16));
			}
		}
	}
}

int raster_check(int n_bins, const int *bins, int n_channels, const rxb200_ddc *ddc)
{
	if (n_bins < 3 || n_bins > 4096) { set_error("raster n_bins %d: need 3 <= n_bins <= 4096", n_bins); return RXB200_EINVAL; }
	if (!bins || n_channels < 1) { set_error("bad raster bins (NULL, or n_channels < 1)"); return RXB200_EINVAL; }
	for (int c = 0; c < n_channels; c++) {
		if (bins[c] < 0 || bins[c] >= n_bins) {
			set_error("raster bin %d of channel %d outside [0, %d)", bins[c], c, n_bins);
			return RXB200_EINVAL;
		}
	}
	unsigned long long sum = 0;
	for (int j = 0; j < ddc->n_taps; j++) {
		const long long h = ddc->taps[j];
		sum += (unsigned long long)(h < 0 ? -h : h);
	}
	if (sum >= (1ull << 22)) { set_error("raster taps: sum |h| = %llu >= 2^22", sum); return RXB200_EINVAL; }
	return RXB200_OK;
}

int RasterPlan::plan(int n_bins, const int *bins, int n_channels)
{
	K = n_bins; C = n_channels;
	Kp = (2 * K + RAS_BK - 1) / RAS_BK * RAS_BK;
	Np = (2 * C + RAS_BN - 1) / RAS_BN * RAS_BN;
	group = (long long)(RXB200_RASTER_SCRATCH_BYTES / ((size_t)Kp * sizeof(double))) / RAS_BM * RAS_BM;
	std::vector<int32_t> tw(2 * (size_t)K);
	size_t L = 0;
	const int rc = rxb200_fm_mix_table(K, 1, tw.data(), tw.size(), &L);
	if (rc != RXB200_OK) { return rc; }
	wt.assign((size_t)Np * Kp, 0.0);
	for (int c = 0; c < C; c++) {
		double *re = wt.data() + (size_t)(2 * c) * Kp, *im = re + Kp;
		for (int rho = 0; rho < K; rho++) {
			const int r = (int)(((long long)bins[c] * rho) % K);
			const double cw = tw[2 * (size_t)r], sw = tw[2 * (size_t)r + 1];
			re[2 * rho] = cw; re[2 * rho + 1] = -sw;      // I = c vr - s vi
			im[2 * rho] = sw; im[2 * rho + 1] = cw;       // Q = s vr + c vi
		}
	}
	return RXB200_OK;
}

int raster_front(const RasterPlan &p, const double *d_wt, double *V, const uint32_t *src, const uint32_t *hist,
                 const int32_t *taps, int M, int T, int S, long long r0, unsigned p0, long long n_out, void *dst,
                 long long stride, cudaStream_t st, int fmt)
{
	void (*const dft)(DftArgs) = fmt == RXB200_CVT_CS16_CS8  ? raster_dft_kernel<RXB200_CVT_CS16_CS8>
	                           : fmt == RXB200_CVT_CS16_CU8  ? raster_dft_kernel<RXB200_CVT_CS16_CU8>
	                           : fmt == RXB200_CVT_CS16_CF32 ? raster_dft_kernel<RXB200_CVT_CS16_CF32>
	                                                         : raster_dft_kernel<RXB200_SDR_OUT_CS16>;
	int dev = 0, n_sm = 0;
	RXB_CUDA(cudaGetDevice(&dev));
	RXB_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
	BranchArgs b{};
	b.src = src; b.hist = hist; b.taps = taps; b.V = V;
	b.K = p.K; b.Kp = p.Kp; b.M = M; b.T = T; b.p0 = p0;
	b.ws = T >= M ? M : T;
	b.ws_m = 0xffffffffu / (unsigned)b.ws;
	DftArgs d{};
	d.V = V; d.Wt = d_wt; d.Kp = p.Kp; d.n_col = 2 * p.C; d.S = S; d.stride = stride;
	for (long long f0 = 0; f0 < n_out; f0 += p.group) {
		const long long F = std::min(p.group, n_out - f0);
		b.F = F;
		b.b0 = f0 * M + r0 - (T - 1);
		long long U = (long long)(RAS_SPAN - T) / b.ws + 1;
		U = std::max(1ll, std::min(U, (F + 2ll * n_sm - 1) / (2ll * n_sm)));
		b.U = (int)U;
		const size_t smem = ((size_t)T + (size_t)(U - 1) * b.ws + T + (size_t)U) * sizeof(int32_t);
		RXB_CUDA(cudaFuncSetAttribute(raster_branch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
		raster_branch_kernel<<<(unsigned)((F + U - 1) / U), RAS_THREADS, smem, st>>>(b);
		RXB_CUDA(cudaGetLastError());
		d.F = F;
		d.dst = static_cast<unsigned char *>(dst) + f0 * sdr_elem_bytes(fmt);
		dft<<<dim3((unsigned)((F + RAS_BM - 1) / RAS_BM), (unsigned)(p.Np / RAS_BN)), RAS_THREADS, 0, st>>>(d);
		RXB_CUDA(cudaGetLastError());
	}
	return RXB200_OK;
}

}  // namespace rxb

using namespace rxb;

extern "C" int rxb200_raster_device(int n_bins, const int *bins, int n_channels, unsigned long long n0,
                                    const rxb200_ddc *ddc, const int16_t *d_src, size_t n_complex, int16_t *d_dst,
                                    void *stream)
{
	if (!d_src || !d_dst) { set_error("bad raster request (null pointer)"); return RXB200_EINVAL; }
	if (((uintptr_t)d_src & 3u) || ((uintptr_t)d_dst & 3u)) { set_error("pointers must be 4-byte aligned"); return RXB200_EINVAL; }
	int rc = rxb::ddc_check(ddc, nullptr);
	if (rc != RXB200_OK) { return rc; }
	rc = raster_check(n_bins, bins, n_channels, ddc);
	if (rc != RXB200_OK) { return rc; }
	const long long n_out = (long long)(n_complex / (size_t)ddc->decim);
	if (n_out == 0) { return RXB200_OK; }
	RasterPlan p;
	rc = p.plan(n_bins, bins, n_channels);
	if (rc != RXB200_OK) { return rc; }
	const cudaStream_t st = (cudaStream_t)stream;
	std::vector<unsigned char> h(p.w_bytes());
	memcpy(h.data(), p.wt.data(), h.size());
	DdcBlock blk;
	rc = ddc_upload(h, ddc, st, &blk);
	if (rc != RXB200_OK) { return rc; }
	double *V = nullptr;
	if (cudaMallocAsync((void **)&V, p.v_bytes(std::min(n_out, p.group)), st) != cudaSuccess) {
		set_error("raster scratch allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
		cudaFreeAsync(blk.d, st);
		return RXB200_ECUDA;
	}
	rc = raster_front(p, reinterpret_cast<const double *>(blk.d), V, reinterpret_cast<const uint32_t *>(d_src), blk.hist,
	                  blk.taps, ddc->decim, ddc->n_taps, ddc->shift, ddc->decim - 1, (unsigned)(n0 % (unsigned)n_bins),
	                  n_out, reinterpret_cast<uint32_t *>(d_dst), n_out, st);
	cudaFreeAsync(V, st);
	cudaFreeAsync(blk.d, st);
	return rc;
}
