// resample.cu — the rational resampler (include/rxb200.h, "capture from a device at its own rate"): a device's CS16
// stream at the rate it runs at, R_dev, to a capture plan's rate R = R_dev L / N, by the exact polyphase rule.  The
// handle carries the device-sample count and the last J - 1 raw samples between calls in a DdcFilter (ddc.cuh), whose
// taps are here the prototype phase-major, so that the bytes never depend on how the stream is cut into calls.
#include <algorithm>
#include <cstring>
#include <new>
#include <vector>
#include "common.cuh"
#include "resample_stage.cuh"

namespace rxb {

#define RS_THREADS 256
#define RS_SPAN 8192                 // device samples a CTA stages at most (J <= 1024: one output always fits)
#define RS_MAX_U 512                 // outputs per CTA at most: u * (N mod L) + L stays below 2^31
#define RS_SMEM_TAPS 12288           // taps held in shared memory at most (48 KiB); more are read through L1 / L2

typedef unsigned __int128 u128;

struct ResampleArgs {
	const uint32_t *src;             // the call's samples, one word per complex sample
	const uint32_t *hist;            // the J - 1 raw samples before src
	uint32_t *dst;                   // one word per output
	const int32_t *taps;             // phase-major: taps[p J + j] = h[p + j L]
	long long n_out;                 // outputs of the call
	long long q0;                    // src index of the first output's q (>= 0)
	long long nq;                    // floor(N / L)
	int p0;                          // the first output's phase
	int L, J, S;
	int nr;                          // N mod L
	unsigned L_m;                    // floor((2^32 - 1) / L)
	int U;                           // outputs per CTA
	int lpo;                         // lanes per output (a power of two <= 32)
};

// One CTA: outputs [b U, b U + U) of the call.  Output i = b U + u has t - t_first = i N, so with N = nq L + nr its q is
// q0 + i nq + floor((p0 + i nr) / L) and its phase (p0 + i nr) mod L; the CTA's first is found with one 64-bit division
// and the rest from v = pa + u nr < 2^31 with a multiply-high and one correction.  The CTA stages the samples its
// outputs read once, [q_first - (J - 1), q_last], and runs each J-tap dot product on lpo lanes with a shuffle reduction.
// Acc: int when max_p sum |h_p| * 32768 + 2^(S-1) < 2^31, else long long (no partial sum can overflow either way).
template <typename Acc, bool SmemTaps>
__global__ void __launch_bounds__(RS_THREADS) resample_kernel(const ResampleArgs a)
{
	extern __shared__ int4 rs_smem[];
	const int J = a.J, L = a.L;
	uint32_t *s_x = reinterpret_cast<uint32_t *>(rs_smem);
	const long long i0 = (long long)blockIdx.x * a.U;
	const int U = (int)min((long long)a.U, a.n_out - i0);
	const unsigned long long v0 = (unsigned long long)a.p0 + (unsigned long long)i0 * (unsigned long long)a.nr;
	const unsigned long long qa = v0 / (unsigned long long)L;
	const int pa = (int)(v0 - qa * (unsigned long long)L);
	const long long qt = a.q0 + i0 * a.nq + (long long)qa;             // src index of the CTA's first output's q
	const unsigned vl = (unsigned)pa + (unsigned)(U - 1) * (unsigned)a.nr;
	const int n = (int)((long long)(U - 1) * a.nq + (long long)(vl / (unsigned)L)) + J;   // staged samples
	const long long b0 = qt - (J - 1);                                  // src index of the first staged sample
	const int32_t *h_all = a.taps;
	if (SmemTaps) {
		int32_t *s_h = reinterpret_cast<int32_t *>(s_x + ((n + 3) & ~3));
		for (int k = threadIdx.x; k < L * J; k += blockDim.x) { s_h[k] = __ldg(a.taps + k); }
		h_all = s_h;
	}
	for (int s = threadIdx.x; s < n; s += blockDim.x) {
		const long long i = b0 + s;
		s_x[s] = i >= 0 ? __ldg(a.src + i) : a.hist[(J - 1) + i];
	}
	__syncthreads();
	const int lane = (int)threadIdx.x & (a.lpo - 1), sub = (int)threadIdx.x / a.lpo, n_sub = (int)blockDim.x / a.lpo;
	for (int ub = 0; ub < U; ub += n_sub) {                              // the same trip count on every lane of a warp
		const int u = ub + sub;
		Acc ai = 0, aq = 0;
		if (u < U) {
			const unsigned v = (unsigned)pa + (unsigned)u * (unsigned)a.nr;
			unsigned d = __umulhi(v, a.L_m);
			int p = (int)(v - d * (unsigned)L);
			if (p >= L) { d++; p -= L; }
			const uint32_t *z = s_x + ((long long)u * a.nq + d) + (J - 1);   // z[-j] = x[q - j]
			const int32_t *h = h_all + (long long)p * J;
			for (int j = lane; j < J; j += a.lpo) {
				const uint32_t w = z[-j];
				const Acc c = (Acc)h[j];
				ai += c * (Acc)(int16_t)(w & 0xffffu);
				aq += c * (Acc)(int16_t)(w >> 16);
			}
		}
		for (int o = a.lpo >> 1; o > 0; o >>= 1) {
			ai += __shfl_xor_sync(0xffffffffu, ai, o);
			aq += __shfl_xor_sync(0xffffffffu, aq, o);
		}
		if (u < U && lane == 0) {
			a.dst[i0 + u] = ((uint32_t)ddc_out(ai, a.S) & 0xffffu) | ((uint32_t)ddc_out(aq, a.S) << 16);
		}
	}
}

// (resample_stage.cuh)
int resample_check(const rxb200_resampler *rs, bool *wide)
{
	if (!rs || !rs->taps) { set_error("null resampler or taps"); return RXB200_EINVAL; }
	if (rs->up < 1 || rs->down < 1 || rs->taps_per_phase < 1 || rs->taps_per_phase > 1024 ||
	    (long long)rs->taps_per_phase * rs->up > (1ll << 22) || rs->shift < 0 || rs->shift > 62) {
		set_error("resampler up %d, down %d, taps_per_phase %d, shift %d: need up, down >= 1, 1 <= taps_per_phase <= "
		          "1024, taps_per_phase * up <= 2^22 and 0 <= shift <= 62", rs->up, rs->down, rs->taps_per_phase,
		          rs->shift);
		return RXB200_EINVAL;
	}
	// The 2^63 refusal below is the stated bound, but the checks above already keep it from firing: J <= 1024 taps of
	// |h| <= 2^31 give sum |h_p| <= 2^41, so g <= 2^56 + 2^61 < 2^62.  Only the int32 / int64 choice depends on the taps.
	unsigned long long worst = 0;
	for (int p = 0; p < rs->up; p++) {
		unsigned long long s = 0;
		for (int j = 0; j < rs->taps_per_phase; j++) {
			const long long h = rs->taps[p + (long long)j * rs->up];
			s += (unsigned long long)(h < 0 ? -h : h);
		}
		worst = std::max(worst, s);
	}
	const unsigned long long g = worst * 32768ull + (rs->shift ? 1ull << (rs->shift - 1) : 0ull);
	if (g >= (1ull << 63)) { set_error("max over phases of sum |taps| * 32768 + 2^(shift-1) >= 2^63"); return RXB200_EINVAL; }
	*wide = g >= (1ull << 31);
	return RXB200_OK;
}

namespace {

// the prototype phase-major: pm[p J + j] = h[p + j L]
std::vector<int32_t> phase_major(const rxb200_resampler *rs)
{
	const size_t L = (size_t)rs->up, J = (size_t)rs->taps_per_phase;
	std::vector<int32_t> pm(L * J);
	for (size_t p = 0; p < L; p++) {
		for (size_t j = 0; j < J; j++) { pm[p * J + j] = rs->taps[p + j * L]; }
	}
	return pm;
}

// ceil(n L / N), exactly
u128 first_out(u128 n, long long L, long long N) { return (n * (u128)L + (u128)(N - 1)) / (u128)N; }

}  // namespace

// (resample_stage.cuh)
size_t out_count(unsigned long long n0, size_t c, long long L, long long N)
{
	return (size_t)(first_out((u128)n0 + c, L, N) - first_out(n0, L, N));
}

// (resample_stage.cuh)
int resample_launch(long long L, long long N, int J, int S, bool wide, const int32_t *taps, const uint32_t *src,
                    const uint32_t *hist, unsigned long long n0, size_t c, uint32_t *dst, cudaStream_t st)
{
	const u128 m0 = first_out(n0, L, N), t0 = m0 * (u128)N;
	ResampleArgs a{};
	a.n_out = (long long)(first_out((u128)n0 + c, L, N) - m0);
	if (a.n_out == 0) { return RXB200_OK; }
	a.src = src; a.hist = hist; a.dst = dst; a.taps = taps;
	a.q0 = (long long)(t0 / (u128)L - (u128)n0);
	a.p0 = (int)(t0 % (u128)L);
	a.nq = N / L; a.nr = (int)(N % L);
	a.L = (int)L; a.J = J; a.S = S;
	a.L_m = 0xffffffffu / (unsigned)L;
	a.lpo = 1;
	while (a.lpo < 32 && a.lpo < J) { a.lpo <<= 1; }
	int dev = 0, n_sm = 0;
	RXB_CUDA(cudaGetDevice(&dev));
	RXB_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
	// U outputs read at most (L - 1 + (U - 1) N) / L + J samples: keep that within RS_SPAN, and leave two CTAs per SM
	long long U = std::min<long long>(RS_MAX_U, (long long)(RS_SPAN - J - 1) * L / N + 1);
	U = std::max(1ll, std::min(U, (a.n_out + 2ll * n_sm - 1) / (2ll * n_sm)));
	a.U = (int)U;
	const long long room = (L - 1 + (U - 1) * N) / L + J;
	const bool smem_taps = L * J <= RS_SMEM_TAPS;
	const size_t smem = (size_t)((room + 3) & ~3ll) * sizeof(uint32_t) + (smem_taps ? (size_t)(L * J) * sizeof(int32_t) : 0);
	void (*kern)(ResampleArgs) = wide ? (smem_taps ? resample_kernel<long long, true> : resample_kernel<long long, false>)
	                                  : (smem_taps ? resample_kernel<int, true> : resample_kernel<int, false>);
	RXB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
	kern<<<(unsigned)((a.n_out + U - 1) / U), RS_THREADS, smem, st>>>(a);
	RXB_CUDA(cudaGetLastError());
	return RXB200_OK;
}

size_t ResampleStage::max_out(size_t c) const
{
	return on() ? (size_t)(((u128)c * (u128)L + (u128)(N - 1)) / (u128)N) : c;
}

int ResampleStage::attach(const rxb200_resampler *rs)
{
	bool wide = false;
	const int rc = resample_check(rs, &wide);
	if (rc != RXB200_OK) { return rc; }
	const std::vector<int32_t> pm = phase_major(rs);
	DdcFilter g;
	g.M = 1; g.T = rs->taps_per_phase; g.S = rs->shift; g.wide = wide;
	cudaError_t e = cudaMalloc(&g.taps, pm.size() * sizeof(int32_t));
	if (e == cudaSuccess) { e = cudaMemcpy(g.taps, pm.data(), pm.size() * sizeof(int32_t), cudaMemcpyHostToDevice); }
	const int hc = e == cudaSuccess ? g.alloc_hist() : RXB200_ECUDA;
	if (hc != RXB200_OK) {
		if (e != cudaSuccess) { set_error("resampler upload failed: %s", cudaGetErrorString(e)); }
		g.release();
		return hc;
	}
	L = rs->up; N = rs->down;
	f = g;
	pos = 0;
	return RXB200_OK;
}

int ResampleStage::run(const uint32_t *src, size_t c, cudaStream_t st, const uint32_t **out)
{
	if (!on()) { *out = src; return RXB200_OK; }
	RXB_CUDA(reserve(d_y, y_cap, std::max<size_t>(1, out_len(c))));   // at least one word: the front's carry reads it
	const int rc = resample_launch(L, N, f.T, f.S, f.wide, f.taps, src, f.hist[f.cur], pos, c, d_y, st);
	if (rc != RXB200_OK) { return rc; }
	*out = d_y;
	return f.carry(src, c, st);
}

int ResampleStage::reset(cudaStream_t st)
{
	if (on()) {
		const int rc = f.reset(st);
		if (rc != RXB200_OK) { return rc; }
	}
	pos = 0;
	return RXB200_OK;
}

void ResampleStage::release()
{
	if (on()) { f.release(); }
	cudaFree(d_y);
}

}  // namespace rxb

using namespace rxb;

struct rxb200_resample {
	int device = 0;
	long long L = 1, N = 1;
	cudaStream_t st = nullptr;
	DdcFilter f;                                 // T = J, S; taps: the prototype phase-major; the raw history
	unsigned long long pos = 0;                  // device samples since create or reset
	cudaEvent_t ev0 = nullptr, ev1 = nullptr;    // around the kernels of the last call (group)
	int16_t *d_cap = nullptr; size_t cap_cap = 0;         // host calls: the stream (int16 elements)
	int16_t *d_out = nullptr; size_t out_cap = 0;         // host calls: the outputs (int16 elements)
};

namespace {

int check_call(const rxb200_resample *r, const int16_t *cs16, size_t n_int16, const int16_t *out, size_t out_cap,
               bool device, size_t *n)
{
	if (!r || !cs16 || !out) { set_error("null argument"); return RXB200_EINVAL; }
	if (n_int16 % 2 != 0) { set_error("n_int16=%zu must be even", n_int16); return RXB200_EINVAL; }
	if (device && (((uintptr_t)cs16 & 3u) || ((uintptr_t)out & 3u))) {
		set_error("d_cs16 and d_out must be 4-byte aligned");
		return RXB200_EINVAL;
	}
	*n = out_count(r->pos, n_int16 / 2, r->L, r->N);
	if (*n > out_cap) { set_error("%zu outputs need out_cap >= %zu (have %zu)", *n, *n, out_cap); return RXB200_ECAPACITY; }
	return RXB200_OK;
}

// One checked call on device pointers: the kernel over the c samples at src, then the history and the count, which
// become live only when everything was enqueued.
int device_call(rxb200_resample *r, const int16_t *src, size_t c, int16_t *dst)
{
	const uint32_t *s = reinterpret_cast<const uint32_t *>(src);
	RXB_CUDA(cudaEventRecord(r->ev0, r->st));
	int rc = resample_launch(r->L, r->N, r->f.T, r->f.S, r->f.wide, r->f.taps, s, r->f.hist[r->f.cur], r->pos, c,
	                         reinterpret_cast<uint32_t *>(dst), r->st);
	if (rc != RXB200_OK) { return rc; }
	RXB_CUDA(cudaEventRecord(r->ev1, r->st));
	rc = r->f.carry(s, c, r->st);
	if (rc != RXB200_OK) { return rc; }
	r->f.commit();
	r->pos += c;
	return RXB200_OK;
}

}  // namespace

extern "C" void rxb200_resample_destroy(rxb200_resample *r)
{
	if (!r) { return; }
	cudaSetDevice(r->device);
	if (r->st) { cudaStreamSynchronize(r->st); }
	r->f.release();
	cudaFree(r->d_cap); cudaFree(r->d_out);
	if (r->ev0) { cudaEventDestroy(r->ev0); }
	if (r->ev1) { cudaEventDestroy(r->ev1); }
	if (r->st) { cudaStreamDestroy(r->st); }
	delete r;
}

extern "C" int rxb200_resample_create(const rxb200_resampler *rs, int device, rxb200_resample **out)
{
	if (!out) { set_error("null argument"); return RXB200_EINVAL; }
	*out = nullptr;
	bool wide = false;
	const int rc = resample_check(rs, &wide);
	if (rc != RXB200_OK) { return rc; }
	rxb200_resample *r = new (std::nothrow) rxb200_resample();
	if (!r) { return RXB200_ENOMEM; }
	r->device = device;
	r->L = rs->up; r->N = rs->down;
	r->f.M = 1; r->f.T = rs->taps_per_phase; r->f.S = rs->shift; r->f.wide = wide;
	const std::vector<int32_t> pm = phase_major(rs);
	RXB_CUDA_OR(cudaSetDevice(device), delete r);
	RXB_CUDA_OR(cudaStreamCreateWithFlags(&r->st, cudaStreamNonBlocking), delete r);
	RXB_CUDA_OR(cudaEventCreate(&r->ev0), rxb200_resample_destroy(r));
	RXB_CUDA_OR(cudaEventCreate(&r->ev1), rxb200_resample_destroy(r));
	RXB_CUDA_OR(cudaMalloc(&r->f.taps, pm.size() * sizeof(int32_t)), rxb200_resample_destroy(r));
	RXB_CUDA_OR(cudaMemcpy(r->f.taps, pm.data(), pm.size() * sizeof(int32_t), cudaMemcpyHostToDevice),
	            rxb200_resample_destroy(r));
	const int hc = r->f.alloc_hist();
	if (hc != RXB200_OK) { rxb200_resample_destroy(r); return hc; }
	*out = r;
	return RXB200_OK;
}

extern "C" int rxb200_resample_reset(rxb200_resample *r)
{
	if (!r) { set_error("null argument"); return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(r->device));
	const int rc = r->f.reset(r->st);               // behind any call still running on the handle's stream
	if (rc != RXB200_OK) { return rc; }
	r->pos = 0;
	return RXB200_OK;
}

extern "C" int rxb200_resample_out_len(const rxb200_resample *r, size_t n_int16, size_t *n_out)
{
	if (!r || !n_out) { set_error("null argument"); return RXB200_EINVAL; }
	*n_out = out_count(r->pos, n_int16 / 2, r->L, r->N);
	return RXB200_OK;
}

extern "C" int rxb200_resample_process_device(rxb200_resample *r, const int16_t *d_cs16, size_t n_int16, int16_t *d_out,
                                              size_t out_cap, size_t *n_out, int sync)
{
	size_t n = 0;
	int rc = check_call(r, d_cs16, n_int16, d_out, out_cap, true, &n);
	if (rc != RXB200_OK) { return rc; }
	if (n_int16 > 0) {
		RXB_CUDA(cudaSetDevice(r->device));
		rc = device_call(r, d_cs16, n_int16 / 2, d_out);
		if (rc != RXB200_OK) { return rc; }
		if (sync) { RXB_CUDA(cudaStreamSynchronize(r->st)); }
	}
	if (n_out) { *n_out = n; }
	return RXB200_OK;
}

extern "C" int rxb200_resample_process(rxb200_resample *r, const int16_t *cs16, size_t n_int16, int16_t *out,
                                       size_t out_cap, size_t *n_out)
{
	size_t n = 0;
	int rc = check_call(r, cs16, n_int16, out, out_cap, false, &n);
	if (rc != RXB200_OK) { return rc; }
	if (n_int16 > 0) {
		RXB_CUDA(cudaSetDevice(r->device));
		// samples per group: 4 g bytes in and at most 4 (g L / N + 1) out within the scratch bytes
		const size_t c = n_int16 / 2, words = RXB200_RESAMPLE_SCRATCH_BYTES / 4 - 1;
		const size_t g = std::max<size_t>(1, (size_t)((u128)words * (u128)r->N / (u128)(r->N + r->L)));
		const size_t gn = (size_t)(((u128)g * (u128)r->L + (u128)(r->N - 1)) / (u128)r->N) + 1;
		RXB_CUDA(reserve(r->d_cap, r->cap_cap, 2 * std::min(g, c)));
		RXB_CUDA(reserve(r->d_out, r->out_cap, 2 * std::min(gn, n + 1)));
		size_t done = 0;                                           // outputs written so far
		for (size_t s = 0; s < c; s += g) {
			const size_t cg = std::min(g, c - s), ng = out_count(r->pos, cg, r->L, r->N);
			RXB_CUDA(cudaMemcpyAsync(r->d_cap, cs16 + 2 * s, cg * 2 * sizeof(int16_t), cudaMemcpyHostToDevice, r->st));
			rc = device_call(r, r->d_cap, cg, r->d_out);
			if (rc != RXB200_OK) { return rc; }
			if (ng) {
				RXB_CUDA(cudaMemcpyAsync(out + 2 * done, r->d_out, ng * 2 * sizeof(int16_t), cudaMemcpyDeviceToHost, r->st));
			}
			done += ng;
		}
		RXB_CUDA(cudaStreamSynchronize(r->st));
	}
	if (n_out) { *n_out = n; }
	return RXB200_OK;
}

extern "C" void *rxb200_resample_stream(rxb200_resample *r) { return r ? (void *)r->st : nullptr; }

extern "C" int rxb200_resample_kernel_ms(rxb200_resample *r, float *ms)
{
	if (!r || !ms) { set_error("null argument"); return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(r->device));
	RXB_CUDA(cudaEventSynchronize(r->ev1));
	RXB_CUDA(cudaEventElapsedTime(ms, r->ev0, r->ev1));
	return RXB200_OK;
}

extern "C" int rxb200_resample_device(const rxb200_resampler *rs, unsigned long long n0, const int16_t *d_src,
                                      size_t n_complex, int16_t *d_dst, void *stream)
{
	bool wide = false;
	const int rc = resample_check(rs, &wide);
	if (rc != RXB200_OK) { return rc; }
	if (!d_src || !d_dst || ((uintptr_t)d_src & 3u) || ((uintptr_t)d_dst & 3u)) {
		set_error("d_src and d_dst must be non-NULL and 4-byte aligned");
		return RXB200_EINVAL;
	}
	if (out_count(n0, n_complex, rs->up, rs->down) == 0) { return RXB200_OK; }
	cudaStream_t st = static_cast<cudaStream_t>(stream);
	// one block: the phase-major taps, then a zero history of J - 1 samples (at least one word)
	const std::vector<int32_t> pm = phase_major(rs);
	const size_t tb = pm.size() * sizeof(int32_t), hb = (size_t)std::max(1, rs->taps_per_phase - 1) * sizeof(uint32_t);
	std::vector<unsigned char> h(tb + hb, 0);
	memcpy(h.data(), pm.data(), tb);
	unsigned char *d = nullptr;
	RXB_CUDA(cudaMallocAsync((void **)&d, h.size(), st));
	// from pageable memory: the copy has read its source when it returns
	if (cudaMemcpyAsync(d, h.data(), h.size(), cudaMemcpyHostToDevice, st) != cudaSuccess) {
		set_error("resampler upload failed: %s", cudaGetErrorString(cudaGetLastError()));
		cudaFreeAsync(d, st);
		return RXB200_ECUDA;
	}
	const int lc = resample_launch(rs->up, rs->down, rs->taps_per_phase, rs->shift, wide,
	                               reinterpret_cast<const int32_t *>(d), reinterpret_cast<const uint32_t *>(d_src),
	                               reinterpret_cast<const uint32_t *>(d + tb), n0, n_complex,
	                               reinterpret_cast<uint32_t *>(d_dst), st);
	RXB_CUDA(cudaFreeAsync(d, st));
	return lc;
}
