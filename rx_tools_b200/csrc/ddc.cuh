// ddc.cuh — the digital down-converter the mixing handles run: fm_ddc_kernel (fm_mix.cu: rx_fm channels, each mixed
// with its integer table) and power_ddc_kernel (power_mix.cu: rx_power hops, each mixed with a phase-accumulator NCO).
// Both kernels are ddc_body with their mixer policy: it stages the capture samples its outputs' windows cover, mixes
// them per channel into shared memory with mix_one, and runs the T-tap dot product at the emission points only; the
// policy supplies the mixer index and the output address, the two things they differ in.  fine_ddc_kernel
// (fm_two_stage.cu) is ddc_body too, with an NCO mixer and the staging hook ddc_row giving each grid row its own
// stream.  sdr_nco_kernel (sdr_mix.cu) is ddc_body with the NCO mixer and the output hook ddc_store writing an rx_sdr
// format (SdrOut), and fine_ddc_kernel has such instances too.  The host side they share is here too (the launch, the
// filter state a handle carries between calls, the NCO bank) and in ddc.cu (the argument check, the stateless entries'
// upload).  The front stage a handle runs on one capture, of whichever kind, is capture_front.cuh's.
#pragma once
#include <algorithm>
#include <vector>
#include "common.cuh"
#include "sdr_cvt.cuh"

namespace rxb {

#define MIX_GROUP 256                // channels per grid row (blockIdx.y): the capture is read once per group
#define DDC_THREADS 256
#define DDC_SPAN 8192                // capture samples a CTA stages at most (T <= 8192: one output always fits)
#define DDC_REACH (1 << 20)          // capture samples a CTA's span covers at most: table offsets stay below 2^21

// one complex sample through the mixer: (I + jQ)(c + js) in Q15, rounded, arithmetic shift, int16 wrap
__device__ __forceinline__ uint32_t mix_one(uint32_t w, int2 cs)
{
	const int I = (int)(int16_t)(w & 0xffffu), Q = (int)(int16_t)(w >> 16);
	const int i2 = (I * cs.x - Q * cs.y + 16384) >> 15;      // |x| |(c, s)| sqrt(2) < 2^31: no overflow
	const int q2 = (I * cs.y + Q * cs.x + 16384) >> 15;
	return ((uint32_t)i2 & 0xffffu) | ((uint32_t)q2 << 16);
}

// The arguments of one DDC launch: the fields every DDC takes, then the mixer policy's own (Mix).
template <typename Mix>
struct DdcArgs {
	const uint32_t *src;             // the call's capture, one word per complex sample
	const uint32_t *hist;            // the T - 1 raw capture samples before src
	long long n_out;                 // outputs per channel
	long long r0;                    // src index of the first emission point
	unsigned long long pos;          // the mixer's position (capture sample index) of src[0]
	uint32_t *dst;                   // one word per output, at the address Mix gives
	const int32_t *taps;             // reversed: taps[t] = h[T - 1 - t]
	int n_ch, M, T, S;
	int ws;                          // staged samples between two outputs' windows: M when T >= M, else T
	unsigned ws_m;                   // floor((2^32 - 1) / ws)
	int U;                           // outputs per CTA
	int lpo;                         // lanes per output (a power of two <= 32)
	Mix mix;
};

// staged sample s -> its offset from the CTA's first staged sample: windows of T samples, M apart, stored ws apart
template <typename Args>
__device__ __forceinline__ int ddc_off(int s, const Args &a)
{
	unsigned q = __umulhi((unsigned)s, a.ws_m);
	int r = s - (int)q * a.ws;
	if (r >= a.ws) { q++; r -= a.ws; }
	return (int)q * a.M + r;
}

// one output: y = S == 0 ? A : (A + 2^(S-1)) >> S (arithmetic), saturated to int16
template <typename Acc>
__device__ __forceinline__ int ddc_out(Acc acc, int S)
{
	long long y = (long long)acc;
	if (S) { y = (y + (1ll << (S - 1))) >> S; }
	return (int)(y < -32768 ? -32768 : (y > 32767 ? 32767 : y));
}

// The staging hook: grid row blockIdx.y's channels [c0, c0 + nc) in the policy's order, and the stream it stages (src,
// with the T - 1 samples before src[0] at hist).  By default every grid row stages the one capture and holds channels
// [y MIX_GROUP, y MIX_GROUP + MIX_GROUP); a policy whose grid rows read different streams specialises it.
struct DdcRow {
	int c0, nc;
	const uint32_t *src, *hist;
};
template <typename Mix>
__device__ __forceinline__ DdcRow ddc_row(const DdcArgs<Mix> &a)
{
	const int c0 = (int)blockIdx.y * MIX_GROUP;
	return DdcRow{c0, min(MIX_GROUP, a.n_ch - c0), a.src, a.hist};
}

// The output hook: the store of the current channel's call output u, w its int16 pair (I low, Q high).  By default w
// goes to the word row.out(u); a policy that writes another format overloads it (SdrOut below).
template <typename Mix, typename Row>
__device__ __forceinline__ void ddc_store(const DdcArgs<Mix> &, const Row &row, int u, uint32_t w)
{
	*row.out(u) = w;
}

// One CTA: U consecutive outputs of every channel of its grid row (up to 256 channels, blockIdx.y).  It stages the
// capture samples its outputs' windows cover once (the history before the call's first sample), then per channel mixes
// them into shared memory and runs the T-tap dot product at the emission points only, lpo lanes per output.  Acc: int
// when sum |h| * 32768 + 2^(S-1) < 2^31, else long long (no partial sum can overflow either way).  The mixer policy:
//   typename Mix::Row row(a, c0, nc, u0, g0)   the grid row's set-up, g0 the first staged sample's mixer position
//   row.chan(c)                                 takes channel c's mixer state
//   row.entry(off)                              the channel's table entry for the staged sample at offset off
//   row.out(u)                                  the address of the channel's call output u (ddc_store writes it)
template <typename Acc, typename Mix>
__device__ __forceinline__ void ddc_body(const DdcArgs<Mix> &a)
{
	extern __shared__ int4 ddc_smem[];
	const int T = a.T;
	const int room = (a.U - 1) * a.ws + T;
	int32_t *s_h = reinterpret_cast<int32_t *>(ddc_smem);
	uint32_t *s_x = reinterpret_cast<uint32_t *>(s_h + T);
	uint32_t *s_z = s_x + room;
	const DdcRow g = ddc_row(a);
	const int c0 = g.c0, nc = g.nc;
	const long long u0 = (long long)blockIdx.x * a.U;
	const int U = (int)min((long long)a.U, a.n_out - u0);
	const int n = (U - 1) * a.ws + T;
	const long long b0 = u0 * a.M + a.r0 - (T - 1);       // src index of the first staged sample, >= -(T - 1)
	const long long g0 = (long long)a.pos + b0;            // its mixer position
	for (int j = threadIdx.x; j < T; j += blockDim.x) { s_h[j] = a.taps[j]; }
	typename Mix::Row row(a, c0, nc, u0, g0);
	for (int s = threadIdx.x; s < n; s += blockDim.x) {
		const long long i = b0 + ddc_off(s, a);
		s_x[s] = i >= 0 ? __ldg(g.src + i) : g.hist[(T - 1) + i];
	}
	__syncthreads();
	const int lane = (int)threadIdx.x & (a.lpo - 1), sub = (int)threadIdx.x / a.lpo, n_sub = (int)blockDim.x / a.lpo;
	for (int c = 0; c < nc; c++) {
		row.chan(c);
		for (int s = threadIdx.x; s < n; s += blockDim.x) {
			const int2 *e = row.entry(ddc_off(s, a));
			s_z[s] = mix_one(s_x[s], __ldg(e));
		}
		__syncthreads();
		for (int ub = 0; ub < U; ub += n_sub) {                  // the same trip count on every lane of a warp
			const int u = ub + sub;
			Acc ai = 0, aq = 0;
			if (u < U) {
				const uint32_t *z = s_z + u * a.ws;
				for (int j = lane; j < T; j += a.lpo) {
					const uint32_t w = z[j];
					const Acc h = (Acc)s_h[j];
					ai += h * (Acc)(int16_t)(w & 0xffffu);
					aq += h * (Acc)(int16_t)(w >> 16);
				}
			}
			for (int o = a.lpo >> 1; o > 0; o >>= 1) {
				ai += __shfl_xor_sync(0xffffffffu, ai, o);
				aq += __shfl_xor_sync(0xffffffffu, aq, o);
			}
			if (u < U && lane == 0) {
				ddc_store(a, row, u, ((uint32_t)ddc_out(ai, a.S) & 0xffffu) | ((uint32_t)ddc_out(aq, a.S) << 16));
			}
		}
		__syncthreads();                    // every output of this channel is made before s_z is overwritten
	}
}

// A mixer policy Base whose outputs are written in rx_sdr format F (RXB200_SDR_OUT_CS16 or a RXB200_CVT_CS16_* kind)
// instead of as int16 pair words: Base's row.out(u) names the output's complex element, counted in elements from
// a.dst, and the store converts the word there (sdr_put).  Base's Row is its RowOf template on these arguments.
template <typename Base, int F>
struct SdrOut : Base {
	using Row = typename Base::template RowOf<DdcArgs<SdrOut>>;
};
template <typename Base, int F, typename Row>
__device__ __forceinline__ void ddc_store(const DdcArgs<SdrOut<Base, F>> &a, const Row &row, int u, uint32_t w)
{
	sdr_put<F>(a.dst, row.out(u) - a.dst, w);
}

// the arguments b with the mixer policy Mix, built from b's (a base of Mix), for a launch of another instance
template <typename Mix, typename Base>
DdcArgs<Mix> ddc_args_as(const DdcArgs<Base> &b)
{
	DdcArgs<Mix> a{};
	a.src = b.src; a.hist = b.hist; a.n_out = b.n_out; a.r0 = b.r0; a.pos = b.pos; a.dst = b.dst; a.taps = b.taps;
	a.n_ch = b.n_ch; a.M = b.M; a.T = b.T; a.S = b.S;
	static_cast<Base &>(a.mix) = b.mix;
	return a;
}

// ddc_body's rx_power NCO mixer policy (power_ddc_kernel, sdr_nco_kernel): channel c's capture sample n mixed by NCO
// entry ((n w_c + 2^15) mod 2^32) >> 16, the phase taken per CTA and channel as (uint32)g0 * w_c (g0 < 0 only for the
// zero samples before create or reset, which mix to zero at any phase) and stepped by off * w_c in uint32 arithmetic;
// and channel c's call output u at (u / B) * n_ch * B + c * B + u mod B, in the pass-major hop buffers of rx_power
// (with B >= n_out, one pass: channel-major rows B apart)
#define NCO_ENTRIES 65536            // the shared table: index j = ((theta + 2^15) mod 2^32) >> 16
struct NcoMix {
	const int2 *nco;                 // NCO_ENTRIES (c, s) pairs
	const uint32_t *w;               // each hop's frequency word
	int B;                           // outputs per hop buffer (buf_len / 2)
	template <typename Args>
	struct RowOf {
		const Args &a;
		int c0, c;
		uint32_t g0, w, th0;             // hop c's word and its phase at the CTA's first staged sample
		long long q0, pass_words;        // the pass of the CTA's first output, and the words of one pass
		int rb;                          // the first output's place in its pass
		__device__ RowOf(const Args &a, int c0, int, long long u0, long long g0)
		    : a(a), c0(c0), g0((uint32_t)(unsigned long long)g0), q0(u0 / a.mix.B), pass_words((long long)a.n_ch * a.mix.B),
		      rb((int)(u0 - q0 * a.mix.B)) {}
		__device__ void chan(int k) { c = k; w = __ldg(a.mix.w + c0 + k); th0 = g0 * w; }
		__device__ const int2 *entry(int off) const { return a.mix.nco + ((th0 + (uint32_t)off * w + 32768u) >> 16); }
		__device__ uint32_t *out(int u) const
		{
			const int r = rb + u, q = r / a.mix.B;               // rb + u < B + DDC_SPAN
			return a.dst + q0 * pass_words + (long long)(c0 + c) * a.mix.B + (q * pass_words + (r - q * a.mix.B));
		}
	};
	using Row = RowOf<DdcArgs<NcoMix>>;
};

// NcoMix's device data on the current device: the shared table (rxb200_nco_table) and each channel's word
struct NcoBank {
	int2 *nco = nullptr;
	uint32_t *w = nullptr;
	int upload(const std::vector<uint32_t> &words);   // the caller releases the bank when it fails
	void release() { cudaFree(w); cudaFree(nco); }
};

// w = floor((f 2^32 + floor(R/2)) / R) mod 2^32 for each of the n offsets, exactly, with the refusals of R <= 0 and
// |f| >= R/2 (power_mix.cu)
int nco_words(int capture_rate, const int *offsets_hz, int n, std::vector<uint32_t> &w);

// Launches kern (a DDC kernel) on the current device for a.n_out > 0 outputs per channel, with its launch shape: a.ws,
// a.ws_m, a.lpo, and as many outputs per CTA (a.U) as the staging room and the reach allow, but at least two CTAs per
// SM when there is work.  The dynamic shared memory holds the reversed taps, the staged and the mixed span.  rows: the
// grid rows of a policy that specialises ddc_row (0: one per MIX_GROUP channels).
template <typename Mix>
int ddc_launch(DdcArgs<Mix> a, void (*kern)(DdcArgs<Mix>), cudaStream_t st, int rows = 0)
{
	const int groups = rows ? rows : (a.n_ch + MIX_GROUP - 1) / MIX_GROUP;
	a.ws = a.T >= a.M ? a.M : a.T;
	a.ws_m = 0xffffffffu / (unsigned)a.ws;
	a.lpo = 1;
	while (a.lpo < 32 && a.lpo < a.T) { a.lpo <<= 1; }
	int dev = 0, n_sm = 0;
	RXB_CUDA(cudaGetDevice(&dev));
	RXB_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
	long long U = std::min((long long)(DDC_SPAN - a.T) / a.ws, (long long)(DDC_REACH - a.T) / a.M) + 1;
	const long long ctas = std::max(1ll, (2ll * n_sm + groups - 1) / groups);
	U = std::max(1ll, std::min(U, (a.n_out + ctas - 1) / ctas));
	a.U = (int)U;
	const size_t smem = ((size_t)a.T + 2 * ((size_t)(a.U - 1) * a.ws + a.T)) * sizeof(uint32_t);
	const long long bx = (a.n_out + U - 1) / U;
	RXB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
	kern<<<dim3((unsigned)bx, (unsigned)groups), DDC_THREADS, smem, st>>>(a);
	RXB_CUDA(cudaGetLastError());
	return RXB200_OK;
}

// The filter state a mixing handle carries between calls (the rule of include/rxb200.h's rxb200_ddc): M, T and S, the
// reversed taps, and the raw capture's last T - 1 samples before the handle's position (zero before create or reset,
// which is exactly the rule's z = 0 before sample 0, since a zero sample mixes to zero) in two device buffers.  A
// handle's kernels read hist[cur]; carry then writes the next history into the other buffer behind them on the same
// stream, and commit makes it live.  Each handle commits once no later launch of the call reads the old history:
// rx_fm once at the end of a successful call, after the member's call, so a failed call leaves the old history live;
// rx_power after each group's launch, since the next group of passes reads the new history.
struct DdcFilter {
	int M = 1, T = 1, S = 0;             // T = 1 (a plain rx_fm mixing handle): no history, carry and commit do nothing
	bool wide = false;                   // the kernel accumulates in 64 bits
	int32_t *taps = nullptr;
	uint32_t *hist[2] = {nullptr, nullptr};
	int cur = 0;
	// the buffers hold at least one sample, so that T = 1 needs no special case
	size_t hist_bytes() const { return std::max<size_t>(1, (size_t)T - 1) * sizeof(uint32_t); }
	// on the current device, for a checked ddc; the caller releases the filter when it fails
	int create(const rxb200_ddc *ddc, bool w)
	{
		M = ddc->decim; T = ddc->n_taps; S = ddc->shift; wide = w;
		std::vector<int32_t> rev(ddc->taps, ddc->taps + T);
		std::reverse(rev.begin(), rev.end());
		RXB_CUDA(cudaMalloc(&taps, (size_t)T * sizeof(int32_t)));
		RXB_CUDA(cudaMemcpy(taps, rev.data(), (size_t)T * sizeof(int32_t), cudaMemcpyHostToDevice));
		return alloc_hist();
	}
	// the two zeroed histories of T - 1 samples (create; the resampler, whose taps are its own, sets T and calls it)
	int alloc_hist()
	{
		for (int i = 0; i < 2; i++) {
			RXB_CUDA(cudaMalloc(&hist[i], hist_bytes()));
			RXB_CUDA(cudaMemset(hist[i], 0, hist_bytes()));
		}
		return RXB200_OK;
	}
	// the last T - 1 samples of (hist[cur], the c capture samples at src), into hist[cur ^ 1]
	int carry(const uint32_t *src, size_t c, cudaStream_t st) const
	{
		const size_t H = (size_t)T - 1, w = sizeof(uint32_t);
		if (H == 0) { return RXB200_OK; }
		if (c >= H) {
			RXB_CUDA(cudaMemcpyAsync(hist[cur ^ 1], src + (c - H), H * w, cudaMemcpyDeviceToDevice, st));
		} else {
			RXB_CUDA(cudaMemcpyAsync(hist[cur ^ 1], hist[cur] + c, (H - c) * w, cudaMemcpyDeviceToDevice, st));
			RXB_CUDA(cudaMemcpyAsync(hist[cur ^ 1] + (H - c), src, c * w, cudaMemcpyDeviceToDevice, st));
		}
		return RXB200_OK;
	}
	void commit() { if (T > 1) { cur ^= 1; } }
	// both histories zeroed behind any call still running on st, on the current device
	int reset(cudaStream_t st)
	{
		RXB_CUDA(cudaMemsetAsync(hist[0], 0, hist_bytes(), st));
		RXB_CUDA(cudaMemsetAsync(hist[1], 0, hist_bytes(), st));
		cur = 0;
		return RXB200_OK;
	}
	void release() { cudaFree(taps); cudaFree(hist[0]); cudaFree(hist[1]); }
};

// The device block of a stateless call: the mixer data at the front of h (a multiple of 16 bytes), then for a DDC the
// reversed taps and a zero history, uploaded with one allocation and one copy on st.  The caller frees d with
// cudaFreeAsync on st behind its launch.
struct DdcBlock {
	unsigned char *d = nullptr;
	const int32_t *taps = nullptr;
	const uint32_t *hist = nullptr;
};
int ddc_upload(std::vector<unsigned char> &h, const rxb200_ddc *ddc, cudaStream_t st, DdcBlock *b);

}  // namespace rxb
