// power_kernels.cu — rx_power hot path on sm_90a: scanner()'s per-hop body
// (src/rtl_power.c:709-771) batched over (hop, pass) work items.
//
//   copy (:715-720) -> remove_dc x2 (:609-624, :744-745) -> per N-point block:
//   window multiply with int16 wrap (:749-758) -> fix_fft (:264-320) -> real_conj accumulate
//   (:664-668, :760-768);  rms_power (:403-429) when bin_e == 0.
//
// One CTA owns a hop and a slice of that hop's passes.  Each hop buffer (buf_len int16, 32 KiB in
// the BASELINE configs) is staged HBM -> shared memory by ONE bulk-TMA copy (cp.async.bulk +
// mbarrier), transformed in place in shared memory, and only the |X|^2 sums leave the SM: they are
// accumulated in registers across the CTA's passes and flushed with one 64-bit atomic per bin per
// CTA (integer sums / max are order independent, so the result is bit-exact).  Algorithmic HBM
// traffic: 4 B per used complex sample.  The FFT is the reference's radix-2 DIT with its per-stage
// halving and FIX_MPY rounding reproduced exactly — this is integer-issue bound, not HBM bound
// (DESIGN.md "rx_power kernel"); tensor cores do not apply (per-stage rounding).
#include <math.h>
#include <string.h>
#include <new>
#include <vector>
#include "common.cuh"
#include "nccl_dyn.h"

namespace rxb {

struct PowArgs {
	const int16_t *bufs;     // [n_pass][n_hops_call][buf_len]
	long long *avg;          // [n_hops_total][N]
	const int16_t *sine;     // 3N/4
	const int16_t *window;   // N (low 16 bits of window_coefs; exact, see below)
	int n_pass, n_hops_call, hop_begin;
	int buf_len, bin_e, slices, peak_hold;
	int ds, ds_passes, boxcar, fir_on;   // small-span decimators (src/rtl_power.c:721-743)
	int fir[6];                          // cic_9_tables[ds_passes][0..5]
	int tables_in_smem;                  // 0: sine/window stay in global memory (very large N)
	int triv;                            // Sinewave[0] == 0 and Sinewave[N/2] in {0, 1}: W^0 and W^(N/4) have a zero component
};

__device__ __forceinline__ int plo(uint32_t w) { return (int)(int16_t)(w & 0xffffu); }
__device__ __forceinline__ int phi(uint32_t w) { return (int)(int16_t)(w >> 16); }
__device__ __forceinline__ uint32_t ppack(int re, int im) { return ((uint32_t)re & 0xffffu) | ((uint32_t)im << 16); }

// FIX_MPY (src/rtl_power.c:256-262): c = (a*b)>>14; (c>>1)+(c&1)  ==  (a*b + 2^14) >> 15.
// The int16 truncation of its result and of tr/ti is deferred to the final pack: everything in
// between is addition modulo 2^16.
__device__ __forceinline__ int q15(int a, int b)
{
	return (a * b + 16384) >> 15;     // (a mulhi-by-2^17 form on the multiplier pipe instead of the shifter measured slower)
}

// wi = -Sinewave[j] >> 1 (src/rtl_power.c:298-301): the negation is stored in an int16 before the shift, so -(-32768)
// stays -32768.  Only a caller's table can hold -32768 (sine_table's entries are round(32767 sin)).
__device__ __forceinline__ int neg_half(int s) { return (int)(int16_t)(-s) >> 1; }

__device__ __forceinline__ long long block_sum(long long v, long long *red, int tid, int nthreads)
{
	for (int o = 16; o > 0; o >>= 1) { v += __shfl_down_sync(0xffffffffu, v, o); }
	__syncthreads();
	if ((tid & 31) == 0) { red[tid >> 5] = v; }
	__syncthreads();
	long long t = 0;
	for (int w = 0; w < (nthreads >> 5); w++) { t += red[w]; }
	return t;
}

// ---- the reference's steps, one sample, bin or butterfly at a time.  The shared-memory kernel below and the
// global-memory kernels of large hop buffers both call these; a buffer is packed I/Q words in either memory.

// one component (sel 0 = I, 1 = Q) of sample i
__device__ __forceinline__ int pw_get(const uint32_t *buf, int i, int sel) { return sel ? phi(buf[i]) : plo(buf[i]); }
__device__ __forceinline__ void pw_put(uint32_t *buf, int i, int sel, int v)
{
	uint16_t *h = reinterpret_cast<uint16_t *>(buf + i);
	h[sel] = (uint16_t)v;
}

// boxcar slot k (src/rtl_power.c:723-733): the int16-wrapped sums of samples [k*ds, (k+1)*ds) of the first n
__device__ __forceinline__ uint32_t boxcar_slot(const uint32_t *x, int k, int ds, int n)
{
	const int e = (k + 1) * ds < n ? (k + 1) * ds : n;
	int si = 0, sq = 0;
	for (int i = k * ds; i < e; i++) { const uint32_t w = x[i]; si += plo(w); sq += phi(w); }
	return ppack(si, sq);
}

__device__ __forceinline__ int hb_taps(int a, int b, int c, int d, int e, int f) { return (a + (b + e) * 5 + (c + d) * 10 + f) >> 4; }

// fifth_order output k with its "ease-in" head (src/rtl_power.c:582-607) of one component from the level window x,
// which starts at level index lo
__device__ __forceinline__ int hb_out(const uint32_t *x, int lo, int k, int sel)
{
	const uint32_t *w = x - lo;             // w[i] = level sample i
	if (k < 3) {
		const int a = pw_get(w, 0, sel), b = pw_get(w, 1, sel), c = pw_get(w, 2, sel);
		const int d = pw_get(w, 3, sel), e = pw_get(w, 4, sel), f = pw_get(w, 5, sel);
		if (k == 0) { return ((a + b) * 10 + (c + d) * 5 + d + f) >> 4; }
		if (k == 1) { return ((b + c) * 10 + (a + d) * 5 + e + f) >> 4; }
		return hb_taps(a, b, c, d, e, f);
	}
	if (k == 3) { return hb_taps(pw_get(w, 2, sel), pw_get(w, 3, sel), pw_get(w, 4, sel), pw_get(w, 5, sel), pw_get(w, 5, sel), pw_get(w, 6, sel)); }
	if (k == 4) { return hb_taps(pw_get(w, 4, sel), pw_get(w, 5, sel), pw_get(w, 5, sel), pw_get(w, 6, sel), pw_get(w, 7, sel), pw_get(w, 8, sel)); }
	const int i = 2 * k - 5;
	return hb_taps(pw_get(w, i, sel), pw_get(w, i + 1, sel), pw_get(w, i + 2, sel), pw_get(w, i + 3, sel), pw_get(w, i + 4, sel), pw_get(w, i + 5, sel));
}

// generic_fir (src/rtl_power.c:626-654) output d >= 9 of one component: the 9-tap sum over ORIGINAL samples
// d-9 .. d-1 of the window x, which starts at index lo
__device__ __forceinline__ int fir_out(const uint32_t *x, int lo, int d, int sel, const int *c)
{
	const uint32_t *w = x - lo;
	int acc = mul_w(pw_get(w, d - 9, sel) + pw_get(w, d - 1, sel), c[1]);
	acc = add_w(acc, mul_w(pw_get(w, d - 8, sel) + pw_get(w, d - 2, sel), c[2]));
	acc = add_w(acc, mul_w(pw_get(w, d - 7, sel) + pw_get(w, d - 3, sel), c[3]));
	acc = add_w(acc, mul_w(pw_get(w, d - 6, sel) + pw_get(w, d - 4, sel), c[4]));
	acc = add_w(acc, mul_w(pw_get(w, d - 5, sel), c[5]));
	return acc >> 15;
}

// remove_dc (src/rtl_power.c:609-624, :744-745) over the first `used` int16: I is summed over samples < n_i and
// divided by used, Q over samples < n_q and divided by used - 1
struct Dc { int n_i, n_q, ave_i, ave_q; };
__device__ __forceinline__ Dc dc_average(long long si, long long sq, int used)
{
	return {(used + 1) / 2, used / 2, (int)(int16_t)(si / (long long)used), (int)(int16_t)(sq / (long long)(used - 1))};
}

// window multiply of sample g (word u) with int16 wrap (:749-758)
__device__ __forceinline__ uint32_t dc_window(uint32_t u, int g, const Dc &dc, int w)
{
	return ppack((plo(u) - (g < dc.n_i ? dc.ave_i : 0)) * w, (phi(u) - (g < dc.n_q ? dc.ave_q : 0)) * w);
}

// butterfly t of radix-2 DIT stage s on the N-block x, every stage halves (:291-318)
__device__ __forceinline__ void dit_bfly(uint32_t *x, int t, int s, int bin_e, const int16_t *sine)
{
	const int N = 1 << bin_e;
	const int l = 1 << s, k = bin_e - 1 - s;
	const int m = t & (l - 1);
	const int i = ((t >> s) << (s + 1)) + m, j = i + l;
	const int jt = m << k;
	const int wr = (int)sine[jt + N / 4] >> 1;
	const int wi = neg_half(sine[jt]);
	const uint32_t u = x[i], v = x[j];
	const int vr = plo(v), vi = phi(v);
	const int tr = q15(wr, vr) - q15(wi, vi);
	const int ti = q15(wr, vi) + q15(wi, vr);
	const int qr = plo(u) >> 1, qi = phi(u) >> 1;
	x[j] = ppack(qr - tr, qi - ti);
	x[i] = ppack(qr + tr, qi + ti);
}

// real_conj (:664-668) of one bin, its sum or peak hold (:760-768), and the flush of a partial result to avg
__device__ __forceinline__ long long bin_power(uint32_t w)
{
	const int re = plo(w), im = phi(w);
	return (long long)(re * re) + (long long)(im * im);
}
__device__ __forceinline__ void fold(long long &acc, long long v, int peak_hold) { if (peak_hold) { acc = v > acc ? v : acc; } else { acc += v; } }
__device__ __forceinline__ void flush(long long *dst, long long v, int peak_hold)
{
	if (peak_hold) { atomicMax(dst, v); } else { atomicAdd(reinterpret_cast<unsigned long long *>(dst), (unsigned long long)v); }
}

// ---- small-span decimators, in place on the shared hop buffer (rare path: only when the planner
// chose downsample > 1).  Every output depends only on ORIGINAL samples at higher (or equal) positions
// than where it is stored, so each is done in rounds of "all threads read, barrier, all threads write".

// boxcar: slot k replaces sample k; the sources are zeroed, so everything past the last slot is zero.
__device__ void pw_boxcar(uint32_t *buf, int ncomplex, int ds, int tid, int T)
{
	const int nslots = (ncomplex + ds - 1) / ds;
	for (int base = 0; base < nslots; base += T) {
		const int k = base + tid;
		const uint32_t y = k < nslots ? boxcar_slot(buf, k, ds, ncomplex) : 0u;
		__syncthreads();
		if (k < nslots) { buf[k] = y; }
		__syncthreads();
	}
	for (int i = nslots + tid; i < ncomplex; i += T) { buf[i] = 0u; }
	__syncthreads();
}

// stateless fifth_order on one component.  `length` is the reference's argument (an int16 span); outputs
// k = 0 .. while 4k < length.
__device__ void pw_halfband(uint32_t *buf, int length, int sel, int tid, int T)
{
	const int nout = (length + 3) / 4 > 3 ? (length + 3) / 4 : 3;
	for (int base = 0; base < nout; base += T) {
		const int k = base + tid;
		const int y = k < nout ? hb_out(buf, 0, k, sel) : 0;
		__syncthreads();
		if (k < nout) { pw_put(buf, k, sel, y); }
		__syncthreads();
	}
}

// stateless generic_fir on one component: samples 0..8 pass through.  Done from the top down so that a round's
// stores never touch what a later round still has to read.
__device__ void pw_droop9(uint32_t *buf, int length, int sel, const int *c, int tid, int T)
{
	const int ncomp = (length + 1) / 2;           // samples d with 2d < length
	if (ncomp <= 9) { return; }
	const int nfil = ncomp - 9;
	for (int top = nfil; top > 0; top -= T) {
		const int j = top - 1 - tid;              // filtered index within [0, nfil)
		const int y = j >= 0 ? fir_out(buf, 0, j + 9, sel, c) : 0;
		__syncthreads();
		if (j >= 0) { pw_put(buf, j + 9, sel, y); }
		__syncthreads();
	}
}

// NB = bins accumulated in registers per thread (N / blockDim); NB == 0: N too large, accumulate
// straight into global memory after every block.
template <int NB>
__global__ void __launch_bounds__(256) power_fft_kernel(const PowArgs a)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	const int tid = threadIdx.x, T = blockDim.x;
	const int N = 1 << a.bin_e;
	uint64_t *bar = reinterpret_cast<uint64_t *>(smem_raw);
	long long *red = reinterpret_cast<long long *>(smem_raw + 16);            // 32 x 8 B
	uint32_t *buf = reinterpret_cast<uint32_t *>(smem_raw + 16 + 256);        // buf_len/2 words
	int16_t *sine_s = reinterpret_cast<int16_t *>(buf + a.buf_len / 2);       // 3N/4
	int16_t *win_s = sine_s + ((N * 3 / 4 + 7) & ~7);                         // N
	const int hop_local = blockIdx.x / a.slices;
	const int slice = blockIdx.x % a.slices;
	const int hop = a.hop_begin + hop_local;
	const int16_t *sine = a.sine, *win = a.window;
	if (a.tables_in_smem) {
		for (int i = tid; i < N * 3 / 4; i += T) { sine_s[i] = a.sine[i]; }
		for (int i = tid; i < N; i += T) { win_s[i] = a.window[i]; }
		sine = sine_s; win = win_s;
	}
	if (tid == 0) { mbar_init(bar, 1); }
	__syncthreads();

	long long acc[NB > 0 ? NB : 1];
#pragma unroll
	for (int b = 0; b < (NB > 0 ? NB : 1); b++) { acc[b] = 0; }

	const int used = a.buf_len / a.ds;          // int16 span after decimation (src/rtl_power.c:744-747)
	const int nblk = (used + 2 * N - 1) / (2 * N);
	const int n_i = (used + 1) / 2, n_q = used / 2;   // samples remove_dc touches per component
	uint32_t parity = 0;
	for (int pass = slice; pass < a.n_pass; pass += a.slices) {
		const int16_t *src = a.bufs + ((size_t)pass * a.n_hops_call + hop_local) * (size_t)a.buf_len;
		if (tid == 0) {
			fence_async_smem();                  // earlier generic-proxy writes to buf are ordered before the TMA write
			mbar_expect_tx(bar, (uint32_t)a.buf_len * 2u);
			bulk_load(buf, src, (uint32_t)a.buf_len * 2u, bar);
		}
		mbar_wait(bar, parity);
		parity ^= 1u;
		if (a.ds > 1) {
			__syncthreads();
			if (a.boxcar) { pw_boxcar(buf, a.buf_len / 2, a.ds, tid, T); }
			else if (a.ds_passes) {
				for (int dp = 0; dp < a.ds_passes; dp++) {       // downsample_iq (:656-662)
					pw_halfband(buf, a.buf_len >> dp, 0, tid, T);
					pw_halfband(buf, (a.buf_len >> dp) - 1, 1, tid, T);
				}
				if (a.fir_on) {
					pw_droop9(buf, a.buf_len >> a.ds_passes, 0, a.fir, tid, T);
					pw_droop9(buf, (a.buf_len >> a.ds_passes) - 1, 1, a.fir, tid, T);
				}
			}
		}
		long long si = 0, sq = 0;
		for (int i = tid; i < n_i; i += T) { uint32_t w = buf[i]; si += plo(w); if (i < n_q) { sq += phi(w); } }
		const Dc dc = dc_average(block_sum(si, red, tid, T), block_sum(sq, red, tid, T), used);
		for (int blk = 0; blk < nblk; blk++) {
			uint32_t *x = buf + (size_t)blk * N;
			// window multiply fused with the bit-reversal swap (:275-290)
			for (int i = tid; i < N; i += T) {
				const int r = (int)(__brev((unsigned)i) >> (32 - a.bin_e));
				if (i <= r) {
					const uint32_t u = dc_window(x[i], blk * N + i, dc, win[i]), v = dc_window(x[r], blk * N + r, dc, win[r]);
					x[r] = u;
					x[i] = v;
				}
			}
			__syncthreads();
			for (int s = 0; s < a.bin_e; s++) {
				for (int t = tid; t < N / 2; t += T) { dit_bfly(x, t, s, a.bin_e, sine); }
				__syncthreads();
			}
			if (NB > 0) {
#pragma unroll
				for (int b = 0; b < (NB > 0 ? NB : 1); b++) {
					const int j = tid + b * T;
					if (j < N) { fold(acc[b], bin_power(x[j]), a.peak_hold); }
				}
			} else {
				long long *row = a.avg + (size_t)hop * N;
				for (int j = tid; j < N; j += T) { flush(row + j, bin_power(x[j]), a.peak_hold); }
			}
		}
		__syncthreads();       // everyone done with buf before the next TMA overwrites it
	}
	if (NB > 0) {
		long long *row = a.avg + (size_t)hop * N;
#pragma unroll
		for (int b = 0; b < (NB > 0 ? NB : 1); b++) {
			const int j = tid + b * T;
			if (j < N) { flush(row + j, acc[b], a.peak_hold); }
		}
	}
}

// ---------------------------------------------------------------------------------------------
// power_fft8_kernel<E>: the fast path for the BASELINE shapes (hop buffer = 16384 int16, N = 2^E,
// 3 <= E <= 13, no decimation).  1024 threads own one hop buffer; every thread keeps EIGHT points
// of one N-block in registers and runs three fix_fft stages per trip through shared memory.
//
// The reference bit-reverses first and then pairs positions p, p + 2^s in stage s
// (src/rtl_power.c:275-318).  Position p holds input n = rev(p), so the same butterfly graph in
// NATURAL input order pairs slots n, n + N/2^(s+1) (the slot whose bit is 0 is the reference's
// "i", the other its "j = i + l"), with twiddle index m = (p mod 2^s) = the top s bits of n,
// reversed.  Running the graph in natural order needs no permutation pass: after the last stage
// slot n simply holds bin rev(n), which only matters when the per-thread accumulators are flushed.
// Every butterfly is the reference's, bit for bit: wr = Sinewave[j + N/4] >> 1, wi = -Sinewave[j] >> 1,
// FIX_MPY(a,b) = (a*b + 2^14) >> 15, the halving of the "i" input and the int16 wrap of all four
// results.
// Shared-memory layout between trips: slot n of a block lives at n + (n / (8*Bw)) * Bw where Bw is
// the spacing of a thread's eight points in the NEXT trip, so that the 32 lanes of a warp (which
// differ in the low bits of n and in the bits above the thread's three) hit 32 different banks.
// A point is kept as a plain int whose LOW 16 bits are its int16 value; the bits above may hold the
// carry-out of the last add ("unwrapped").  The reference's int16 store is applied where the value
// is consumed: sign-extended for the multiplies of the "j" input, and folded into the halving of the
// "i" input ((s << 16) >> 17) — that keeps one shift per value off the ALU pipe, which bounds this
// kernel.
struct Cx { int re, im; };

__device__ __forceinline__ void bfly(Cx &lo, Cx &hi, int wr, int wi)
{
	// lo = reference's x[i], hi = x[j]
	const int vr = (int)(int16_t)hi.re, vi = (int)(int16_t)hi.im;
	const int tr = q15(wr, vr) - q15(wi, vi);
	const int ti = q15(wr, vi) + q15(wi, vr);
	// unsigned shift: the wrap is intended (a signed multiply would let the compiler fold it away)
	const int qr = (int)((unsigned)lo.re << 16) >> 17, qi = (int)((unsigned)lo.im << 16) >> 17;
	hi.re = qr - tr;
	hi.im = qi - ti;
	lo.re = qr + tr;
	lo.im = qi + ti;
}

// The same butterfly when the twiddle has a zero component: FIX_MPY(0, v) = (0 + 2^14) >> 15 = 0 exactly,
// so W^0 (wi == 0) and W^(N/4) (wr == 0) need two products instead of four.
__device__ __forceinline__ void bfly_w0(Cx &lo, Cx &hi, int wr)
{
	const int vr = (int)(int16_t)hi.re, vi = (int)(int16_t)hi.im;
	const int tr = q15(wr, vr), ti = q15(wr, vi);
	const int qr = (int)((unsigned)lo.re << 16) >> 17, qi = (int)((unsigned)lo.im << 16) >> 17;
	hi.re = qr - tr; hi.im = qi - ti; lo.re = qr + tr; lo.im = qi + ti;
}
__device__ __forceinline__ void bfly_wq(Cx &lo, Cx &hi, int wi)
{
	const int vr = (int)(int16_t)hi.re, vi = (int)(int16_t)hi.im;
	const int tr = -q15(wi, vi), ti = q15(wi, vr);
	const int qr = (int)((unsigned)lo.re << 16) >> 17, qi = (int)((unsigned)lo.im << 16) >> 17;
	hi.re = qr - tr; hi.im = qi - ti; lo.re = qr + tr; lo.im = qi + ti;
}

__device__ __forceinline__ void tw_unpack(uint32_t w, int &wr, int &wi) { wr = plo(w); wi = phi(w); }

// three (or, on the last trip, the last `nst`) stages on the eight points x[j], j = (j2 j1 j0)
template <int E>
__device__ __forceinline__ void trip_stages(Cx (&x)[8], const uint32_t *tw, int rA, int s0, int first)
{
	constexpr int N = 1 << E;
	int wr, wi;
	if (first <= 0) {           // stage s0: pairs (j, j+4), one twiddle
		tw_unpack(tw[rA << (E - 1 - s0)], wr, wi);
#pragma unroll
		for (int j = 0; j < 4; j++) { bfly(x[j], x[j + 4], wr, wi); }
	}
	if (first <= 1) {           // stage s0+1: pairs (j, j+2), twiddle depends on j2
#pragma unroll
		for (int j2 = 0; j2 < 2; j2++) {
			tw_unpack(tw[(rA << (E - 2 - s0)) + j2 * (N / 4)], wr, wi);
			bfly(x[4 * j2], x[4 * j2 + 2], wr, wi);
			bfly(x[4 * j2 + 1], x[4 * j2 + 3], wr, wi);
		}
	}
	{                           // stage s0+2: pairs (j, j+1), twiddle depends on j2, j1
#pragma unroll
		for (int jj = 0; jj < 4; jj++) {
			const int j2 = jj >> 1, j1 = jj & 1;
			tw_unpack(tw[(rA << (E - 3 - s0)) + j2 * (N / 8) + j1 * (N / 4)], wr, wi);
			bfly(x[2 * jj], x[2 * jj + 1], wr, wi);
		}
	}
}

// stages 0..2 (the first trip): the twiddle index depends only on the point's position j among the
// thread's eight, and ten of the twelve butterflies use W^0 or W^(N/4)
template <int E>
__device__ __forceinline__ void trip_first_triv(Cx (&x)[8], const uint32_t *tw)
{
	constexpr int N = 1 << E;
	int w0r, w0i, wqr, wqi, wr, wi;
	tw_unpack(tw[0], w0r, w0i);
	tw_unpack(tw[N / 4], wqr, wqi);
#pragma unroll
	for (int j = 0; j < 4; j++) { bfly_w0(x[j], x[j + 4], w0r); }
	bfly_w0(x[0], x[2], w0r); bfly_w0(x[1], x[3], w0r);
	bfly_wq(x[4], x[6], wqi); bfly_wq(x[5], x[7], wqi);
	bfly_w0(x[0], x[1], w0r);
	bfly_wq(x[2], x[3], wqi);
	tw_unpack(tw[N / 8], wr, wi);
	bfly(x[4], x[5], wr, wi);
	tw_unpack(tw[N / 8 + N / 4], wr, wi);
	bfly(x[6], x[7], wr, wi);
}

// T = threads per CTA.  1024: one thread per eight points of the hop buffer, one CTA per SM.  512: two CTAs per SM, each
// walking its hop buffer in two halves (upper half of the N-blocks first, see the layout note below) -- the barriers,
// the TMA wait and the DC reduction of one CTA hide behind the butterflies of the other.  A thread meets the same
// eight bins in both halves, so the accumulators are shared.
template <int E, int T>
__global__ void __launch_bounds__(T, 1024 / T) power_fft8_kernel(const PowArgs a)
{
	constexpr int N = 1 << E;
	constexpr int UPB = N / 8;                 // threads per N-block
	constexpr int NT = (E + 2) / 3;            // trips through shared memory
	constexpr int REM = E % 3;                 // stages in the last trip when not a multiple of 3
	constexpr int BUFW = 8192 + 1024;          // words per hop buffer incl. padding
	constexpr int NH = 1024 / T;               // halves of the hop buffer a CTA walks through
	static_assert(UPB <= T, "an N-block's threads must sit in one half");
	extern __shared__ __align__(128) unsigned char smem_raw[];
	uint64_t *bar = reinterpret_cast<uint64_t *>(smem_raw);                   // two mbarriers
	long long *red = reinterpret_cast<long long *>(smem_raw + 16);            // 64 x 8 B
	uint32_t *bufs = reinterpret_cast<uint32_t *>(smem_raw + 16 + 512);       // 2 x BUFW words
	uint32_t *tw = bufs + 2 * BUFW;                                           // N/2 packed twiddles
	int16_t *win = reinterpret_cast<int16_t *>(tw + (N / 2 > 4 ? N / 2 : 4)); // N window coefficients
	const int tid = threadIdx.x;
	const int hop_local = blockIdx.x / a.slices;
	const int slice = blockIdx.x % a.slices;
	const int hop = a.hop_begin + hop_local;
	const int uu = tid & (UPB - 1);            // the same in every half (UPB divides T)

	// tables: packed twiddles (wr = Sinewave[j + N/4] >> 1, wi = (int16)(-Sinewave[j]) >> 1, src/rtl_power.c:298-301)
	for (int i = tid; i < N / 2; i += T) {
		int wr = (int)a.sine[i + N / 4] >> 1;
		int wi = neg_half(a.sine[i]);
		tw[i] = ppack(wr, wi);
	}
	for (int i = tid; i < N; i += T) { win[i] = a.window[i]; }
	if (tid == 0) { mbar_init(&bar[0], 1); mbar_init(&bar[1], 1); }
	__syncthreads();

	long long acc[8];
#pragma unroll
	for (int j = 0; j < 8; j++) { acc[j] = 0; }

	const size_t hop_stride = (size_t)a.n_hops_call * (size_t)a.buf_len;
	const int16_t *src0 = a.bufs + (size_t)hop_local * (size_t)a.buf_len;
	if (tid == 0 && slice < a.n_pass) {
		mbar_expect_tx(&bar[0], 32768u);
		bulk_load(bufs, src0 + (size_t)slice * hop_stride, 32768u, &bar[0]);
	}
	uint32_t parity[2] = {0u, 0u};
	int it = 0;
	for (int pass = slice; pass < a.n_pass; pass += a.slices, it++) {
		const int cur = it & 1;
		uint32_t *buf = bufs + cur * BUFW;
		mbar_wait(&bar[cur], parity[cur]);
		parity[cur] ^= 1u;
		__syncthreads();                       // everyone is done with the other buffer (previous iteration)
		if (tid == 0 && pass + a.slices < a.n_pass) {
			fence_async_smem();
			mbar_expect_tx(&bar[cur ^ 1], 32768u);
			bulk_load(bufs + (cur ^ 1) * BUFW, src0 + (size_t)(pass + a.slices) * hop_stride, 32768u, &bar[cur ^ 1]);
		}
		// remove_dc over the whole hop buffer (src/rtl_power.c:609-624, :744-745): every thread sums the points it
		// will transform, straight from the TMA image
		long long si = 0, sq = 0;
#pragma unroll
		for (int hf = 0; hf < NH; hf++) {
			const int blk = (tid + hf * T) >> (E - 3);
#pragma unroll
			for (int j = 0; j < 8; j++) {
				const uint32_t w = buf[blk * N + j * UPB + uu];
				si += plo(w); sq += phi(w);
			}
		}
		for (int o = 16; o > 0; o >>= 1) { si += __shfl_down_sync(0xffffffffu, si, o); sq += __shfl_down_sync(0xffffffffu, sq, o); }
		if ((tid & 31) == 0) { red[tid >> 5] = si; red[32 + (tid >> 5)] = sq; }
		__syncthreads();
		long long ti_ = 0, tq_ = 0;
#pragma unroll 8
		for (int w = 0; w < T / 32; w++) { ti_ += red[w]; tq_ += red[32 + w]; }
		const int ave_i = (int)(int16_t)(ti_ / 16384LL);
		const int ave_q = (int)(int16_t)(tq_ / 16383LL);
		// Layout note: trip t > 0 keeps block b at b * (N + UPB) (padded), the TMA image has it at b * N.  The padded
		// region of the upper half of the blocks starts past the raw image of the lower half, so the upper half goes
		// first and the lower half's raw samples are still intact when their turn comes.
#pragma unroll
		for (int hf = NH - 1; hf >= 0; hf--) {
			const int blk = (tid + hf * T) >> (E - 3);
			Cx x[8];
#pragma unroll
			for (int j = 0; j < 8; j++) {      // trip 0 loads: n = j*N/8 + uu of block blk; window multiply with int16 wrap (:749-758)
				const uint32_t raw = buf[blk * N + j * UPB + uu];
				const int w = win[j * UPB + uu];
				x[j].re = (plo(raw) - ave_i) * w;             // low 16 bits = the reference's int16 store
				x[j].im = (phi(raw) - ave_q) * w;
			}
#pragma unroll
			for (int t = 0; t < NT; t++) {
				const bool last = (t == NT - 1);
				// geometry of this trip: stages s0, s0+1, s0+2 (the last trip of a non-multiple-of-3 E re-uses
				// s0 = E-3 and skips the stages an earlier trip already did)
				const int s0 = (last && REM != 0) ? (E - 3) : 3 * t;
				const int first = (last && REM != 0) ? (3 - REM) : 0;
				const int lbw = E - 3 - s0;               // log2 of the spacing of the thread's points
				const int B = uu & ((1 << lbw) - 1);
				const int A = uu >> lbw;
				if (t > 0) {
#pragma unroll
					for (int j = 0; j < 8; j++) {
						uint32_t w = buf[blk * (N + UPB) + A * (9 << lbw) + (j << lbw) + B];
						x[j].re = plo(w); x[j].im = phi(w);
					}
				}
				const int rA = s0 > 0 ? (int)(__brev((unsigned)A) >> (32 - (s0 > 0 ? s0 : 1))) : 0;
				if (t == 0 && first == 0 && a.triv) { trip_first_triv<E>(x, tw); }
				else { trip_stages<E>(x, tw, rA, s0, first); }
				if (!last) {
					// store in the layout of the next trip: slot n -> n + (n >> (lbw' + 3)) << lbw'
					const int s0n = (t + 1 == NT - 1 && REM != 0) ? (E - 3) : 3 * (t + 1);
					const int lbn = E - 3 - s0n;
					__syncthreads();               // all loads of this trip are done: the buffer may be rewritten in place
#pragma unroll
					for (int j = 0; j < 8; j++) {
						const int n = (A << (lbw + 3)) + (j << lbw) + B;
						buf[blk * (N + UPB) + n + ((n >> (lbn + 3)) << lbn)] = ppack(x[j].re, x[j].im);
					}
					__syncthreads();
				}
			}
			// real_conj accumulate (:664-668, :760-768): this thread's slots are n = 8*uu + j
#pragma unroll
			for (int j = 0; j < 8; j++) {
				const int vr = (int)(int16_t)x[j].re, vi = (int)(int16_t)x[j].im;      // the reference's int16 store
				const long long pw = (long long)((unsigned)(vr * vr) + (unsigned)(vi * vi));   // <= 2^31: fits 32 bits unsigned
				if (a.peak_hold) { acc[j] = pw > acc[j] ? pw : acc[j]; } else { acc[j] += pw; }
			}
		}
	}
	// slot n of a block holds bin rev(n)
	long long *row = a.avg + (size_t)hop * N;
#pragma unroll
	for (int j = 0; j < 8; j++) {
		const int n = 8 * uu + j;
		const int bin = (int)(__brev((unsigned)n) >> (32 - E));
		if (a.peak_hold) { atomicMax(row + bin, acc[j]); }
		else { atomicAdd(reinterpret_cast<unsigned long long *>(row + bin), (unsigned long long)acc[j]); }
	}
}

// rms_power (src/rtl_power.c:403-429): one value per hop buffer.
__global__ void __launch_bounds__(256) power_rms_kernel(const PowArgs a)
{
	__shared__ long long red[32];
	const int tid = threadIdx.x, T = blockDim.x;
	const int hop_local = blockIdx.x / a.slices;
	const int slice = blockIdx.x % a.slices;
	const int hop = a.hop_begin + hop_local;
	long long acc = 0;
	for (int pass = slice; pass < a.n_pass; pass += a.slices) {
		const int16_t *src = a.bufs + ((size_t)pass * a.n_hops_call + hop_local) * (size_t)a.buf_len;
		const uint4 *src4 = reinterpret_cast<const uint4 *>(src);
		long long t = 0, p = 0;
		for (int i = tid; i < a.buf_len / 8; i += T) {
			uint4 v = __ldg(src4 + i);
			uint32_t ws[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
			for (int q = 0; q < 4; q++) {
				int s0 = plo(ws[q]), s1 = phi(ws[q]);
				t += s0 + s1;
				p += (long long)(s0 * s0) + (long long)(s1 * s1);
			}
		}
		t = block_sum(t, red, tid, T);
		p = block_sum(p, red, tid, T);
		if (tid == 0) {
			// dc = t/buf_len; err = t*2*dc - dc*dc*buf_len; p -= round(err): same operation order as the
			// reference, no fused multiply-add
			double dc = __ddiv_rn((double)t, (double)a.buf_len);
			double e1 = __dmul_rn((double)(t * 2), dc);
			double e2 = __dmul_rn(__dmul_rn(dc, dc), (double)a.buf_len);
			double err = __dsub_rn(e1, e2);
			p -= (long long)round(err);
			fold(acc, p, a.peak_hold);
		}
	}
	if (tid == 0) { flush(a.avg + hop, acc, a.peak_hold); }
}


// ---------------------------------------------------------------------------------------------
// Hop buffers that do not fit shared memory (bin_e 16..21, src/rtl_power.c:485-491): the same arithmetic with the
// work buffer in global memory, one launch per step of the reference's loop (:715-771).  A rare, bandwidth-heavy path
// (the planner only gets here for sub-50-Hz bins); it exists for coverage, the shared-memory kernels are the product.
//   big_load:  copy (:715-720) + boxcar (:723-733) + the two remove_dc sums (:609-624)
//   big_window: (x - ave) * w with int16 wrap (:749-758), stored bit-reversed (fix_fft's swap pass, :275-290)
//   big_stage:  one radix-2 stage over every N-block (:291-318)
//   big_accum:  real_conj accumulate / peak hold (:760-768)
__global__ void __launch_bounds__(256) power_big_load(const uint32_t *src, uint32_t *work, int n_complex, int ds, int used_int16,
                                                      long long *sums)
{
	const int n_out = (n_complex + ds - 1) / ds;
	// remove_dc sums the first used_int16 int16 (:744-745): a partial last slot of the boxcar may lie past that span
	const int n_i = (used_int16 + 1) / 2, n_q = used_int16 / 2;
	long long si = 0, sq = 0;
	for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n_out; k += gridDim.x * blockDim.x) {
		const uint32_t v = boxcar_slot(src, k, ds, n_complex);
		work[k] = v;
		if (k < n_i) { si += plo(v); }
		if (k < n_q) { sq += phi(v); }
	}
	for (int o = 16; o > 0; o >>= 1) { si += __shfl_down_sync(0xffffffffu, si, o); sq += __shfl_down_sync(0xffffffffu, sq, o); }
	if ((threadIdx.x & 31) == 0) {
		atomicAdd(reinterpret_cast<unsigned long long *>(sums), (unsigned long long)si);
		atomicAdd(reinterpret_cast<unsigned long long *>(sums + 1), (unsigned long long)sq);
	}
}

// big_decim: copy + the -F decimator (downsample_iq x P, then the droop FIR, :734-743) + the two remove_dc sums, in place
// of big_load when boxcar == 0.  The host only routes shapes here whose every pass length buf_len >> j is a multiple of
// 4 int16 and whose decimated span is whole N-blocks (buf_len = k * 2N * 2^P: every planner shape), so I and Q have
// the same sample count n_l = buf_len >> (l+1) at every level l and the blocks read nothing past the decimated span.
//
// Each output of a pass is a pure function of ORIGINAL samples of its input (the in-place loop of fifth_order only ever
// reads what it has not yet overwritten), so a CTA can produce a tile [m0, m1) of final samples from the level-0 span
// that tile depends on: level l+1 sample k reads level-l samples 2k-5 .. 2k (k >= 5) or 0 .. 8 (the ease-in head,
// k < 5), and the FIR adds final samples m0-9 .. m0-1.  The span is staged by one bulk copy from a 16-byte-aligned
// start, every pass runs in place in shared memory, and only the tile's final samples go back to HBM.
#define RXB_DECIM_RNG 16                    // byte offset of the per-level window table in shared memory
#define RXB_DECIM_DATA 256                  // byte offset of the level-0 span
#define RXB_DECIM_R 4                       // outputs per thread per in-place round
__host__ __device__ __forceinline__ void decim_window(int m0, int m1, int P, int fir_on, int *lo, int *hi)
{
	// level-l window [lo[l], hi[l]] of a tile [m0, m1) of final samples, l = P down to 0
	lo[P] = m0 - 9 * fir_on > 0 ? m0 - 9 * fir_on : 0;
	hi[P] = m1 - 1;
	for (int l = P; l > 0; l--) {
		lo[l - 1] = 2 * lo[l] - 5 > 0 ? 2 * lo[l] - 5 : 0;
		hi[l - 1] = hi[l] >= 5 ? 2 * hi[l] : 8;
	}
	lo[0] &= ~3;                            // whole 16-byte words of the hop buffer
	hi[0] |= 3;
}

struct DecimFir { int c[6]; };

__global__ void __launch_bounds__(256) power_big_decim(const int16_t *src, uint32_t *work, int n_final, int tile, int P, int fir_on,
                                                       const DecimFir fir, long long *sums)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	uint64_t *bar = reinterpret_cast<uint64_t *>(smem_raw);
	int *win_lo = reinterpret_cast<int *>(smem_raw + RXB_DECIM_RNG);      // [11]
	int *win_hi = win_lo + 11;                                             // [11]
	uint32_t *x = reinterpret_cast<uint32_t *>(smem_raw + RXB_DECIM_DATA);
	const int tid = threadIdx.x, T = blockDim.x;
	const int m0 = blockIdx.x * tile;
	const int m1 = m0 + tile < n_final ? m0 + tile : n_final;
	if (tid == 0) {
		decim_window(m0, m1, P, fir_on, win_lo, win_hi);
		mbar_init(bar, 1);
		const uint32_t bytes = (uint32_t)(win_hi[0] - win_lo[0] + 1) * 4u;
		mbar_expect_tx(bar, bytes);
		bulk_load(x, src + 2 * (size_t)win_lo[0], bytes, bar);
	}
	__syncthreads();
	mbar_wait(bar, 0);
	// downsample_iq, pass l: level l (window at win_lo[l]) -> level l+1, in place.  Output k lands at k - lo1 while the
	// outputs of later rounds read at >= 2 (k' - lo1) > k - lo1 (lo = max(0, 2 lo1 - 5), rounded down), so a round only
	// has to finish its reads before it writes.
	for (int l = 0; l < P; l++) {
		const int lo = win_lo[l], lo1 = win_lo[l + 1], n1 = win_hi[l + 1] - lo1 + 1;
		for (int base = 0; base < n1; base += T * RXB_DECIM_R) {
			uint32_t y[RXB_DECIM_R];
#pragma unroll
			for (int r = 0; r < RXB_DECIM_R; r++) {
				const int j = base + r * T + tid;
				if (j < n1) { y[r] = ppack(hb_out(x, lo, lo1 + j, 0), hb_out(x, lo, lo1 + j, 1)); }
			}
			__syncthreads();
#pragma unroll
			for (int r = 0; r < RXB_DECIM_R; r++) {
				const int j = base + r * T + tid;
				if (j < n1) { x[j] = y[r]; }
			}
			__syncthreads();
		}
	}
	// droop FIR (samples 0..8 pass through), store the tile, sum it for remove_dc
	const int loP = win_lo[P];
	long long si = 0, sq = 0;
	for (int m = m0 + tid; m < m1; m += T) {
		uint32_t v = x[m - loP];
		if (fir_on && m >= 9) { v = ppack(fir_out(x, loP, m, 0, fir.c), fir_out(x, loP, m, 1, fir.c)); }
		work[m] = v;
		si += plo(v); sq += phi(v);
	}
	for (int o = 16; o > 0; o >>= 1) { si += __shfl_down_sync(0xffffffffu, si, o); sq += __shfl_down_sync(0xffffffffu, sq, o); }
	if ((tid & 31) == 0) {
		atomicAdd(reinterpret_cast<unsigned long long *>(sums), (unsigned long long)si);
		atomicAdd(reinterpret_cast<unsigned long long *>(sums + 1), (unsigned long long)sq);
	}
}

__global__ void __launch_bounds__(256) power_big_window(const uint32_t *work, uint32_t *fft, const int16_t *win, const long long *sums,
                                                        int used_int16, int n_slots, int bin_e, int nblk)
{
	const int N = 1 << bin_e;
	const Dc dc = dc_average(sums[0], sums[1], used_int16);
	const long long total = (long long)nblk * N;
	for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
		const int i = (int)(g & (N - 1));
		const long long base = g - i;
		const int r = (int)(__brev((unsigned)i) >> (32 - bin_e));
		// past the decimated span the reference transforms what the boxcar left there: a partial last slot, then zeros
		fft[base + r] = dc_window(g < n_slots ? work[g] : 0u, (int)g, dc, win[i]);
	}
}

__global__ void __launch_bounds__(256) power_big_stage(uint32_t *fft, const int16_t *sine, int bin_e, int s, int nblk)
{
	const int N = 1 << bin_e;
	const long long total = (long long)nblk * (N / 2);
	for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
		const int t = (int)(g & (N / 2 - 1));
		dit_bfly(fft + (g - t) * 2, t, s, bin_e, sine);
	}
}

__global__ void __launch_bounds__(256) power_big_accum(const uint32_t *fft, long long *row, int bin_e, int nblk, int peak_hold)
{
	const int N = 1 << bin_e;
	for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < N; j += gridDim.x * blockDim.x) {
		long long acc = row[j];
		for (int b = 0; b < nblk; b++) { fold(acc, bin_power(fft[(size_t)b * N + j]), peak_hold); }
		row[j] = acc;
	}
}

}  // namespace rxb

using namespace rxb;

#define RXB_ROW_PAD 16        // >= the largest communicator size - 1
struct rxb200_power {
	rxb200_power_params p;
	int device;
	cudaStream_t stream;
	long long *d_avg;          // [n_hops + RXB_ROW_PAD][N]: the padding rows stay zero; they make the hop rows a whole
	                           // number of equal per-rank blocks so the all-gather runs in place (SURVEY.md §8e)
	int *d_samples;            // [n_hops + RXB_ROW_PAD] staging of `samples` for the gather
	int16_t *d_sine, *d_window;
	int16_t *d_in; size_t d_in_cap;
	std::vector<int> samples;  // tunes[i].samples mirror (deterministic, kept on the host)
	int n_sm;
	cudaEvent_t ev0, ev1;
	unsigned char *d_db = nullptr; size_t db_cap = 0;   // csv_dbm staging (rxb200_power_read_db)
	int triv = 0;                              // see PowArgs::triv
	uint32_t *d_work = nullptr, *d_fft = nullptr; long long *d_sums = nullptr;   // global-memory path (hop buffer beyond shared memory)
	int force_v1 = 0;                          // RXB200_POWER_V1 (A/B knob, read once at create): generic kernel only
	int fft8_threads = 0;                      // RXB200_POWER_THREADS = 512 | 1024 (A/B knob): CTA width of the fast path
	rxb200_power_path path = {};               // what the last accumulate ran (rxb200_power_last_path)
};

#define RXB_SMEM_MAX (227 * 1024)          // dynamic shared memory a CTA may opt in to on sm_90

// power_fft_kernel's shared memory without its tables: the mbarrier, the reduction scratch and the hop buffer.  A hop
// buffer for which this exceeds RXB_SMEM_MAX runs on the global-memory kernels.
static size_t hop_smem(int buf_len) { return 16 + 256 + (size_t)buf_len * 2; }

static int power_validate(const rxb200_power_params *p)
{
	if (p->n_hops < 1 || p->bin_e < 0 || p->bin_e > 21 || p->buf_len < 16 || (p->buf_len % 8) != 0) {
		set_error("bad rx_power parameters"); return RXB200_EINVAL;
	}
	if (p->bin_e > 0) {
		if (p->downsample < 1 || p->downsample_passes < 0 || p->downsample_passes > 10) {
			set_error("bad downsample %d / passes %d", p->downsample, p->downsample_passes);
			return RXB200_EINVAL;
		}
		if ((long long)(2 << p->bin_e) * p->downsample > p->buf_len) {
			set_error("bin_e %d x downsample %d needs more than buf_len %d", p->bin_e, p->downsample, p->buf_len);
			return RXB200_EINVAL;
		}
		if (hop_smem(p->buf_len) > RXB_SMEM_MAX && p->downsample > 1 && !p->boxcar &&
		    (p->downsample_passes < 1 || p->downsample != (1 << p->downsample_passes) ||
		     p->buf_len % ((2LL << p->bin_e) * p->downsample) != 0)) {
			// power_big_decim assumes the planner's geometry (src/rtl_power.c:466-474, :504-507): downsample = 2^passes and
			// the decimated span is whole N-blocks, so every pass keeps I and Q the same length and no block reads the
			// leftovers of earlier passes.  This covers every plan the big path routes to it (boxcar 0, downsample > 1).
			set_error("-F decimation of a hop buffer beyond shared memory needs downsample = 2^passes (%d, %d) and buf_len %d a multiple of 2 x %d x downsample",
			          p->downsample, p->downsample_passes, p->buf_len, 1 << p->bin_e);
			return RXB200_EUNSUPPORTED;
		}
		// the block loop runs while offset < buf_len/downsample (src/rtl_power.c:747): a partial last block is
		// transformed too (over the zeros the decimator left), which only stays inside the hop buffer when the
		// rounded-up block count does -- the planner's shapes do (:504-507); anything else would run past the buffer
		{
			const long long used = p->buf_len / p->downsample, two_n = 2LL << p->bin_e;
			if (((used + two_n - 1) / two_n) * two_n > p->buf_len) {
				set_error("buf_len %d / downsample %d: the last %d-point block would end past the hop buffer", p->buf_len, p->downsample, 1 << p->bin_e);
				return RXB200_EINVAL;
			}
		}
	}
	return RXB200_OK;
}

extern "C" int rxb200_power_create(const rxb200_power_params *params, const int *window_coefs,
                                   const int16_t *sinewave, int device, rxb200_power **out)
{
	if (!params || !out || (params->bin_e > 0 && !window_coefs)) { set_error("null argument"); return RXB200_EINVAL; }
	*out = nullptr;
	int rc = power_validate(params);
	if (rc != RXB200_OK) { return rc; }
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { set_error("no CUDA device: librxb200 has no CPU fallback"); return RXB200_ENODEV; }
	if (device < 0 || device >= ndev) { set_error("device %d out of range (%d)", device, ndev); return RXB200_ENODEV; }
	RXB_CUDA(cudaSetDevice(device));
	rxb200_power *h = new (std::nothrow) rxb200_power();
	if (!h) { return RXB200_ENOMEM; }
	h->p = *params; h->device = device; h->d_avg = nullptr; h->d_samples = nullptr; h->d_sine = nullptr; h->d_window = nullptr;
	h->d_in = nullptr; h->d_in_cap = 0;
	h->samples.assign(params->n_hops, 0);
	h->force_v1 = getenv("RXB200_POWER_V1") ? 1 : 0;
	h->fft8_threads = getenv("RXB200_POWER_THREADS") ? atoi(getenv("RXB200_POWER_THREADS")) : 0;
	cudaDeviceProp prop;
	RXB_CUDA_OR(cudaGetDeviceProperties(&prop, device), rxb200_power_destroy(h));
	h->n_sm = prop.multiProcessorCount;
	RXB_CUDA_OR(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking), rxb200_power_destroy(h));
	RXB_CUDA_OR(cudaEventCreate(&h->ev0), rxb200_power_destroy(h));
	RXB_CUDA_OR(cudaEventCreate(&h->ev1), rxb200_power_destroy(h));
	const size_t N = (size_t)1 << params->bin_e;
	const size_t rows_cap = (size_t)params->n_hops + RXB_ROW_PAD;
	RXB_CUDA_OR(cudaMalloc(&h->d_avg, rows_cap * N * sizeof(long long)), rxb200_power_destroy(h));
	RXB_CUDA_OR(cudaMemset(h->d_avg, 0, rows_cap * N * sizeof(long long)), rxb200_power_destroy(h));
	RXB_CUDA_OR(cudaMalloc(&h->d_samples, rows_cap * sizeof(int)), rxb200_power_destroy(h));
	RXB_CUDA_OR(cudaMemset(h->d_samples, 0, rows_cap * sizeof(int)), rxb200_power_destroy(h));
	if (params->bin_e > 0) {
		std::vector<int16_t> sine(N * 3 / 4 + 8), win(N);
		if (sinewave) { memcpy(sine.data(), sinewave, (N * 3 / 4) * sizeof(int16_t)); }
		else { rxb200_sine_table(params->bin_e, sine.data()); }
		// (int16)(x * w) depends only on w modulo 2^16, so the table is kept as int16
		for (size_t i = 0; i < N; i++) { win[i] = (int16_t)window_coefs[i]; }
		h->triv = (N >= 8 && sine[0] == 0 && (sine[N / 2] == 0 || sine[N / 2] == 1)) ? 1 : 0;
		RXB_CUDA_OR(cudaMalloc(&h->d_sine, sine.size() * sizeof(int16_t)), rxb200_power_destroy(h));
		RXB_CUDA_OR(cudaMalloc(&h->d_window, win.size() * sizeof(int16_t)), rxb200_power_destroy(h));
		RXB_CUDA_OR(cudaMemcpy(h->d_sine, sine.data(), sine.size() * sizeof(int16_t), cudaMemcpyHostToDevice), rxb200_power_destroy(h));
		RXB_CUDA_OR(cudaMemcpy(h->d_window, win.data(), win.size() * sizeof(int16_t), cudaMemcpyHostToDevice), rxb200_power_destroy(h));
	}
	*out = h;
	return RXB200_OK;
}

extern "C" void rxb200_power_destroy(rxb200_power *h)
{
	if (!h) { return; }
	cudaSetDevice(h->device);
	if (h->stream) { cudaStreamSynchronize(h->stream); }
	cudaFree(h->d_avg); cudaFree(h->d_samples); cudaFree(h->d_sine); cudaFree(h->d_window); cudaFree(h->d_in); cudaFree(h->d_db); cudaFree(h->d_work); cudaFree(h->d_fft); cudaFree(h->d_sums);
	if (h->ev0) { cudaEventDestroy(h->ev0); }
	if (h->ev1) { cudaEventDestroy(h->ev1); }
	if (h->stream) { cudaStreamDestroy(h->stream); }
	delete h;
}

extern "C" int rxb200_power_kernel_ms(rxb200_power *h, float *ms)
{
	if (!h || !ms) { return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(h->device));
	RXB_CUDA(cudaEventSynchronize(h->ev1));
	RXB_CUDA(cudaEventElapsedTime(ms, h->ev0, h->ev1));
	return RXB200_OK;
}

template <int NB>
static cudaError_t launch_fft_nb(const PowArgs &a, int blocks, size_t smem, cudaStream_t st)
{
	cudaError_t e = cudaFuncSetAttribute(power_fft_kernel<NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
	if (e != cudaSuccess) { return e; }
	power_fft_kernel<NB><<<blocks, 256, smem, st>>>(a);
	return cudaGetLastError();
}
static cudaError_t launch_fft(int nb, const PowArgs &a, int blocks, size_t smem, cudaStream_t st)
{
	switch (nb) {
	case 1: return launch_fft_nb<1>(a, blocks, smem, st);
	case 2: return launch_fft_nb<2>(a, blocks, smem, st);
	case 4: return launch_fft_nb<4>(a, blocks, smem, st);
	case 8: return launch_fft_nb<8>(a, blocks, smem, st);
	case 16: return launch_fft_nb<16>(a, blocks, smem, st);
	default: return launch_fft_nb<0>(a, blocks, smem, st);
	}
}

template <int E, int T>
static cudaError_t launch_fft8_e(const PowArgs &a, int blocks, size_t smem, cudaStream_t st)
{
	cudaError_t e = cudaFuncSetAttribute(power_fft8_kernel<E, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
	if (e != cudaSuccess) { return e; }
	power_fft8_kernel<E, T><<<blocks, T, smem, st>>>(a);
	return cudaGetLastError();
}
// threads per CTA of the fast path: 512 (two CTAs per SM) wherever an N-block fits half a CTA, i.e. up to N = 4096
static int fft8_threads(int bin_e, int force) { return (force == 512 || force == 1024) ? (bin_e <= 12 ? force : 1024) : (bin_e <= 12 ? 512 : 1024); }
static cudaError_t launch_fft8(int bin_e, int threads, const PowArgs &a, int blocks, size_t smem, cudaStream_t st)
{
#define RXB_FFT8_CASE(E) case E: return threads == 512 ? launch_fft8_e<E, 512>(a, blocks, smem, st) : launch_fft8_e<E, 1024>(a, blocks, smem, st);
	switch (bin_e) {
	RXB_FFT8_CASE(3) RXB_FFT8_CASE(4) RXB_FFT8_CASE(5) RXB_FFT8_CASE(6) RXB_FFT8_CASE(7) RXB_FFT8_CASE(8)
	RXB_FFT8_CASE(9) RXB_FFT8_CASE(10) RXB_FFT8_CASE(11) RXB_FFT8_CASE(12)
	case 13: return launch_fft8_e<13, 1024>(a, blocks, smem, st);
	default: return cudaErrorInvalidValue;
	}
#undef RXB_FFT8_CASE
}

// power_big_decim's tile: about four CTAs per SM (one CTA's serial passes leave the SM mostly idle), but no smaller than
// four times the per-tile halo of 5 (+ 9 with the FIR) final samples, which keeps the level-0 read amplification near
// 1.25 or below, and no larger than a level-0 span that fits shared memory.  `smem` covers the largest span over all
// tiles (the 16-byte rounding varies from tile to tile).
static int decim_span_max(int n_final, int tile, int P, int fir_on)
{
	int lo[11], hi[11], worst = 0;
	for (int m0 = 0; m0 < n_final; m0 += tile) {
		decim_window(m0, m0 + tile < n_final ? m0 + tile : n_final, P, fir_on, lo, hi);
		if (hi[0] - lo[0] + 1 > worst) { worst = hi[0] - lo[0] + 1; }
	}
	return worst;
}
static void decim_plan(int n_final, int P, int fir_on, int n_sm, int *tile, size_t *smem)
{
	const int cap = (RXB_SMEM_MAX - RXB_DECIM_DATA) / 4;                 // level-0 complex samples a CTA can stage
	const int halo = 5 + 9 * fir_on;
	int t = (n_final + 4 * n_sm - 1) / (4 * n_sm);
	if (t < 4 * halo) { t = 4 * halo; }
	const int t_cap = (cap - 7 - 5 * ((1 << P) - 1)) / (1 << P) + 1 - 9 * fir_on;
	if (t > t_cap) { t = t_cap; }
	if (t > n_final) { t = n_final; }
	while (t > 1 && decim_span_max(n_final, t, P, fir_on) > cap) { t--; }
	*tile = t;
	*smem = RXB_DECIM_DATA + (size_t)decim_span_max(n_final, t, P, fir_on) * 4;
}

// droop compensation after the -F passes (src/rtl_power.c:739-742)
static int fir_on(const rxb200_power_params &p) { return (p.comp_fir_size == 9 && p.downsample_passes >= 1 && p.downsample_passes <= 10) ? 1 : 0; }

// One accumulate call's launch
struct PowerPlan {
	rxb200_power_path path;   // what rxb200_power_last_path reports; PowArgs takes its slices and tables_in_smem
	int blocks;               // CTAs of the kernel that reads the hop buffers (the global-memory path: big_load or big_decim)
	size_t smem;              // its dynamic shared memory
	int tile;                 // power_big_decim: final samples per CTA
	int nblk, n_slots;        // bin_e > 0: N-blocks per hop buffer (:747), complex samples after decimation
	int samples;              // added to every hop's `samples` per pass (:428, :769)
};

static void power_plan(const rxb200_power *h, int n_pass, int nh, PowerPlan *pl)
{
	const rxb200_power_params &p = h->p;
	*pl = {};
	// enough CTAs for ~4 per SM, never more slices than passes
	int slices = (h->n_sm * 4 + nh - 1) / nh;
	if (slices > n_pass) { slices = n_pass; }
	if (slices < 1) { slices = 1; }
	pl->blocks = nh * slices;
	if (p.bin_e == 0) {
		pl->path = {RXB200_POWER_PATH_RMS, 0, 256, -1, 0, slices, 1};
		pl->samples = 1;
		return;
	}
	const int N = 1 << p.bin_e;
	pl->nblk = (p.buf_len / p.downsample + 2 * N - 1) / (2 * N);      // over the int16 span after decimation (:744-747)
	pl->n_slots = (p.buf_len / 2 + p.downsample - 1) / p.downsample;  // -F: exactly half that span
	pl->samples = pl->nblk * p.downsample;
	if (hop_smem(p.buf_len) > RXB_SMEM_MAX) {
		// -F passes only when the plan decimates: downsample == 1 keeps the plain copy, as the shared-memory kernel does
		const bool decim = !p.boxcar && p.downsample > 1 && p.downsample_passes > 0;
		pl->path = {decim ? RXB200_POWER_PATH_BIG_DECIM : RXB200_POWER_PATH_BIG_LOAD, p.bin_e, 256, -1, 0, 0, n_pass * nh * (3 + p.bin_e)};
		pl->blocks = h->n_sm * 8;
		if (decim) {
			decim_plan(pl->n_slots, p.downsample_passes, fir_on(p), h->n_sm, &pl->tile, &pl->smem);
			pl->blocks = (pl->n_slots + pl->tile - 1) / pl->tile;
		}
		return;
	}
	if (p.downsample == 1 && p.buf_len == 16384 && p.bin_e >= 3 && p.bin_e <= 13 && !h->force_v1) {
		// one CTA per (hop, pass-slice); 1024 threads: ~1 CTA per SM resident, 512 threads: 2
		const int threads = fft8_threads(p.bin_e, h->fft8_threads);
		// slices of the passes per hop: the launch takes ceil(nh*sl / resident CTAs) rounds of ceil(n_pass / sl) hop
		// buffers each -- pick the split with the fewest buffer-times (a sharded rank owns few hops: 109 of 871 at
		// eight GPUs, where "about one CTA per slot" left 31 CTAs for a second round of 12 buffers each)
		const long long slots = (long long)h->n_sm * (1024 / threads);
		int sl = 1;
		long long best = -1;
		for (int c = 1; c <= n_pass && (long long)c <= 2 * slots; c++) {
			// + 1: a CTA's fixed cost (tables, accumulator flush) is about one hop buffer's worth of work
			const long long rounds = ((long long)nh * c + slots - 1) / slots;
			const long long t = rounds * ((n_pass + c - 1) / c + 1) * 4096 + c;   // ties: fewer slices (fewer atomic flushes)
			if (best < 0 || t < best) { best = t; sl = c; }
		}
		pl->path = {RXB200_POWER_PATH_FFT8, p.bin_e, threads, -1, 1, sl, 1};
		pl->blocks = nh * sl;
		pl->smem = 16 + 512 + 2 * (8192 + 1024) * 4 + (size_t)(N / 2 > 4 ? N / 2 : 4) * 4 + (size_t)N * 2;
		return;
	}
	// the sine and window tables go to shared memory when they fit beside the hop buffer
	const size_t with_tables = hop_smem(p.buf_len) + (size_t)((N * 3 / 4 + 7) & ~7) * 2 + (size_t)N * 2;
	const int in_smem = with_tables <= RXB_SMEM_MAX ? 1 : 0;
	const int nb = N / 256;
	pl->path = {RXB200_POWER_PATH_GENERIC, p.bin_e, 256, nb <= 1 ? 1 : (nb <= 16 ? nb : 0), in_smem, slices, 1};
	pl->smem = in_smem ? with_tables : hop_smem(p.buf_len);
}

extern "C" int rxb200_power_accumulate_device(rxb200_power *h, const int16_t *d_hop_bufs, int n_pass,
                                              int hop_begin, int hop_end, int sync)
{
	if (!h || !d_hop_bufs) { set_error("null argument"); return RXB200_EINVAL; }
	if (n_pass < 0 || hop_begin < 0 || hop_end > h->p.n_hops || hop_begin >= hop_end) { set_error("bad hop range"); return RXB200_EINVAL; }
	if (((uintptr_t)d_hop_bufs & 15u) != 0) { set_error("hop buffers must be 16-byte aligned"); return RXB200_EINVAL; }
	if (n_pass == 0) { return RXB200_OK; }
	RXB_CUDA(cudaSetDevice(h->device));
	const rxb200_power_params &p = h->p;
	const int nh = hop_end - hop_begin;
	PowerPlan pl;
	power_plan(h, n_pass, nh, &pl);
	const bool big = pl.path.kernel == RXB200_POWER_PATH_BIG_LOAD || pl.path.kernel == RXB200_POWER_PATH_BIG_DECIM;
	if (big && !h->d_work) {
		RXB_CUDA(cudaMalloc(&h->d_work, (size_t)pl.n_slots * sizeof(uint32_t)));
		RXB_CUDA(cudaMalloc(&h->d_fft, (size_t)pl.nblk * ((size_t)1 << p.bin_e) * sizeof(uint32_t)));
		RXB_CUDA(cudaMalloc(&h->d_sums, 2 * sizeof(long long)));
	}
	PowArgs a;
	a.bufs = d_hop_bufs; a.avg = h->d_avg; a.sine = h->d_sine; a.window = h->d_window;
	a.n_pass = n_pass; a.n_hops_call = nh; a.hop_begin = hop_begin; a.buf_len = p.buf_len;
	a.bin_e = p.bin_e; a.peak_hold = p.peak_hold; a.triv = h->triv;
	a.ds = p.downsample; a.ds_passes = p.downsample_passes; a.boxcar = p.boxcar;
	a.fir_on = fir_on(p);
	for (int j = 0; j < 6; j++) { a.fir[j] = k_droop9_host[p.downsample_passes <= 10 ? p.downsample_passes : 0][j]; }
	a.slices = pl.path.slices; a.tables_in_smem = pl.path.tables_in_smem;

	RXB_CUDA(cudaEventRecord(h->ev0, h->stream));
	cudaError_t e = cudaSuccess;
	switch (pl.path.kernel) {
	case RXB200_POWER_PATH_RMS:
		power_rms_kernel<<<pl.blocks, 256, 0, h->stream>>>(a);
		e = cudaGetLastError();
		break;
	case RXB200_POWER_PATH_FFT8: e = launch_fft8(p.bin_e, pl.path.threads, a, pl.blocks, pl.smem, h->stream); break;
	case RXB200_POWER_PATH_GENERIC: e = launch_fft(pl.path.nb, a, pl.blocks, pl.smem, h->stream); break;
	default: {
		// the reference's loop step by step on the global work buffers, one hop buffer at a time
		const bool decim = pl.path.kernel == RXB200_POWER_PATH_BIG_DECIM;
		if (decim) {
			// the attribute belongs to the kernel, not to this handle: allow the largest span any handle may plan
			RXB_CUDA(cudaFuncSetAttribute(power_big_decim, cudaFuncAttributeMaxDynamicSharedMemorySize, RXB_SMEM_MAX));
		}
		DecimFir fir;
		for (int j = 0; j < 6; j++) { fir.c[j] = a.fir[j]; }
		const int g = h->n_sm * 8, used = p.buf_len / p.downsample, N = 1 << p.bin_e;
		for (int pass = 0; pass < n_pass; pass++) {
			for (int hl = 0; hl < nh; hl++) {
				const int16_t *src = d_hop_bufs + ((size_t)pass * nh + hl) * (size_t)p.buf_len;
				RXB_CUDA(cudaMemsetAsync(h->d_sums, 0, 2 * sizeof(long long), h->stream));
				if (decim) {
					power_big_decim<<<pl.blocks, 256, pl.smem, h->stream>>>(src, h->d_work, pl.n_slots, pl.tile, p.downsample_passes,
					                                                         a.fir_on, fir, h->d_sums);
				} else {
					power_big_load<<<pl.blocks, 256, 0, h->stream>>>(reinterpret_cast<const uint32_t *>(src), h->d_work, p.buf_len / 2,
					                                                 p.downsample, used, h->d_sums);
				}
				power_big_window<<<g, 256, 0, h->stream>>>(h->d_work, h->d_fft, h->d_window, h->d_sums, used, pl.n_slots, p.bin_e, pl.nblk);
				for (int st = 0; st < p.bin_e; st++) { power_big_stage<<<g, 256, 0, h->stream>>>(h->d_fft, h->d_sine, p.bin_e, st, pl.nblk); }
				power_big_accum<<<g, 256, 0, h->stream>>>(h->d_fft, h->d_avg + (size_t)(hop_begin + hl) * N, p.bin_e, pl.nblk, p.peak_hold);
				RXB_CUDA(cudaGetLastError());
			}
		}
	}
	}
	if (e != cudaSuccess) { set_error("rx_power launch (path %d): %s", pl.path.kernel, cudaGetErrorString(e)); return RXB200_ECUDA; }
	for (int i = hop_begin; i < hop_end; i++) { h->samples[i] += n_pass * pl.samples; }
	RXB_CUDA(cudaEventRecord(h->ev1, h->stream));
	h->path = pl.path;
	if (sync) { RXB_CUDA(cudaStreamSynchronize(h->stream)); }
	return RXB200_OK;
}

extern "C" int rxb200_power_accumulate(rxb200_power *h, const int16_t *hop_bufs, int n_pass, int hop_begin, int hop_end)
{
	if (!h || !hop_bufs) { set_error("null argument"); return RXB200_EINVAL; }
	if (n_pass < 0 || hop_begin < 0 || hop_end > h->p.n_hops || hop_begin >= hop_end) { set_error("bad hop range"); return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(h->device));
	size_t elems = (size_t)n_pass * (size_t)(hop_end - hop_begin) * (size_t)h->p.buf_len;
	if (elems == 0) { return RXB200_OK; }
	RXB_CUDA(reserve(h->d_in, h->d_in_cap, elems));
	RXB_CUDA(cudaMemcpyAsync(h->d_in, hop_bufs, elems * sizeof(int16_t), cudaMemcpyHostToDevice, h->stream));
	return rxb200_power_accumulate_device(h, h->d_in, n_pass, hop_begin, hop_end, 1);
}

extern "C" int rxb200_power_read(rxb200_power *h, int64_t *avg, int *samples)
{
	if (!h) { return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(h->device));
	if (avg) {
		const size_t N = (size_t)1 << h->p.bin_e;
		RXB_CUDA(cudaMemcpyAsync(avg, h->d_avg, (size_t)h->p.n_hops * N * sizeof(long long), cudaMemcpyDeviceToHost, h->stream));
	}
	RXB_CUDA(cudaStreamSynchronize(h->stream));
	if (samples) { memcpy(samples, h->samples.data(), h->samples.size() * sizeof(int)); }
	return RXB200_OK;
}

// csv_dbm's arithmetic (src/rtl_power.c:783-811) without touching avg: element i of the patched and
// half-swapped row is avg0[(i + N/2) mod N] with avg0[0] := avg[1]; every kept bin goes through
// /rate, /samples, 10*log10 in that order; the trailing value divides by (rate*samples) at once.
__global__ void power_db_kernel(const long long *avg, const int *samples, int n_hops, int bin_e, int i1, int row_len,
                                double rate, double *db, size_t row_stride)
{
	const int hop = blockIdx.y;
	const int N = 1 << bin_e;
	const long long *row = avg + (size_t)hop * N;
	const double smp = (double)samples[hop];
	for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < row_len; j += gridDim.x * blockDim.x) {
		const bool last = (j == row_len - 1);
		int i = last ? i1 + row_len - 2 : i1 + j;          // the last kept bin is printed twice (:807)
		if (bin_e == 0) { i = 0; }
		long long v;
		if (bin_e > 0) {
			int src = (i + N / 2) & (N - 1);
			if (src == 0) { src = 1; }                      // avg[0] = avg[1] (:784)
			v = row[src];
		} else {
			v = row[0];
		}
		double d;
		if (last) { d = __ddiv_rn((double)v, __dmul_rn(rate, smp)); }
		else      { d = __ddiv_rn(__ddiv_rn((double)v, rate), smp); }
		db[(size_t)hop * row_stride + j] = __dmul_rn(10.0, log10(d));
	}
}

extern "C" int rxb200_power_read_db(rxb200_power *h, int rate, double crop, double *db, size_t row_stride, int *samples)
{
	if (!h || !db) { set_error("null argument"); return RXB200_EINVAL; }
	const int row_len = rxb200_power_row_len(h->p.bin_e, crop);
	if (row_len < 2 && h->p.bin_e > 0) { set_error("crop %f leaves no bins", crop); return RXB200_EINVAL; }
	if (row_stride < (size_t)row_len) { set_error("row_stride %zu < row_len %d", row_stride, row_len); return RXB200_ECAPACITY; }
	RXB_CUDA(cudaSetDevice(h->device));
	const int n_hops = h->p.n_hops;
	const size_t need = (size_t)n_hops * row_len * sizeof(double) + (size_t)n_hops * sizeof(int);
	RXB_CUDA(reserve(h->d_db, h->db_cap, need));
	double *d_db = reinterpret_cast<double *>(h->d_db);
	int *d_smp = reinterpret_cast<int *>(d_db + (size_t)n_hops * row_len);
	RXB_CUDA(cudaMemcpyAsync(d_smp, h->samples.data(), (size_t)n_hops * sizeof(int), cudaMemcpyHostToDevice, h->stream));
	const int len = 1 << h->p.bin_e;
	const int i1 = (int)((double)len * crop * 0.5);
	dim3 grid((unsigned)((row_len + 255) / 256 > 64 ? 64 : (row_len + 255) / 256), (unsigned)n_hops);
	power_db_kernel<<<grid, 256, 0, h->stream>>>(h->d_avg, d_smp, n_hops, h->p.bin_e, i1, row_len, (double)rate, d_db, (size_t)row_len);
	RXB_CUDA(cudaGetLastError());
	RXB_CUDA(cudaMemcpy2DAsync(db, row_stride * sizeof(double), d_db, (size_t)row_len * sizeof(double),
	                           (size_t)row_len * sizeof(double), (size_t)n_hops, cudaMemcpyDeviceToHost, h->stream));
	RXB_CUDA(cudaStreamSynchronize(h->stream));
	if (samples) { memcpy(samples, h->samples.data(), h->samples.size() * sizeof(int)); }
	return RXB200_OK;
}

extern "C" int64_t *rxb200_power_device_avg(rxb200_power *h) { return h ? reinterpret_cast<int64_t *>(h->d_avg) : nullptr; }

extern "C" int rxb200_power_reset(rxb200_power *h)
{
	if (!h) { return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(h->device));
	const size_t N = (size_t)1 << h->p.bin_e;
	RXB_CUDA(cudaMemsetAsync(h->d_avg, 0, (size_t)h->p.n_hops * N * sizeof(long long), h->stream));
	for (size_t i = 0; i < h->samples.size(); i++) { h->samples[i] = 0; }
	return RXB200_OK;
}

extern "C" void *rxb200_power_stream(rxb200_power *h) { return h ? (void *)h->stream : nullptr; }
extern "C" int rxb200_power_last_launches(rxb200_power *h) { return h ? h->path.launches : 0; }
extern "C" int rxb200_power_last_path(rxb200_power *h, rxb200_power_path *out)
{
	if (!h || !out) { set_error("null argument"); return RXB200_EINVAL; }
	*out = h->path;
	return RXB200_OK;
}

// ================================================================================ multi-GPU (SURVEY.md §8e)
// Tuner hops are independent; rank r of n owns the contiguous hops [r*per, (r+1)*per), per = ceil(n_hops/n).
// The report needs every row in hop order on the rank that prints (src/rtl_power.c:1047-1050): ONE all-gather of the
// int64 rows (plus the tiny `samples` vector), in place on the accumulator array itself -- its zero padding rows make
// n*per rows available on every rank, so nothing is allocated, zeroed or copied per report.
struct rxb200_comm {
	ncclComm_t comm;
	int n_ranks, rank, device;
};

#define RXB_NCCL(api, call, cleanup)                                                                         \
	do {                                                                                                     \
		ncclResult_t r__ = (call);                                                                           \
		if (r__ != ncclSuccess) {                                                                            \
			set_error("%s failed: %s (%s:%d)", #call, (api)->GetErrorString(r__), __FILE__, __LINE__);       \
			cleanup;                                                                                         \
			return RXB200_ECUDA;                                                                             \
		}                                                                                                    \
	} while (0)

extern "C" int rxb200_comm_unique_id(void *id128)
{
	if (!id128) { set_error("null argument"); return RXB200_EINVAL; }
	const NcclApi *nc = nccl_api();
	if (!nc) { return RXB200_EUNSUPPORTED; }
	ncclUniqueId id;
	RXB_NCCL(nc, nc->GetUniqueId(&id), (void)0);
	memcpy(id128, &id, RXB200_UNIQUE_ID_BYTES);
	return RXB200_OK;
}

extern "C" int rxb200_comm_create(int n_ranks, int rank, const void *id128, int device, rxb200_comm **out)
{
	if (!out || !id128 || n_ranks < 1 || n_ranks > RXB_ROW_PAD || rank < 0 || rank >= n_ranks) {
		set_error("bad communicator arguments (1 <= n_ranks <= %d)", RXB_ROW_PAD); return RXB200_EINVAL;
	}
	*out = nullptr;
	const NcclApi *nc = nccl_api();
	if (!nc) { return RXB200_EUNSUPPORTED; }
	RXB_CUDA(cudaSetDevice(device));
	rxb200_comm *c = new (std::nothrow) rxb200_comm();
	if (!c) { return RXB200_ENOMEM; }
	c->n_ranks = n_ranks; c->rank = rank; c->device = device; c->comm = nullptr;
	ncclUniqueId id;
	memcpy(&id, id128, RXB200_UNIQUE_ID_BYTES);
	RXB_NCCL(nc, nc->CommInitRank(&c->comm, n_ranks, id, rank), delete c);
	*out = c;
	return RXB200_OK;
}

extern "C" int rxb200_comm_create_all(int n_dev, const int *devices, rxb200_comm **out)
{
	if (!out || n_dev < 1 || n_dev > RXB_ROW_PAD) { set_error("bad communicator arguments (1 <= n_dev <= %d)", RXB_ROW_PAD); return RXB200_EINVAL; }
	for (int i = 0; i < n_dev; i++) { out[i] = nullptr; }
	const NcclApi *nc = nccl_api();
	if (!nc) { return RXB200_EUNSUPPORTED; }
	std::vector<ncclComm_t> comms((size_t)n_dev, nullptr);
	std::vector<int> devs((size_t)n_dev);
	for (int i = 0; i < n_dev; i++) { devs[i] = devices ? devices[i] : i; }
	RXB_NCCL(nc, nc->CommInitAll(comms.data(), n_dev, devs.data()), (void)0);
	for (int i = 0; i < n_dev; i++) {
		rxb200_comm *c = new (std::nothrow) rxb200_comm();
		if (!c) {
			for (int j = 0; j < n_dev; j++) { if (j >= i) { nc->CommDestroy(comms[j]); } else { rxb200_comm_destroy(out[j]); out[j] = nullptr; } }
			return RXB200_ENOMEM;
		}
		c->comm = comms[i]; c->n_ranks = n_dev; c->rank = i; c->device = devs[i];
		out[i] = c;
	}
	return RXB200_OK;
}

extern "C" void rxb200_comm_destroy(rxb200_comm *c)
{
	if (!c) { return; }
	const NcclApi *nc = nccl_api();
	if (nc && c->comm) { cudaSetDevice(c->device); nc->CommDestroy(c->comm); }
	delete c;
}

extern "C" int rxb200_comm_size(const rxb200_comm *c) { return c ? c->n_ranks : 0; }
extern "C" int rxb200_comm_rank(const rxb200_comm *c) { return c ? c->rank : -1; }

extern "C" int rxb200_power_shard(int n_hops, int n_ranks, int rank, int *hop_begin, int *hop_end)
{
	if (n_hops < 1 || n_ranks < 1 || rank < 0 || rank >= n_ranks || !hop_begin || !hop_end) { set_error("bad shard arguments"); return RXB200_EINVAL; }
	const int per = (n_hops + n_ranks - 1) / n_ranks;
	*hop_begin = rank * per < n_hops ? rank * per : n_hops;
	*hop_end = (rank + 1) * per < n_hops ? (rank + 1) * per : n_hops;
	return RXB200_OK;
}

// enqueue this rank's part of the collation on the handle's stream (inside a group when several handles of one
// process take part)
static int power_gather_enqueue(const NcclApi *nc, rxb200_power *h, rxb200_comm *c)
{
	const size_t N = (size_t)1 << h->p.bin_e;
	const int per = (h->p.n_hops + c->n_ranks - 1) / c->n_ranks;
	int hb = 0, he = 0;
	rxb200_power_shard(h->p.n_hops, c->n_ranks, c->rank, &hb, &he);
	RXB_CUDA(cudaSetDevice(h->device));
	if (he > hb) {
		RXB_CUDA(cudaMemcpyAsync(h->d_samples + hb, h->samples.data() + hb, (size_t)(he - hb) * sizeof(int), cudaMemcpyHostToDevice, h->stream));
	}
	// in place: this rank's block already sits at rank*per rows from the start of the receive buffer
	RXB_NCCL(nc, nc->AllGather(h->d_avg + (size_t)c->rank * per * N, h->d_avg, (size_t)per * N, ncclInt64, c->comm, h->stream), (void)0);
	RXB_NCCL(nc, nc->AllGather(h->d_samples + (size_t)c->rank * per, h->d_samples, (size_t)per, ncclInt32, c->comm, h->stream), (void)0);
	return RXB200_OK;
}

static int power_gather_finish(rxb200_power *h, int sync)
{
	RXB_CUDA(cudaSetDevice(h->device));
	// the host mirror of `samples` follows the gathered copy (pinned-less D2H of n_hops ints)
	RXB_CUDA(cudaMemcpyAsync(h->samples.data(), h->d_samples, (size_t)h->p.n_hops * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
	if (sync) { RXB_CUDA(cudaStreamSynchronize(h->stream)); }
	return RXB200_OK;
}

static int power_gather_check(const rxb200_power *h, const rxb200_comm *c)
{
	if (!h || !c) { set_error("null argument"); return RXB200_EINVAL; }
	if (c->device != h->device) { set_error("communicator is on device %d, the handle on %d", c->device, h->device); return RXB200_EINVAL; }
	const int per = (h->p.n_hops + c->n_ranks - 1) / c->n_ranks;
	if ((long long)per * c->n_ranks > (long long)h->p.n_hops + RXB_ROW_PAD) { set_error("too many ranks for the row padding"); return RXB200_EINVAL; }
	return RXB200_OK;
}

extern "C" int rxb200_power_gather(rxb200_power *h, rxb200_comm *c, int sync)
{
	int rc = power_gather_check(h, c);
	if (rc != RXB200_OK) { return rc; }
	if (c->n_ranks == 1) { if (sync) { RXB_CUDA(cudaSetDevice(h->device)); RXB_CUDA(cudaStreamSynchronize(h->stream)); } return RXB200_OK; }
	const NcclApi *nc = nccl_api();
	if (!nc) { return RXB200_EUNSUPPORTED; }
	RXB_NCCL(nc, nc->GroupStart(), (void)0);
	rc = power_gather_enqueue(nc, h, c);
	RXB_NCCL(nc, nc->GroupEnd(), (void)0);
	if (rc != RXB200_OK) { return rc; }
	return power_gather_finish(h, sync);
}

// ---- all ranks in ONE process (the C drop-in shell): n_dev handles with identical parameters, one per GPU
struct rxb200_power_group {
	int n_dev;
	std::vector<rxb200_power *> h;
	std::vector<rxb200_comm *> c;
};

extern "C" void rxb200_power_group_destroy(rxb200_power_group *g)
{
	if (!g) { return; }
	for (auto *c : g->c) { rxb200_comm_destroy(c); }
	for (auto *h : g->h) { rxb200_power_destroy(h); }
	delete g;
}

extern "C" int rxb200_power_group_create(const rxb200_power_params *params, const int *window_coefs, const int16_t *sinewave,
                                         int n_dev, const int *devices, rxb200_power_group **out)
{
	if (!out || n_dev < 1 || n_dev > RXB_ROW_PAD) { set_error("bad group arguments (1 <= n_dev <= %d)", RXB_ROW_PAD); return RXB200_EINVAL; }
	*out = nullptr;
	rxb200_power_group *g = new (std::nothrow) rxb200_power_group();
	if (!g) { return RXB200_ENOMEM; }
	g->n_dev = n_dev;
	g->h.assign((size_t)n_dev, nullptr);
	g->c.assign((size_t)n_dev, nullptr);
	for (int i = 0; i < n_dev; i++) {
		int rc = rxb200_power_create(params, window_coefs, sinewave, devices ? devices[i] : i, &g->h[(size_t)i]);
		if (rc != RXB200_OK) { rxb200_power_group_destroy(g); return rc; }
	}
	if (n_dev > 1) {
		int rc = rxb200_comm_create_all(n_dev, devices, g->c.data());
		if (rc != RXB200_OK) { rxb200_power_group_destroy(g); return rc; }
	}
	*out = g;
	return RXB200_OK;
}

extern "C" int rxb200_power_group_size(const rxb200_power_group *g) { return g ? g->n_dev : 0; }
extern "C" rxb200_power *rxb200_power_group_member(rxb200_power_group *g, int i) { return (g && i >= 0 && i < g->n_dev) ? g->h[(size_t)i] : nullptr; }

// hop_bufs as in rxb200_power_accumulate (HOST pointer, [n_pass][hop_end-hop_begin][buf_len]); every member takes the
// hops of the range it owns.  Copies and kernels of the members overlap (one stream per GPU), the call returns when
// all are done.
extern "C" int rxb200_power_group_accumulate(rxb200_power_group *g, const int16_t *hop_bufs, int n_pass, int hop_begin, int hop_end)
{
	if (!g || !hop_bufs) { set_error("null argument"); return RXB200_EINVAL; }
	const rxb200_power_params &p = g->h[0]->p;
	if (n_pass < 0 || hop_begin < 0 || hop_end > p.n_hops || hop_begin >= hop_end) { set_error("bad hop range"); return RXB200_EINVAL; }
	const int nh = hop_end - hop_begin;
	for (int i = 0; i < g->n_dev; i++) {
		int hb, he;
		rxb200_power_shard(p.n_hops, g->n_dev, i, &hb, &he);
		const int b = hb > hop_begin ? hb : hop_begin, e = he < hop_end ? he : hop_end;
		if (b >= e) { continue; }
		rxb200_power *h = g->h[(size_t)i];
		RXB_CUDA(cudaSetDevice(h->device));
		const size_t elems = (size_t)n_pass * (size_t)(e - b) * (size_t)p.buf_len;
		RXB_CUDA(reserve(h->d_in, h->d_in_cap, elems));
		// the member's hops of every pass, packed [n_pass][e-b][buf_len] on its device
		RXB_CUDA(cudaMemcpy2DAsync(h->d_in, (size_t)(e - b) * p.buf_len * sizeof(int16_t),
		                           hop_bufs + (size_t)(b - hop_begin) * p.buf_len, (size_t)nh * p.buf_len * sizeof(int16_t),
		                           (size_t)(e - b) * p.buf_len * sizeof(int16_t), (size_t)n_pass, cudaMemcpyHostToDevice, h->stream));
		int rc = rxb200_power_accumulate_device(h, h->d_in, n_pass, b, e, 0);
		if (rc != RXB200_OK) { return rc; }
	}
	for (int i = 0; i < g->n_dev; i++) {
		RXB_CUDA(cudaSetDevice(g->h[(size_t)i]->device));
		RXB_CUDA(cudaStreamSynchronize(g->h[(size_t)i]->stream));
	}
	return RXB200_OK;
}

// the collation: after it EVERY member holds all rows and samples, so member 0 can be read or reported as if it had
// processed every hop itself
extern "C" int rxb200_power_group_gather(rxb200_power_group *g)
{
	if (!g) { set_error("null argument"); return RXB200_EINVAL; }
	if (g->n_dev == 1) { return RXB200_OK; }
	const NcclApi *nc = nccl_api();
	if (!nc) { return RXB200_EUNSUPPORTED; }
	for (int i = 0; i < g->n_dev; i++) { int rc = power_gather_check(g->h[(size_t)i], g->c[(size_t)i]); if (rc != RXB200_OK) { return rc; } }
	RXB_NCCL(nc, nc->GroupStart(), (void)0);
	int rc = RXB200_OK;
	for (int i = 0; i < g->n_dev && rc == RXB200_OK; i++) { rc = power_gather_enqueue(nc, g->h[(size_t)i], g->c[(size_t)i]); }
	RXB_NCCL(nc, nc->GroupEnd(), (void)0);
	if (rc != RXB200_OK) { return rc; }
	for (int i = 0; i < g->n_dev; i++) { rc = power_gather_finish(g->h[(size_t)i], 1); if (rc != RXB200_OK) { return rc; } }
	return RXB200_OK;
}

extern "C" int rxb200_power_group_reset(rxb200_power_group *g)
{
	if (!g) { return RXB200_EINVAL; }
	for (auto *h : g->h) { int rc = rxb200_power_reset(h); if (rc != RXB200_OK) { return rc; } }
	return RXB200_OK;
}
