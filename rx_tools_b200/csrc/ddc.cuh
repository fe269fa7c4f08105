// ddc.cuh — the pieces the two digital down-converters share: fm_ddc_kernel (fm_mix.cu: rx_fm channels, each mixed
// with its integer table) and power_ddc_kernel (power_mix.cu: rx_power hops, each mixed with a phase-accumulator NCO).
// Both stage the capture samples their outputs' windows cover, mix them per channel into shared memory with mix_one,
// and run the T-tap dot product at the emission points only; they differ in the mixer index and the output address.
#pragma once
#include <algorithm>
#include "common.cuh"

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

// The launch shape both kernels take: a.ws staged samples between two outputs' windows (M when T >= M, else T),
// a.ws_m = floor((2^32 - 1) / ws), a.lpo lanes per output (a power of two <= 32) and a.U outputs per CTA.
struct DdcShape {
	int ws;
	unsigned ws_m;
	int U;
	int lpo;
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

// The shape of a launch of n_out > 0 outputs per channel over `groups` grid rows on the current device; *smem receives
// the dynamic shared memory (the reversed taps, the staged and the mixed span) and *bx the CTAs per grid row.
static inline int ddc_shape(int M, int T, long long n_out, int groups, DdcShape *s, size_t *smem, long long *bx)
{
	s->ws = T >= M ? M : T;
	s->ws_m = 0xffffffffu / (unsigned)s->ws;
	s->lpo = 1;
	while (s->lpo < 32 && s->lpo < T) { s->lpo <<= 1; }
	int dev = 0, n_sm = 0;
	RXB_CUDA(cudaGetDevice(&dev));
	RXB_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
	// as many outputs per CTA as the staging room and the reach allow, but at least two CTAs per SM when there is work
	long long U = std::min((long long)(DDC_SPAN - T) / s->ws, (long long)(DDC_REACH - T) / M) + 1;
	const long long ctas = std::max(1ll, (2ll * n_sm + groups - 1) / groups);
	U = std::max(1ll, std::min(U, (n_out + ctas - 1) / ctas));
	s->U = (int)U;
	*smem = ((size_t)T + 2 * ((size_t)(s->U - 1) * s->ws + T)) * sizeof(uint32_t);
	*bx = (n_out + U - 1) / U;
	return RXB200_OK;
}

}  // namespace rxb
