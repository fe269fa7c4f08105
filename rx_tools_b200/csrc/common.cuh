// common.cuh — shared helpers of librxb200.so (error plumbing, wrap-safe integer helpers).
#pragma once
#include <cuda.h>               // CUtensorMap (types only: the encoder is reached through cudaGetDriverEntryPoint)
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/rxb200.h"

namespace rxb {

void set_error(const char *fmt, ...);

#define RXB_CUDA(call)                                                                   \
	do {                                                                                 \
		cudaError_t e__ = (call);                                                        \
		if (e__ != cudaSuccess) {                                                        \
			rxb::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__),      \
			               __FILE__, __LINE__);                                          \
			return RXB200_ECUDA;                                                         \
		}                                                                                \
	} while (0)

// same, running `cleanup` first (create paths: nothing may leak when a CUDA call fails half way)
#define RXB_CUDA_OR(call, cleanup)                                                       \
	do {                                                                                 \
		cudaError_t e__ = (call);                                                        \
		if (e__ != cudaSuccess) {                                                        \
			rxb::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__),      \
			               __FILE__, __LINE__);                                          \
			cleanup;                                                                     \
			return RXB200_ECUDA;                                                         \
		}                                                                                \
	} while (0)

// ---- two's-complement helpers: the reference relies on x86 wrap-around for int overflow and
// on truncating stores to int16_t (SURVEY.md §7 hard part 5); unsigned arithmetic makes the
// wrap well-defined here.
__host__ __device__ __forceinline__ int wrap16(int v) { return (int)(int16_t)v; }
__host__ __device__ __forceinline__ int mul_w(int a, int b) { return (int)((unsigned)a * (unsigned)b); }
__host__ __device__ __forceinline__ int add_w(int a, int b) { return (int)((unsigned)a + (unsigned)b); }
__host__ __device__ __forceinline__ int sub_w(int a, int b) { return (int)((unsigned)a - (unsigned)b); }
__host__ __device__ __forceinline__ int neg_w(int a) { return (int)(0u - (unsigned)a); }
// C's truncating division; the two inputs that trap on x86 return a fixed value instead.
__host__ __device__ __forceinline__ int div_c(int n, int d)
{
	if (d == 0) { return 0; }
	if (d == -1) { return neg_w(n); }
	return n / d;
}

// (int16)(x/32767.0*128.0+0.4) for every int16 x, in integer form (src/rtl_fm.c:846; the exact
// identity is checked exhaustively against the oracle in tests/test_host_logic.py and on the GPU
// in tests/test_fm_gpu.py).  Result is in [-127, 128].
__host__ __device__ __forceinline__ int scale_cs16(int x)
{
	// t < 0  <=>  x <= -103  <=>  the real value is negative: floor + 1 == truncation toward zero
	int t = x * 32769 + 3355366;
	return (t >> 23) - (t >> 31);
}

#ifdef __CUDACC__
// C's truncating n / d for d > 0 when |n / d| is small (< 2^20): fp32 estimate (error < 1) and an
// exact integer remainder check.  Falls back to div_c otherwise.  Bit-exact with '/'.
__device__ __forceinline__ int div_small_quotient(int n, int d)
{
	if (d <= 0) { return div_c(n, d); }
	int q = __float2int_rz(__int2float_rn(n) * __frcp_rn(__int2float_rn(d)));
	int r = sub_w(n, mul_w(q, d));           // exact in two's complement whenever |q - n/d| <= 1
	if (n >= 0) {
		if (r < 0) { q--; } else if (r >= d) { q++; }
	} else {
		if (r > 0) { q++; } else if (r <= -d) { q--; }
	}
	return q;
}

// ---- mbarrier / bulk-copy plumbing (shared by the rx_power TMA staging and the rx_fm front/back-end hand-off)
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// bulk TMA: contiguous global -> shared, completion signalled on the mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_load(void *dst, const void *src, uint32_t bytes, uint64_t *bar)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
	             ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// tensor TMA: one box of a 2-D tensor map at element coordinates (c0, c1) -> shared, completion on the mbarrier
__device__ __forceinline__ void tensor_load_2d(void *dst, const CUtensorMap *map, int c0, int c1, uint64_t *bar)
{
	asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
	             ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
	uint32_t ok;
	do {
		asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
		             : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
	} while (!ok);
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// one arrival (release semantics at CTA scope: the arriving thread's earlier shared-memory writes are visible to
// whoever observes the phase complete)
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
	asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
#endif

}  // namespace rxb
