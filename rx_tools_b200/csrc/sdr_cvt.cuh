// sdr_cvt.cuh — rx_sdr's conversion of one CS16 int16 (src/rtl_sdr.c:367-386; include/rxb200.h, "rx_sdr"), the one
// copy of that arithmetic: sdr_convert_kernel (sdr_kernels.cu) converts buffers with it, and the I/Q down-converter's
// output store (ddc.cuh, SdrOut) converts each output word with it as it writes the recorded format.
#pragma once
#include "common.cuh"

namespace rxb {

// (x/32767.0*128.0 + 127.4) truncated: same identity as scale_cs16 with the bias moved by 127
// (checked for all 65 536 inputs against the oracle in tests/test_sdr_gpu.py); result 0..255.
__device__ __forceinline__ int scale_cu8(int x)
{
	int t = x * 32769 + 3355366 + 127 * 8388608;     // negative only for x <= -32614: truncation gives 0 there
	return (t >> 23) - (t >> 31);
}

// one int16 x to its CS8 (K = RXB200_CVT_CS16_CS8) or CU8 (K = RXB200_CVT_CS16_CU8) byte, in the low 8 bits: the fp64
// rule (int)(x/32767.0*128.0+0.4), resp. +127.4, in its exact integer form
template <int K>
__device__ __forceinline__ int sdr_byte(int x) { return K == RXB200_CVT_CS16_CS8 ? scale_cs16(x) : scale_cu8(x); }

// one int16 x (exact in fp32) to CF32: x * 1.0f / SHRT_MAX, correctly rounded
__device__ __forceinline__ float sdr_f32(float x) { return __fdiv_rn(x, 32767.0f); }

// bytes of one complex output in format fmt (RXB200_SDR_OUT_CS16 or a CS16 conversion), 0 for any other value
__host__ __device__ __forceinline__ int sdr_elem_bytes(int fmt)
{
	return fmt == RXB200_SDR_OUT_CS16 ? 4 : fmt == RXB200_CVT_CS16_CF32 ? 8
	     : (fmt == RXB200_CVT_CS16_CS8 || fmt == RXB200_CVT_CS16_CU8) ? 2 : 0;
}

// the int16 pair w (I low, Q high) as complex element i of a row of format F at base: a 32-bit store for CS16, one
// 16-bit store for CS8 and CU8, two 32-bit stores for CF32, so base needs only min(element, 4)-byte alignment
template <int F>
__device__ __forceinline__ void sdr_put(void *base, long long i, uint32_t w)
{
	const int a = (int)(int16_t)(w & 0xffffu), b = (int)(int16_t)(w >> 16);
	if (F == RXB200_SDR_OUT_CS16) {
		static_cast<uint32_t *>(base)[i] = w;
	} else if (F == RXB200_CVT_CS16_CF32) {
		float *p = static_cast<float *>(base) + 2 * i;
		p[0] = sdr_f32(a);
		p[1] = sdr_f32(b);
	} else {
		static_cast<uint16_t *>(base)[i] = (uint16_t)((sdr_byte<F>(a) & 0xff) | ((sdr_byte<F>(b) & 0xff) << 8));
	}
}

}  // namespace rxb
