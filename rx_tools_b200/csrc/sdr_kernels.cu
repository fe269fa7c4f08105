// sdr_kernels.cu — rx_sdr's pointwise sample-format conversions (src/rtl_sdr.c:348-391) as one
// bandwidth-bound kernel: 128-bit loads, grid-stride, nothing but the input read and the output written.  The
// per-int16 arithmetic is sdr_cvt.cuh's, shared with the I/Q down-converter's output store.
#include "common.cuh"
#include "sdr_cvt.cuh"

namespace rxb {

__global__ void __launch_bounds__(256) sdr_convert_kernel(int kind, const uint8_t *__restrict__ src, size_t n_elems,
                                                          uint8_t *__restrict__ dst)
{
	const size_t stride = (size_t)gridDim.x * blockDim.x;
	size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (kind == RXB200_CVT_CS12_CS16) {
		// one complex element = 3 bytes b0 b1 b2 -> I = (b1 << 12) | (b0 << 4), Q = (b2 << 8) | (b1 & 0xf0), as int16
		for (; i < n_elems; i += stride) {
			unsigned b0 = src[3 * i], b1 = src[3 * i + 1], b2 = src[3 * i + 2];
			uint32_t iq = (((b1 << 12) | (b0 << 4)) & 0xffffu) | ((((b2 << 8) | (b1 & 0xf0u)) & 0xffffu) << 16);
			reinterpret_cast<uint32_t *>(dst)[i] = iq;
		}
		return;
	}
	// CS16 input: 4 complex elements (16 bytes) per step
	const uint4 *s4 = reinterpret_cast<const uint4 *>(src);
	const size_t n4 = n_elems / 4;
	for (; i < n4; i += stride) {
		uint4 v = __ldg(s4 + i);
		uint32_t w[4] = {v.x, v.y, v.z, v.w};
		if (kind == RXB200_CVT_CS16_CF32) {
			float4 o0, o1;
			o0.x = sdr_f32((int16_t)(w[0] & 0xffffu)); o0.y = sdr_f32((int16_t)(w[0] >> 16));
			o0.z = sdr_f32((int16_t)(w[1] & 0xffffu)); o0.w = sdr_f32((int16_t)(w[1] >> 16));
			o1.x = sdr_f32((int16_t)(w[2] & 0xffffu)); o1.y = sdr_f32((int16_t)(w[2] >> 16));
			o1.z = sdr_f32((int16_t)(w[3] & 0xffffu)); o1.w = sdr_f32((int16_t)(w[3] >> 16));
			reinterpret_cast<float4 *>(dst)[2 * i] = o0;
			reinterpret_cast<float4 *>(dst)[2 * i + 1] = o1;
		} else {
			uint32_t o[2] = {0u, 0u};
#pragma unroll
			for (int q = 0; q < 4; q++) {
				int a = (int)(int16_t)(w[q] & 0xffffu), b = (int)(int16_t)(w[q] >> 16);
				int ya = kind == RXB200_CVT_CS16_CS8 ? sdr_byte<RXB200_CVT_CS16_CS8>(a) : sdr_byte<RXB200_CVT_CS16_CU8>(a);
				int yb = kind == RXB200_CVT_CS16_CS8 ? sdr_byte<RXB200_CVT_CS16_CS8>(b) : sdr_byte<RXB200_CVT_CS16_CU8>(b);
				o[q >> 1] |= ((uint32_t)(ya & 0xff) | ((uint32_t)(yb & 0xff) << 8)) << (16 * (q & 1));
			}
			reinterpret_cast<uint2 *>(dst)[i] = make_uint2(o[0], o[1]);
		}
	}
	// tail (n_elems not a multiple of 4)
	const size_t done = n4 * 4;
	for (size_t e = done + (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_elems; e += stride) {
		uint32_t w = reinterpret_cast<const uint32_t *>(src)[e];
		int a = (int)(int16_t)(w & 0xffffu), b = (int)(int16_t)(w >> 16);
		if (kind == RXB200_CVT_CS16_CF32) {
			reinterpret_cast<float2 *>(dst)[e] = make_float2(sdr_f32(a), sdr_f32(b));
		} else {
			int ya = kind == RXB200_CVT_CS16_CS8 ? sdr_byte<RXB200_CVT_CS16_CS8>(a) : sdr_byte<RXB200_CVT_CS16_CU8>(a);
			int yb = kind == RXB200_CVT_CS16_CS8 ? sdr_byte<RXB200_CVT_CS16_CS8>(b) : sdr_byte<RXB200_CVT_CS16_CU8>(b);
			dst[2 * e] = (uint8_t)ya; dst[2 * e + 1] = (uint8_t)yb;
		}
	}
}

}  // namespace rxb
using namespace rxb;

static size_t in_bytes(int kind, size_t n) { return kind == RXB200_CVT_CS12_CS16 ? 3 * n : 4 * n; }
static size_t out_bytes(int kind, size_t n) { return kind == RXB200_CVT_CS16_CF32 ? 8 * n : (kind == RXB200_CVT_CS12_CS16 ? 4 * n : 2 * n); }

extern "C" int rxb200_sdr_convert_device(int kind, const void *d_src, size_t n_elems, void *d_dst, void *stream)
{
	if (kind < 0 || kind > 3 || !d_src || !d_dst) { set_error("bad convert request"); return RXB200_EINVAL; }
	// the CS12 unpack reads bytes and stores one 32-bit word per element; the CS16 kinds move 16-byte vectors
	if (kind == RXB200_CVT_CS12_CS16 && ((uintptr_t)d_dst & 3u)) { set_error("CS12 d_dst must be 4-byte aligned"); return RXB200_EINVAL; }
	if (kind != RXB200_CVT_CS12_CS16 && (((uintptr_t)d_src & 15u) || ((uintptr_t)d_dst & 15u))) { set_error("pointers must be 16-byte aligned"); return RXB200_EINVAL; }
	if (n_elems == 0) { return RXB200_OK; }
	int dev = 0, sm = 132;
	cudaGetDevice(&dev);
	cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, dev);
	size_t want = (n_elems / 4 + 255) / 256;
	unsigned blocks = (unsigned)(want < (size_t)sm * 8 ? (want ? want : 1) : (size_t)sm * 8);
	sdr_convert_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(kind, (const uint8_t *)d_src, n_elems, (uint8_t *)d_dst);
	RXB_CUDA(cudaGetLastError());
	return RXB200_OK;
}

extern "C" int rxb200_sdr_convert(int kind, const void *src, size_t n_elems, void *dst, int device)
{
	if (kind < 0 || kind > 3 || !src || !dst) { set_error("bad convert request"); return RXB200_EINVAL; }
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { set_error("no CUDA device: librxb200 has no CPU fallback"); return RXB200_ENODEV; }
	if (device < 0 || device >= ndev) { set_error("device %d out of range", device); return RXB200_ENODEV; }
	if (n_elems == 0) { return RXB200_OK; }
	RXB_CUDA(cudaSetDevice(device));
	void *d_in = nullptr, *d_out = nullptr;
	RXB_CUDA(cudaMalloc(&d_in, in_bytes(kind, n_elems) + 16));
	if (cudaMalloc(&d_out, out_bytes(kind, n_elems) + 16) != cudaSuccess) { cudaFree(d_in); set_error("cudaMalloc"); return RXB200_ENOMEM; }
	int rc = RXB200_OK;
	if (cudaMemcpy(d_in, src, in_bytes(kind, n_elems), cudaMemcpyHostToDevice) != cudaSuccess) { rc = RXB200_ECUDA; }
	if (rc == RXB200_OK) { rc = rxb200_sdr_convert_device(kind, d_in, n_elems, d_out, nullptr); }
	if (rc == RXB200_OK && cudaMemcpy(dst, d_out, out_bytes(kind, n_elems), cudaMemcpyDeviceToHost) != cudaSuccess) { rc = RXB200_ECUDA; }
	if (rc == RXB200_ECUDA) { set_error("cuda copy failed: %s", cudaGetErrorString(cudaGetLastError())); }
	cudaFree(d_in); cudaFree(d_out);
	return rc;
}
