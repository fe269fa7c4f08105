// sdr_kernels.cu — rx_sdr's pointwise sample-format conversions (src/rtl_sdr.c:348-391) as one
// bandwidth-bound kernel: 128-bit loads, grid-stride, nothing but the input read and the output written.  The
// per-int16 arithmetic is sdr_cvt.cuh's, shared with the I/Q down-converter's output store.  The widening kinds (CS12,
// CS8, CU8 to CS16) are also the capture handles' input stage (input_stage.cuh, widen_launch below).
#include "common.cuh"
#include "input_stage.cuh"
#include "sdr_cvt.cuh"

namespace rxb {

// one CS12 element, 3 bytes b0 b1 b2 -> I = (b1 << 12) | (b0 << 4), Q = (b2 << 8) | (b1 & 0xf0), as the int16 pair word
__device__ __forceinline__ uint32_t widen_cs12(unsigned b0, unsigned b1, unsigned b2)
{
	return (((b1 << 12) | (b0 << 4)) & 0xffffu) | ((((b2 << 8) | (b1 & 0xf0u)) & 0xffffu) << 16);
}

// the CS8 elements in bytes 0-1 (sel 0x1404) or 2-3 (sel 0x3424) of x as the int16 pair word: each byte b to b << 8,
// which is (int16)((int8)b << 8); CU8 flips each byte's top bit first, (b - 128) mod 256, so ((b - 128) << 8)
__device__ __forceinline__ uint32_t widen_8(uint32_t x, unsigned sel, uint32_t flip) { return __byte_perm(x, 0u, sel) ^ flip; }

__global__ void __launch_bounds__(256) sdr_convert_kernel(int kind, const uint8_t *__restrict__ src, size_t n_elems,
                                                          uint8_t *__restrict__ dst)
{
	const size_t stride = (size_t)gridDim.x * blockDim.x;
	size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	// the widening kinds move 16-byte vectors when src and dst are 16-byte aligned, else bytes in and one word out per
	// element; both cover every element from `done` on
	const bool vec = (((uintptr_t)src | (uintptr_t)dst) & 15u) == 0;
	uint32_t *d32 = reinterpret_cast<uint32_t *>(dst);
	if (kind == RXB200_CVT_CS12_CS16) {
		size_t done = 0;
		if (vec) {                                 // 16 elements: 48 bytes in, 64 out
			const uint4 *s4 = reinterpret_cast<const uint4 *>(src);
			const size_t n16 = n_elems / 16;
			for (size_t u = i; u < n16; u += stride) {
				uint32_t w[12];
#pragma unroll
				for (int q = 0; q < 3; q++) {
					const uint4 v = __ldg(s4 + 3 * u + q);
					w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w;
				}
				uint32_t o[16];
#pragma unroll
				for (int e = 0; e < 16; e++) {
					const int k = 3 * e;
					o[e] = widen_cs12((w[k >> 2] >> (8 * (k & 3))) & 0xffu, (w[(k + 1) >> 2] >> (8 * ((k + 1) & 3))) & 0xffu,
					                  (w[(k + 2) >> 2] >> (8 * ((k + 2) & 3))) & 0xffu);
				}
				uint4 *d4 = reinterpret_cast<uint4 *>(dst) + 4 * u;
#pragma unroll
				for (int q = 0; q < 4; q++) { d4[q] = make_uint4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]); }
			}
			done = n16 * 16;
		}
		for (size_t e = done + i; e < n_elems; e += stride) { d32[e] = widen_cs12(src[3 * e], src[3 * e + 1], src[3 * e + 2]); }
		return;
	}
	if (kind == RXB200_CVT_CS8_CS16 || kind == RXB200_CVT_CU8_CS16) {
		const uint32_t flip = kind == RXB200_CVT_CU8_CS16 ? 0x80008000u : 0u;
		size_t done = 0;
		if (vec) {                                 // 8 elements: 16 bytes in, 32 out
			const uint4 *s4 = reinterpret_cast<const uint4 *>(src);
			uint4 *d4 = reinterpret_cast<uint4 *>(dst);
			const size_t n8 = n_elems / 8;
			for (size_t u = i; u < n8; u += stride) {
				const uint4 v = __ldg(s4 + u);
				d4[2 * u] = make_uint4(widen_8(v.x, 0x1404u, flip), widen_8(v.x, 0x3424u, flip), widen_8(v.y, 0x1404u, flip),
				                       widen_8(v.y, 0x3424u, flip));
				d4[2 * u + 1] = make_uint4(widen_8(v.z, 0x1404u, flip), widen_8(v.z, 0x3424u, flip),
				                           widen_8(v.w, 0x1404u, flip), widen_8(v.w, 0x3424u, flip));
			}
			done = n8 * 8;
		}
		for (size_t e = done + i; e < n_elems; e += stride) {
			d32[e] = widen_8((uint32_t)src[2 * e] | ((uint32_t)src[2 * e + 1] << 8), 0x1404u, flip);
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

static bool widening(int kind)
{
	return kind == RXB200_CVT_CS12_CS16 || kind == RXB200_CVT_CS8_CS16 || kind == RXB200_CVT_CU8_CS16;
}
static bool good_kind(int kind) { return (kind >= RXB200_CVT_CS16_CS8 && kind <= RXB200_CVT_CS12_CS16) || widening(kind); }
static size_t in_bytes(int kind, size_t n)
{
	return kind == RXB200_CVT_CS12_CS16 ? 3 * n : (kind == RXB200_CVT_CS8_CS16 || kind == RXB200_CVT_CU8_CS16) ? 2 * n : 4 * n;
}
static size_t out_bytes(int kind, size_t n) { return kind == RXB200_CVT_CS16_CF32 ? 8 * n : widening(kind) ? 4 * n : 2 * n; }

// the launch of every convert: a grid of at most 8 CTAs per SM over n_elems / 4 threads' worth of elements
static int convert_launch(int kind, const void *d_src, size_t n_elems, void *d_dst, cudaStream_t st)
{
	int dev = 0, sm = 132;
	cudaGetDevice(&dev);
	cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, dev);
	size_t want = (n_elems / 4 + 255) / 256;
	unsigned blocks = (unsigned)(want < (size_t)sm * 8 ? (want ? want : 1) : (size_t)sm * 8);
	sdr_convert_kernel<<<blocks, 256, 0, st>>>(kind, (const uint8_t *)d_src, n_elems, (uint8_t *)d_dst);
	RXB_CUDA(cudaGetLastError());
	return RXB200_OK;
}

extern "C" int rxb200_sdr_convert_device(int kind, const void *d_src, size_t n_elems, void *d_dst, void *stream)
{
	if (!good_kind(kind) || !d_src || !d_dst) { set_error("bad convert request"); return RXB200_EINVAL; }
	// the widening kinds read bytes (16-byte vectors when both pointers allow) and store one 32-bit word per element;
	// the CS16 kinds move 16-byte vectors
	if (widening(kind) && ((uintptr_t)d_dst & 3u)) { set_error("widening d_dst must be 4-byte aligned"); return RXB200_EINVAL; }
	if (!widening(kind) && (((uintptr_t)d_src & 15u) || ((uintptr_t)d_dst & 15u))) { set_error("pointers must be 16-byte aligned"); return RXB200_EINVAL; }
	if (n_elems == 0) { return RXB200_OK; }
	return convert_launch(kind, d_src, n_elems, d_dst, (cudaStream_t)stream);
}

namespace rxb {

int InputStage::set(int in_fmt)
{
	if (in_fmt < RXB200_IN_CS16 || in_fmt > RXB200_IN_CS12) {
		set_error("input format %d: need RXB200_IN_CS16, _CS8, _CU8 or _CS12", in_fmt);
		return RXB200_EINVAL;
	}
	fmt = in_fmt;
	return RXB200_OK;
}

int InputStage::run(const void *src, size_t c, cudaStream_t st, const uint32_t **out)
{
	if (fmt == RXB200_IN_CS16 || c == 0) { *out = static_cast<const uint32_t *>(src); return RXB200_OK; }
	RXB_CUDA(reserve(d_w, w_cap, c));
	const int kind = fmt == RXB200_IN_CS8 ? RXB200_CVT_CS8_CS16 : fmt == RXB200_IN_CU8 ? RXB200_CVT_CU8_CS16
	                                                                                     : RXB200_CVT_CS12_CS16;
	const int rc = convert_launch(kind, src, c, d_w, st);
	if (rc != RXB200_OK) { return rc; }
	*out = d_w;
	return RXB200_OK;
}

void InputStage::release()
{
	cudaFree(d_w);
	d_w = nullptr;
	w_cap = 0;
}

}  // namespace rxb

extern "C" int rxb200_sdr_convert(int kind, const void *src, size_t n_elems, void *dst, int device)
{
	if (!good_kind(kind) || !src || !dst) { set_error("bad convert request"); return RXB200_EINVAL; }
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
