// load_probe.cu -- how fast the row front end's launch shape can stream its input, per load pattern.
//
// The shape of fm_split_kernel on the wbfm workload (fm2b): 2 CTAs per SM, 8 warps each, every warp walking its own
// contiguous stretch of a 1 GiB CS16 buffer in rows of 1024 samples (4 KB, 32 lines of 128 bytes).  The compute is a
// XOR of everything into one word per thread.  Three patterns:
//   a  per-lane line: lane l reads line l of the row as 8 x two 128-bit ld.global.nc.L2::256B, the next row is loaded
//      into registers during the current one, prefetch.global.L2 three rows ahead (the front end before the TMA ring)
//   b  coalesced: each 128-bit load instruction of the warp covers 512 contiguous bytes
//   c  2-D cp.async.bulk.tensor of each row (box 32 lines x 128 B, 128-byte swizzle) into a per-warp ring of S
//      stages, one mbarrier each; lane l reads its line's chunk q at 128 l + 16 (q ^ (l & 7)) (no bank conflicts)
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o load_probe.bin load_probe.cu && ./load_probe.bin
#include <cstdio>
#include <cstdint>
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

constexpr int WARPS = 8, ROW_BYTES = 4096;

__device__ __forceinline__ void ld_pair(const char *p, uint32_t *v)
{
	asm volatile("ld.global.nc.L2::256B.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
	             "ld.global.nc.L2::256B.v4.u32 {%4,%5,%6,%7}, [%8+16];"
	             : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]), "=r"(v[4]), "=r"(v[5]), "=r"(v[6]), "=r"(v[7])
	             : "l"(p));
}

__device__ __forceinline__ void stretch(long long rows, int nwarps, int gw, long long &r0, long long &r1)
{
	const long long per = (rows + nwarps - 1) / nwarps;
	r0 = gw * per; r1 = r0 + per < rows ? r0 + per : rows;
}

// pattern a (COAL 0) and b (COAL 1)
template <int COAL>
__global__ void __launch_bounds__(WARPS * 32, 2) k_ldg(const char *in, long long rows, uint32_t *out)
{
	const int lane = threadIdx.x & 31, gw = blockIdx.x * WARPS + (threadIdx.x >> 5);
	long long r0, r1;
	stretch(rows, gridDim.x * WARPS, gw, r0, r1);
	uint32_t acc = 0, v[32];
	auto load = [&](long long r) {
		const char *row = in + r * ROW_BYTES;
		if (COAL) {
#pragma unroll
			for (int q = 0; q < 8; q++) {
				const uint4 w = __ldg(reinterpret_cast<const uint4 *>(row + 512 * q + 16 * lane));
				v[4 * q] = w.x; v[4 * q + 1] = w.y; v[4 * q + 2] = w.z; v[4 * q + 3] = w.w;
			}
		} else {
#pragma unroll
			for (int q = 0; q < 4; q++) { ld_pair(row + 128 * lane + 32 * q, &v[8 * q]); }
		}
	};
	if (r0 < r1) { load(r0); }
	for (long long r = r0; r < r1; r++) {
		uint32_t x = 0;
#pragma unroll
		for (int j = 0; j < 32; j++) { x ^= v[j] * (2 * j + 1); }
		acc ^= x;
		if (!COAL) {
			const long long pf = r + 3 < r1 ? r + 3 : r1 - 1;
			asm volatile("prefetch.global.L2 [%0];" ::"l"(in + pf * ROW_BYTES + 128 * lane));
		}
		load(r + 1 < r1 ? r + 1 : r);
	}
	out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

__device__ __forceinline__ uint32_t sa(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

template <int S>
__global__ void __launch_bounds__(WARPS * 32, 2) k_tma(const __grid_constant__ CUtensorMap map, long long rows, uint32_t *out)
{
	extern __shared__ uint8_t smem_raw[];
	__shared__ __align__(8) uint64_t bar[WARPS * S];
	const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, gw = blockIdx.x * WARPS + w;
	uint8_t *ring = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023) + w * S * ROW_BYTES;
	uint64_t *b = bar + w * S;
	if (lane < S) {
		asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(sa(b + lane)));
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncwarp();
	long long r0, r1;
	stretch(rows, gridDim.x * WARPS, gw, r0, r1);
	auto issue = [&](long long r) {
		const int s = (int)((r - r0) % S);
		asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sa(b + s)), "r"(ROW_BYTES) : "memory");
		asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
		             ::"r"(sa(ring + s * ROW_BYTES)), "l"(&map), "r"(0), "r"((int)(r * 32)), "r"(sa(b + s)) : "memory");
	};
	if (lane == 0) {
		for (long long r = r0; r < r0 + S && r < r1; r++) { issue(r); }
	}
	uint32_t acc = 0;
	for (long long r = r0; r < r1; r++) {
		const int s = (int)((r - r0) % S);
		const uint32_t par = (uint32_t)(((r - r0) / S) & 1);
		uint32_t done = 0;
		while (!done) {
			asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
			             : "=r"(done) : "r"(sa(b + s)), "r"(par) : "memory");
		}
		uint32_t v[32];
		const uint8_t *line = ring + s * ROW_BYTES + 128 * lane;
#pragma unroll
		for (int q = 0; q < 8; q++) {
			const uint4 x = *reinterpret_cast<const uint4 *>(line + 16 * (q ^ (lane & 7)));
			v[4 * q] = x.x; v[4 * q + 1] = x.y; v[4 * q + 2] = x.z; v[4 * q + 3] = x.w;
		}
		uint32_t x = 0;
#pragma unroll
		for (int j = 0; j < 32; j++) { x ^= v[j] * (2 * j + 1); }
		acc ^= x;
		__syncwarp();                               // every lane has its line: the stage can take row r + S
		if (lane == 0 && r + S < r1) { issue(r + S); }
	}
	out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

__global__ void k_fill(uint32_t *p, size_t n)
{
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) { p[i] = (uint32_t)(i * 2654435761u); }
}

template <typename F>
static float time_ms(F launch, int reps)
{
	cudaEvent_t e0, e1;
	cudaEventCreate(&e0); cudaEventCreate(&e1);
	for (int i = 0; i < 2; i++) { launch(); }
	cudaEventRecord(e0);
	for (int i = 0; i < reps; i++) { launch(); }
	cudaEventRecord(e1);
	cudaEventSynchronize(e1);
	float ms = 0.f;
	cudaEventElapsedTime(&ms, e0, e1);
	cudaEventDestroy(e0); cudaEventDestroy(e1);
	return ms / reps;
}

static uint32_t checksum(const uint32_t *d, int n)
{
	static uint32_t h[1 << 20];
	cudaMemcpy(h, d, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost);
	uint32_t x = 0;
	for (int i = 0; i < n; i++) { x ^= h[i] * (2u * (uint32_t)i + 1u); }
	return x;
}

int main()
{
	const size_t bytes = (size_t)1 << 30;
	const long long rows = (long long)(bytes / ROW_BYTES);
	cudaDeviceProp prop;
	CK(cudaGetDeviceProperties(&prop, 0));
	const int grid = prop.multiProcessorCount * 2;
	char *in; uint32_t *out;
	CK(cudaMalloc(&in, bytes));
	CK(cudaMalloc(&out, (size_t)grid * WARPS * 32 * sizeof(uint32_t)));
	k_fill<<<1024, 256>>>(reinterpret_cast<uint32_t *>(in), bytes / 4);
	CK(cudaDeviceSynchronize());

	PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
	cudaDriverEntryPointQueryResult qr;
	CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", reinterpret_cast<void **>(&encode), cudaEnableDefault, &qr));
	if (!encode || qr != cudaDriverEntryPointSuccess) { printf("no cuTensorMapEncodeTiled\n"); return 1; }
	CUtensorMap map;
	const cuuint64_t dims[2] = {32, (cuuint64_t)(bytes / 128)};   // 32 words x lines
	const cuuint64_t strides[1] = {128};
	const cuuint32_t box[2] = {32, 32}, estr[2] = {1, 1};
	if (encode(&map, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, in, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
	           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
		printf("cuTensorMapEncodeTiled failed\n"); return 1;
	}
	const int reps = 10;
	auto report = [&](const char *name, float ms) { printf("%-44s %8.3f ms  %7.1f GB/s\n", name, ms, bytes / (ms * 1e6)); };
	printf("%s, %d SMs, grid %d x %d threads, %lld rows of %d B\n", prop.name, prop.multiProcessorCount, grid, WARPS * 32, rows, ROW_BYTES);
	report("a per-lane line, 2 x LDG.128 L2::256B + pf", time_ms([&] { k_ldg<0><<<grid, WARPS * 32>>>(in, rows, out); }, reps));
	report("b coalesced LDG.128 (512 B per instruction)", time_ms([&] { k_ldg<1><<<grid, WARPS * 32>>>(in, rows, out); }, reps));
	const int sm2 = WARPS * 2 * ROW_BYTES + 1024, sm3 = WARPS * 3 * ROW_BYTES + 1024;
	CK(cudaFuncSetAttribute(k_tma<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm2));
	CK(cudaFuncSetAttribute(k_tma<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm3));
	report("c TMA 2-D ring, S = 2", time_ms([&] { k_tma<2><<<grid, WARPS * 32, sm2>>>(map, rows, out); }, reps));
	const uint32_t sum_c = checksum(out, grid * WARPS * 32);
	report("c TMA 2-D ring, S = 3", time_ms([&] { k_tma<3><<<grid, WARPS * 32, sm3>>>(map, rows, out); }, reps));
	CK(cudaGetLastError());
	CK(cudaDeviceSynchronize());
	// a and c read the same words into the same registers: the same XOR (checks the swizzled addressing)
	k_ldg<0><<<grid, WARPS * 32>>>(in, rows, out);
	const uint32_t sum_a = checksum(out, grid * WARPS * 32);
	printf("checksum a %08x c %08x: %s\n", sum_a, sum_c, sum_a == sum_c ? "same" : "DIFFERENT");
	cudaFree(in); cudaFree(out);
	return 0;
}
