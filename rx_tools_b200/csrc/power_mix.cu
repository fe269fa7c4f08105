// power_mix.cu — every hop of an rx_power sweep from one wideband capture (include/rxb200.h, "rx_power hops of one
// capture").  power_ddc_kernel mixes the capture to baseband once per hop with a phase-accumulator NCO, filters and
// decimates it, and writes each hop's outputs straight into the pass-major hop buffers ([pass][hop][buf_len]) that
// rxb200_power_accumulate_device reads; the member rxb200_power handle then accumulates them on its own stream.  The
// handle carries the sample count (the NCO phases) and the capture's last T - 1 samples between calls.
#include <math.h>
#include <algorithm>
#include <cstring>
#include <new>
#include <vector>
#include "common.cuh"
#include "ddc.cuh"

namespace rxb {

#define NCO_ENTRIES 65536            // the shared table: index j = ((theta + 2^15) mod 2^32) >> 16

struct PowDdcArgs {
	const uint32_t *src;             // the call's capture, one word per complex sample
	const uint32_t *hist;            // the T - 1 raw capture samples before src
	long long n_out;                 // outputs per hop
	long long r0;                    // src index of the first emission point
	unsigned long long pos;          // capture sample index of src[0]: its NCO phase is pos * w mod 2^32
	uint32_t *dst;                   // hop c, call output u at (u / B) * n_ch * B + c * B + u mod B, one word per output
	int B;                           // outputs per hop buffer (buf_len / 2)
	const int32_t *taps;             // reversed: taps[t] = h[T - 1 - t]
	const int2 *nco;                 // NCO_ENTRIES (c, s) pairs
	const uint32_t *w;               // each hop's frequency word
	int n_ch, M, T, S;
	int ws;                          // staged samples between two outputs' windows: M when T >= M, else T
	unsigned ws_m;                   // floor((2^32 - 1) / ws)
	int U;                           // outputs per CTA
	int lpo;                         // lanes per output (a power of two <= 32)
};

// fm_ddc_kernel with two changes: sample n of hop c is mixed with NCO entry ((n w_c + 2^15) mod 2^32) >> 16, the phase
// taken per CTA and hop as (uint32)g0 * w and stepped by off * w in uint32 arithmetic; and outputs go to the
// pass-major hop buffers.  Acc as there: int when sum |h| * 32768 + 2^(S-1) < 2^31, else long long.
template <typename Acc>
__global__ void __launch_bounds__(DDC_THREADS) power_ddc_kernel(const PowDdcArgs a)
{
	extern __shared__ int4 ddc_smem[];
	const int T = a.T;
	const int room = (a.U - 1) * a.ws + T;
	int32_t *s_h = reinterpret_cast<int32_t *>(ddc_smem);
	uint32_t *s_x = reinterpret_cast<uint32_t *>(s_h + T);
	uint32_t *s_z = s_x + room;
	const int c0 = (int)blockIdx.y * MIX_GROUP;
	const int nc = min(MIX_GROUP, a.n_ch - c0);
	const long long u0 = (long long)blockIdx.x * a.U;
	const int U = (int)min((long long)a.U, a.n_out - u0);
	const int n = (U - 1) * a.ws + T;
	const long long b0 = u0 * a.M + a.r0 - (T - 1);       // src index of the first staged sample, >= -(T - 1)
	// its capture index (< 0 only for the zero samples before create or reset, which mix to zero at any phase)
	const uint32_t g0 = (uint32_t)(unsigned long long)((long long)a.pos + b0);
	for (int j = threadIdx.x; j < T; j += blockDim.x) { s_h[j] = a.taps[j]; }
	for (int s = threadIdx.x; s < n; s += blockDim.x) {
		const long long i = b0 + ddc_off(s, a);
		s_x[s] = i >= 0 ? __ldg(a.src + i) : a.hist[(T - 1) + i];
	}
	__syncthreads();
	const int lane = (int)threadIdx.x & (a.lpo - 1), sub = (int)threadIdx.x / a.lpo, n_sub = (int)blockDim.x / a.lpo;
	const long long q0 = u0 / a.B;                           // the pass of the CTA's first output and its place in it
	const int rb = (int)(u0 - q0 * a.B);
	const long long pass_words = (long long)a.n_ch * a.B;
	for (int c = 0; c < nc; c++) {
		const uint32_t w = __ldg(a.w + c0 + c);
		const uint32_t th0 = g0 * w;
		for (int s = threadIdx.x; s < n; s += blockDim.x) {
			const uint32_t th = th0 + (uint32_t)ddc_off(s, a) * w;
			s_z[s] = mix_one(s_x[s], __ldg(a.nco + ((th + 32768u) >> 16)));
		}
		__syncthreads();
		uint32_t *row = a.dst + q0 * pass_words + (long long)(c0 + c) * a.B;
		for (int ub = 0; ub < U; ub += n_sub) {                  // the same trip count on every lane of a warp
			const int u = ub + sub;
			Acc ai = 0, aq = 0;
			if (u < U) {
				const uint32_t *z = s_z + u * a.ws;
				for (int j = lane; j < T; j += a.lpo) {
					const uint32_t x = z[j];
					const Acc h = (Acc)s_h[j];
					ai += h * (Acc)(int16_t)(x & 0xffffu);
					aq += h * (Acc)(int16_t)(x >> 16);
				}
			}
			for (int o = a.lpo >> 1; o > 0; o >>= 1) {
				ai += __shfl_xor_sync(0xffffffffu, ai, o);
				aq += __shfl_xor_sync(0xffffffffu, aq, o);
			}
			if (u < U && lane == 0) {
				const int r = rb + u, q = r / a.B;               // rb + u < B + DDC_SPAN
				row[q * pass_words + (r - q * a.B)] = ((uint32_t)ddc_out(ai, a.S) & 0xffffu) | ((uint32_t)ddc_out(aq, a.S) << 16);
			}
		}
		__syncthreads();                    // every output of this hop is made before s_z is overwritten
	}
}

// Launches power_ddc_kernel on the current device for a.n_out > 0 outputs per hop; fills a's launch shape
static int power_ddc_launch(PowDdcArgs a, bool wide, cudaStream_t st)
{
	const int groups = (a.n_ch + MIX_GROUP - 1) / MIX_GROUP;
	DdcShape sh;
	size_t smem = 0;
	long long bx = 0;
	const int rc = ddc_shape(a.M, a.T, a.n_out, groups, &sh, &smem, &bx);
	if (rc != RXB200_OK) { return rc; }
	a.ws = sh.ws; a.ws_m = sh.ws_m; a.U = sh.U; a.lpo = sh.lpo;
	void (*kern)(const PowDdcArgs) = wide ? power_ddc_kernel<long long> : power_ddc_kernel<int>;
	RXB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
	kern<<<dim3((unsigned)bx, (unsigned)groups), DDC_THREADS, smem, st>>>(a);
	RXB_CUDA(cudaGetLastError());
	return RXB200_OK;
}

// w = floor((f 2^32 + floor(R/2)) / R) mod 2^32, exactly: |f| < R/2 <= 2^30, so the numerator fits 63 bits
static int nco_words(int capture_rate, const int *offsets_hz, int n, std::vector<uint32_t> &w)
{
	const long long R = capture_rate;
	if (R <= 0) { set_error("capture_rate %d must be > 0", capture_rate); return RXB200_EINVAL; }
	w.resize((size_t)std::max(n, 0));
	for (int i = 0; i < n; i++) {
		const long long f = offsets_hz[i];
		if (2 * (f < 0 ? -f : f) >= R) {
			set_error("hop %d: offset %lld needs |offset| < capture_rate/2 (%lld)", i, f, R);
			return RXB200_EINVAL;
		}
		const long long num = f * (1ll << 32) + R / 2;
		long long q = num / R;
		if (num % R != 0 && num < 0) { q--; }             // C truncates toward zero; the rule floors
		w[(size_t)i] = (uint32_t)(unsigned long long)q;
	}
	return RXB200_OK;
}

}  // namespace rxb

using namespace rxb;

extern "C" int rxb200_nco_table(int32_t *table)
{
	if (!table) { set_error("null argument"); return RXB200_EINVAL; }
	for (int j = 0; j < NCO_ENTRIES; j++) {
		const int jr = j > NCO_ENTRIES / 2 ? j - NCO_ENTRIES : j;   // (-32768, 32768]: j and 65536 - j are conjugates
		const double t = -2.0 * M_PI * (double)jr / (double)NCO_ENTRIES;
		table[2 * j] = (int32_t)round(32768.0 * cos(t));
		table[2 * j + 1] = (int32_t)round(32768.0 * sin(t));
	}
	return RXB200_OK;
}

struct rxb200_power_mix {
	rxb200_power *h = nullptr;                   // the member: accumulators, report, path, stream
	int device = 0;
	int n_hops = 0, buf_len = 0;
	bool wide = false;                           // the kernel accumulates in 64 bits
	int decim = 1, n_taps = 1, shift = 0;
	int32_t *d_taps = nullptr;                   // reversed
	uint32_t *d_w = nullptr;                     // each hop's frequency word
	int2 *d_nco = nullptr;                       // the shared NCO table
	int16_t *d_hist[2] = {nullptr, nullptr};     // the raw capture's last T - 1 samples before pos (zero before 0)
	int cur_hist = 0;                            // d_hist[cur_hist] is the live one, the other the next group's
	unsigned long long pos = 0;                  // capture samples since create or reset (whole passes)
	int16_t *d_cap = nullptr; size_t cap_cap = 0;     // host calls: the capture (int16 elements)
	int16_t *d_bufs = nullptr; size_t bufs_cap = 0;   // the hop buffers of one group of passes, [P][n_hops][buf_len]
	std::vector<cudaEvent_t> ev;                 // pairs around each DDC launch of the last call
	int n_ev = 0;                                // pairs recorded by the last call
};

extern "C" void rxb200_power_mix_destroy(rxb200_power_mix *m)
{
	if (!m) { return; }
	rxb200_power_destroy(m->h);                  // synchronises the stream the DDC runs on
	cudaSetDevice(m->device);
	cudaFree(m->d_taps); cudaFree(m->d_w); cudaFree(m->d_nco); cudaFree(m->d_hist[0]); cudaFree(m->d_hist[1]);
	cudaFree(m->d_cap); cudaFree(m->d_bufs);
	for (cudaEvent_t e : m->ev) { cudaEventDestroy(e); }
	delete m;
}

extern "C" int rxb200_power_mix_create(const rxb200_power_params *params, const int *window_coefs,
                                       const int16_t *sinewave, int capture_rate, const int *offsets_hz,
                                       const rxb200_ddc *ddc, int device, rxb200_power_mix **out)
{
	if (!params || !out || !offsets_hz) { set_error("null argument"); return RXB200_EINVAL; }
	*out = nullptr;
	std::vector<uint32_t> w;
	int rc = nco_words(capture_rate, offsets_hz, params->n_hops, w);
	if (rc != RXB200_OK) { return rc; }
	bool wide = false;
	rc = ddc_check(ddc, &wide);
	if (rc != RXB200_OK) { return rc; }
	rxb200_power_mix *m = new (std::nothrow) rxb200_power_mix();
	if (!m) { return RXB200_ENOMEM; }
	rc = rxb200_power_create(params, window_coefs, sinewave, device, &m->h);   // its params refusals precede any device work
	if (rc != RXB200_OK) { delete m; return rc; }
	m->device = device;
	m->n_hops = params->n_hops; m->buf_len = params->buf_len;
	m->wide = wide;
	m->decim = ddc->decim; m->n_taps = ddc->n_taps; m->shift = ddc->shift;
	const size_t T = (size_t)ddc->n_taps, hist_bytes = std::max<size_t>(1, T - 1) * 2 * sizeof(int16_t);
	std::vector<int32_t> rev(ddc->taps, ddc->taps + T), nco(2 * NCO_ENTRIES);
	std::reverse(rev.begin(), rev.end());
	rxb200_nco_table(nco.data());
	RXB_CUDA_OR(cudaSetDevice(device), rxb200_power_mix_destroy(m));
	RXB_CUDA_OR(cudaMalloc(&m->d_taps, T * sizeof(int32_t)), rxb200_power_mix_destroy(m));
	RXB_CUDA_OR(cudaMalloc(&m->d_w, w.size() * sizeof(uint32_t)), rxb200_power_mix_destroy(m));
	RXB_CUDA_OR(cudaMalloc(&m->d_nco, nco.size() * sizeof(int32_t)), rxb200_power_mix_destroy(m));
	RXB_CUDA_OR(cudaMemcpy(m->d_taps, rev.data(), T * sizeof(int32_t), cudaMemcpyHostToDevice), rxb200_power_mix_destroy(m));
	RXB_CUDA_OR(cudaMemcpy(m->d_w, w.data(), w.size() * sizeof(uint32_t), cudaMemcpyHostToDevice), rxb200_power_mix_destroy(m));
	RXB_CUDA_OR(cudaMemcpy(m->d_nco, nco.data(), nco.size() * sizeof(int32_t), cudaMemcpyHostToDevice), rxb200_power_mix_destroy(m));
	for (int i = 0; i < 2; i++) {
		RXB_CUDA_OR(cudaMalloc(&m->d_hist[i], hist_bytes), rxb200_power_mix_destroy(m));
		RXB_CUDA_OR(cudaMemset(m->d_hist[i], 0, hist_bytes), rxb200_power_mix_destroy(m));
	}
	*out = m;
	return RXB200_OK;
}

extern "C" rxb200_power *rxb200_power_mix_member(rxb200_power_mix *m) { return m ? m->h : nullptr; }

extern "C" int rxb200_power_mix_reset(rxb200_power_mix *m)
{
	if (!m) { return RXB200_EINVAL; }
	const int rc = rxb200_power_reset(m->h);
	if (rc != RXB200_OK) { return rc; }
	// behind any call still running on the member's stream
	const cudaStream_t st = (cudaStream_t)rxb200_power_stream(m->h);
	const size_t hist_bytes = std::max<size_t>(1, (size_t)m->n_taps - 1) * 2 * sizeof(int16_t);
	RXB_CUDA(cudaSetDevice(m->device));
	RXB_CUDA(cudaMemsetAsync(m->d_hist[0], 0, hist_bytes, st));
	RXB_CUDA(cudaMemsetAsync(m->d_hist[1], 0, hist_bytes, st));
	m->cur_hist = 0;
	m->pos = 0;
	return RXB200_OK;
}

namespace {

// The next history: the last T - 1 samples of (history, the group's c capture samples at src), into the spare buffer
int hist_carry(rxb200_power_mix *m, const int16_t *src, size_t c, cudaStream_t st)
{
	const size_t H = (size_t)m->n_taps - 1, w = 2 * sizeof(int16_t);
	if (H == 0) { return RXB200_OK; }
	const int16_t *old = m->d_hist[m->cur_hist];
	int16_t *next = m->d_hist[m->cur_hist ^ 1];
	if (c >= H) {
		RXB_CUDA(cudaMemcpyAsync(next, src + 2 * (c - H), H * w, cudaMemcpyDeviceToDevice, st));
	} else {
		RXB_CUDA(cudaMemcpyAsync(next, old + 2 * c, (H - c) * w, cudaMemcpyDeviceToDevice, st));
		RXB_CUDA(cudaMemcpyAsync(next + 2 * (H - c), src, c * w, cudaMemcpyDeviceToDevice, st));
	}
	m->cur_hist ^= 1;
	return RXB200_OK;
}

// One call of either entry point: the capture's passes in groups of at most RXB200_POWER_MIX_SCRATCH_BYTES of hop
// buffers, each group one DDC launch into the scratch buffer and one accumulate of the member.  device: cs16 is a device
// pointer, else a host pointer staged through the handle's buffer.
int power_mix_call(rxb200_power_mix *m, const int16_t *cs16, size_t n_int16, bool device, int sync)
{
	if (!m || !cs16) { set_error("null argument"); return RXB200_EINVAL; }
	if (device && ((uintptr_t)cs16 & 3u) != 0) { set_error("d_cs16 must be 4-byte aligned"); return RXB200_EINVAL; }
	const size_t M = (size_t)m->decim, L = (size_t)m->buf_len, pass16 = M * L;
	if (n_int16 % pass16 != 0) {
		set_error("n_int16=%zu must be a multiple of decim * buf_len = %zu (whole passes)", n_int16, pass16);
		return RXB200_EUNSUPPORTED;
	}
	if (n_int16 == 0) { return RXB200_OK; }
	const size_t n_pass = n_int16 / pass16, hops = (size_t)m->n_hops;
	const size_t per_pass = hops * L * sizeof(int16_t);
	const size_t group = std::max<size_t>(1, std::min<size_t>(n_pass, RXB200_POWER_MIX_SCRATCH_BYTES / per_pass));
	RXB_CUDA(cudaSetDevice(m->device));
	const cudaStream_t st = (cudaStream_t)rxb200_power_stream(m->h);
	RXB_CUDA(reserve(m->d_bufs, m->bufs_cap, group * hops * L));
	const size_t n_groups = (n_pass + group - 1) / group;
	while (m->ev.size() < 2 * n_groups) {
		cudaEvent_t e = nullptr;
		RXB_CUDA(cudaEventCreate(&e));
		m->ev.push_back(e);
	}
	const int16_t *src = cs16;
	if (!device) {
		RXB_CUDA(reserve(m->d_cap, m->cap_cap, n_int16));
		RXB_CUDA(cudaMemcpyAsync(m->d_cap, cs16, n_int16 * sizeof(int16_t), cudaMemcpyHostToDevice, st));
		src = m->d_cap;
	}
	m->n_ev = 0;
	for (size_t p0 = 0; p0 < n_pass; p0 += group) {
		const size_t P = std::min(group, n_pass - p0);
		const int16_t *gs = src + p0 * pass16;
		PowDdcArgs a{};
		a.src = reinterpret_cast<const uint32_t *>(gs);
		a.hist = reinterpret_cast<const uint32_t *>(m->d_hist[m->cur_hist]);
		a.n_out = (long long)(P * L / 2);
		a.r0 = (long long)M - 1;                             // pos is a whole number of passes, so of M
		a.pos = m->pos;
		a.dst = reinterpret_cast<uint32_t *>(m->d_bufs);
		a.B = (int)(L / 2);
		a.taps = m->d_taps; a.nco = m->d_nco; a.w = m->d_w;
		a.n_ch = m->n_hops; a.M = m->decim; a.T = m->n_taps; a.S = m->shift;
		RXB_CUDA(cudaEventRecord(m->ev[(size_t)2 * m->n_ev], st));
		int rc = power_ddc_launch(a, m->wide, st);
		if (rc != RXB200_OK) { return rc; }
		RXB_CUDA(cudaEventRecord(m->ev[(size_t)2 * m->n_ev + 1], st));
		m->n_ev++;
		rc = hist_carry(m, gs, P * pass16 / 2, st);
		if (rc != RXB200_OK) { return rc; }
		m->pos += P * pass16 / 2;
		rc = rxb200_power_accumulate_device(m->h, m->d_bufs, (int)P, 0, m->n_hops, 0);
		if (rc != RXB200_OK) { return rc; }
	}
	if (!device || sync) { RXB_CUDA(cudaStreamSynchronize(st)); }
	return RXB200_OK;
}

}  // namespace

extern "C" int rxb200_power_mix_accumulate(rxb200_power_mix *m, const int16_t *cs16, size_t n_int16)
{
	return power_mix_call(m, cs16, n_int16, false, 1);
}

extern "C" int rxb200_power_mix_accumulate_device(rxb200_power_mix *m, const int16_t *d_cs16, size_t n_int16, int sync)
{
	return power_mix_call(m, d_cs16, n_int16, true, sync);
}

extern "C" int rxb200_power_mix_kernel_ms(rxb200_power_mix *m, float *ms)
{
	if (!m || !ms) { return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(m->device));
	float sum = 0.f;
	for (int i = 0; i < m->n_ev; i++) {
		float t = 0.f;
		RXB_CUDA(cudaEventSynchronize(m->ev[(size_t)2 * i + 1]));
		RXB_CUDA(cudaEventElapsedTime(&t, m->ev[(size_t)2 * i], m->ev[(size_t)2 * i + 1]));
		sum += t;
	}
	*ms = sum;
	return RXB200_OK;
}

extern "C" int rxb200_power_ddc_device(int capture_rate, int offset_hz, unsigned long long n0, const rxb200_ddc *ddc,
                                       const int16_t *d_src, size_t n_complex, int16_t *d_dst, void *stream)
{
	if (!d_src || !d_dst) { set_error("bad ddc request (null pointer)"); return RXB200_EINVAL; }
	if (((uintptr_t)d_src & 3u) || ((uintptr_t)d_dst & 3u)) { set_error("pointers must be 4-byte aligned"); return RXB200_EINVAL; }
	std::vector<uint32_t> w;
	int rc = nco_words(capture_rate, &offset_hz, 1, w);
	if (rc != RXB200_OK) { return rc; }
	bool wide = false;
	rc = ddc_check(ddc, &wide);
	const size_t n_out = n_complex / (size_t)(ddc && ddc->decim > 0 ? ddc->decim : 1);
	if (rc != RXB200_OK || n_out == 0) { return rc; }
	// one upload: the table, the word, the reversed taps and a zero history, freed behind the launch
	const size_t T = (size_t)ddc->n_taps;
	const size_t o_w = 2 * NCO_ENTRIES * sizeof(int32_t), o_taps = o_w + 16, o_hist = o_taps + T * sizeof(int32_t);
	const size_t bytes = o_hist + std::max<size_t>(1, T - 1) * sizeof(uint32_t);
	std::vector<unsigned char> h(bytes, 0);
	rxb200_nco_table(reinterpret_cast<int32_t *>(h.data()));
	memcpy(h.data() + o_w, w.data(), sizeof(uint32_t));
	for (size_t j = 0; j < T; j++) { memcpy(h.data() + o_taps + j * sizeof(int32_t), ddc->taps + (T - 1 - j), sizeof(int32_t)); }
	const cudaStream_t st = (cudaStream_t)stream;
	unsigned char *d = nullptr;
	RXB_CUDA(cudaMallocAsync((void **)&d, bytes, st));
	// from pageable memory: the copy has read its source when it returns
	if (cudaMemcpyAsync(d, h.data(), bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) {
		set_error("ddc upload failed: %s", cudaGetErrorString(cudaGetLastError()));
		cudaFreeAsync(d, st);
		return RXB200_ECUDA;
	}
	PowDdcArgs a{};
	a.src = reinterpret_cast<const uint32_t *>(d_src);
	a.hist = reinterpret_cast<const uint32_t *>(d + o_hist);
	a.n_out = (long long)n_out;
	a.r0 = ddc->decim - 1;
	a.pos = n0;
	a.dst = reinterpret_cast<uint32_t *>(d_dst);
	a.B = 1 << 20;                                       // one hop: any B maps output u to word u
	a.taps = reinterpret_cast<const int32_t *>(d + o_taps);
	a.nco = reinterpret_cast<const int2 *>(d);
	a.w = reinterpret_cast<const uint32_t *>(d + o_w);
	a.n_ch = 1; a.M = ddc->decim; a.T = ddc->n_taps; a.S = ddc->shift;
	rc = power_ddc_launch(a, wide, st);
	cudaFreeAsync(d, st);
	return rc;
}
