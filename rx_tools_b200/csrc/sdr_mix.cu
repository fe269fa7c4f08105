// sdr_mix.cu — rx_sdr I/Q down-converter handles (include/rxb200.h, "rx_sdr channels of one capture"): several
// channels of one wideband capture, each down-converted and decimated and written in the recorded format, with the
// capture count and the filter histories carried between calls so that a recording made of many calls is one stream.
// A single-stage handle runs sdr_nco_kernel, ddc.cuh's down-converter with power_mix.cu's NCO mixer (NcoMix, its pass
// length set to the row stride so that every channel's outputs form one row) and the rx_sdr output store (SdrOut).  A
// two-stage handle runs fm_two_stage.cu's coarse and fine stages (TwoStage::front), the fine stage writing the format.
// A raster handle runs fm_raster.cu's polyphase channelizer (raster_front), its DFT epilogue writing the format.
#include <algorithm>
#include <new>
#include <vector>
#include "common.cuh"
#include "ddc.cuh"
#include "two_stage.cuh"

namespace rxb {

template <typename Acc, int F>
__global__ void __launch_bounds__(DDC_THREADS) sdr_nco_kernel(const DdcArgs<SdrOut<NcoMix, F>> a) { ddc_body<Acc>(a); }

namespace {

template <int F>
int nco_launch(const DdcArgs<NcoMix> &b, bool wide, cudaStream_t st)
{
	const DdcArgs<SdrOut<NcoMix, F>> a = ddc_args_as<SdrOut<NcoMix, F>>(b);
	return ddc_launch(a, wide ? sdr_nco_kernel<long long, F> : sdr_nco_kernel<int, F>, st);
}

}  // namespace

}  // namespace rxb

using namespace rxb;

struct rxb200_sdr_mix {
	int device = 0;
	int n_ch = 0;
	cudaStream_t st = nullptr;                   // every launch and copy of the handle
	DdcFilter f;                                 // the single stage's filter, or the coarse stage's (two stages)
	uint32_t *d_w = nullptr;                     // single stage: each channel's NCO word
	int2 *d_nco = nullptr;                       // single stage: the shared NCO table
	TwoStage *ts = nullptr;                      // two stages: the plan, the fine stage and the bins' histories
	RasterPlan r;                                // raster (r.K > 0): the raster's shape, its twiddle matrix at d_wt
	double *d_wt = nullptr;
	double *d_v = nullptr; size_t v_cap = 0;     // two stages, raster: the (coarse) branch sums (doubles)
	uint32_t *d_y = nullptr; size_t y_cap = 0;   // two stages: the coarse rows (words)
	unsigned long long pos = 0;                  // capture samples since create or reset
	int16_t *d_cap = nullptr; size_t cap_cap = 0;         // host calls: the capture (int16 elements)
	unsigned char *d_out = nullptr; size_t out_cap = 0;   // host calls: the output rows (bytes)
	cudaEvent_t ev0 = nullptr, ev1 = nullptr;    // around the down-converter kernels of the last call (or group)
};

namespace {

size_t decim(const rxb200_sdr_mix *m) { return (size_t)m->f.M * (size_t)(m->ts ? m->ts->M2 : 1); }

// the outputs per channel of a call of c capture samples after pos: floor((pos + c) / M) - floor(pos / M)
size_t out_len(const rxb200_sdr_mix *m, size_t c)
{
	const unsigned long long M = decim(m);
	return (size_t)((m->pos + c) / M - m->pos / M);
}

bool good_format(int fmt) { return sdr_elem_bytes(fmt) != 0; }

// Every refusal of a process call, in the order the call reports them; *n receives the outputs per channel.
int check_call(const rxb200_sdr_mix *m, const int16_t *cs16, size_t n_int16, int fmt, const void *out, size_t out_cap,
               size_t stride, bool device, size_t *n)
{
	if (!m || !cs16 || !out) { set_error("null argument"); return RXB200_EINVAL; }
	if (!good_format(fmt)) { set_error("output format %d: need RXB200_SDR_OUT_CS16 or RXB200_CVT_CS16_CS8/CU8/CF32", fmt); return RXB200_EINVAL; }
	if (n_int16 % 2 != 0) { set_error("n_int16=%zu must be even", n_int16); return RXB200_EINVAL; }
	const size_t E = (size_t)sdr_elem_bytes(fmt), align = std::min<size_t>(E, 4);
	if (device && (((uintptr_t)cs16 & 3u) || ((uintptr_t)out & (align - 1)))) {
		set_error("d_cs16 must be 4-byte aligned and d_out %zu-byte aligned", align);
		return RXB200_EINVAL;
	}
	if (stride > RXB200_SDR_MIX_MAX_STRIDE) {
		set_error("out_stride %zu above %u elements", stride, (unsigned)RXB200_SDR_MIX_MAX_STRIDE);
		return RXB200_EINVAL;
	}
	*n = out_len(m, n_int16 / 2);
	if (stride < *n || (size_t)(m->n_ch - 1) * stride + *n > out_cap) {
		set_error("%zu outputs per channel need out_stride >= %zu and out_cap >= %zu elements (have %zu, %zu)", *n, *n,
		          (size_t)(m->n_ch - 1) * stride + *n, stride, out_cap);
		return RXB200_ECAPACITY;
	}
	return RXB200_OK;
}

// One checked call on device pointers: the down-converter from the c capture samples at src (a device pointer) to the
// n outputs per channel at dst (rows stride elements apart), then the histories and the count; nothing becomes live
// unless everything was enqueued.
int device_call(rxb200_sdr_mix *m, const int16_t *src, size_t c, int fmt, void *dst, size_t stride, size_t n)
{
	const cudaStream_t st = m->st;
	DdcFilter &f = m->f;
	RXB_CUDA(cudaEventRecord(m->ev0, st));
	if (m->ts) {
		// the coarse outputs whose emission points fall in the call advance the bins' histories even without a fine one
		TwoStage &t = *m->ts;
		const unsigned long long M1 = (unsigned long long)f.M, ma = m->pos / M1;
		const long long n1 = (long long)((m->pos + c) / M1 - ma);
		if (n1 > 0) {
			const long long F = std::min(t.G, n1);
			RXB_CUDA(reserve(m->d_v, m->v_cap, (size_t)F * (size_t)t.r.Kp));
			RXB_CUDA(reserve(m->d_y, m->y_cap, t.y_words(F)));
			const int rc = t.front(f, reinterpret_cast<const uint32_t *>(src), (long long)(ma * M1 + M1 - 1 - m->pos),
			                       (unsigned)(m->pos % (unsigned long long)t.r.K), n1, ma,
			                       (int)(ma % (unsigned long long)t.M2), m->d_v, m->d_y, static_cast<uint32_t *>(dst),
			                       (long long)stride, st, fmt);
			if (rc != RXB200_OK) { return rc; }
		}
	} else if (m->r.K && n) {
		RXB_CUDA(reserve(m->d_v, m->v_cap, (size_t)std::min((long long)n, m->r.group) * (size_t)m->r.Kp));
		const int rc = raster_front(m->r, m->d_wt, m->d_v, reinterpret_cast<const uint32_t *>(src), f.hist[f.cur], f.taps,
		                            f.M, f.T, f.S, (long long)(f.M - 1) - (long long)(m->pos % (unsigned long long)f.M),
		                            (unsigned)(m->pos % (unsigned long long)m->r.K), (long long)n, dst, (long long)stride,
		                            st, fmt);
		if (rc != RXB200_OK) { return rc; }
	} else if (n) {
		DdcArgs<NcoMix> a{};
		a.src = reinterpret_cast<const uint32_t *>(src);
		a.hist = f.hist[f.cur];
		a.n_out = (long long)n;
		a.r0 = (long long)(f.M - 1) - (long long)(m->pos % (unsigned long long)f.M);
		a.pos = m->pos;
		a.dst = static_cast<uint32_t *>(dst);
		a.taps = f.taps;
		a.n_ch = m->n_ch; a.M = f.M; a.T = f.T; a.S = f.S;
		// one "pass" of stride outputs: channel c's output u goes to element c * stride + u (stride >= n)
		a.mix = NcoMix{m->d_nco, m->d_w, (int)std::max<size_t>(stride, 1)};
		const int rc = fmt == RXB200_CVT_CS16_CS8  ? nco_launch<RXB200_CVT_CS16_CS8>(a, f.wide, st)
		             : fmt == RXB200_CVT_CS16_CU8  ? nco_launch<RXB200_CVT_CS16_CU8>(a, f.wide, st)
		             : fmt == RXB200_CVT_CS16_CF32 ? nco_launch<RXB200_CVT_CS16_CF32>(a, f.wide, st)
		                                           : nco_launch<RXB200_SDR_OUT_CS16>(a, f.wide, st);
		if (rc != RXB200_OK) { return rc; }
	}
	RXB_CUDA(cudaEventRecord(m->ev1, st));
	const int rc = f.carry(reinterpret_cast<const uint32_t *>(src), c, st);
	if (rc != RXB200_OK) { return rc; }
	f.commit();
	if (m->ts) { m->ts->commit(); }
	m->pos += c;
	return RXB200_OK;
}

// capture samples per group of a host call: the staged capture and output of a group fit RXB200_SDR_MIX_SCRATCH_BYTES,
// a multiple of M and at least M.  Each group is a device_call, which commits when it succeeds, as rx_power's groups do
// (DdcFilter): the next group reads the history the last one left.
size_t host_group(const rxb200_sdr_mix *m, int fmt)
{
	const size_t M = decim(m), per = 4 * M + (size_t)m->n_ch * (size_t)sdr_elem_bytes(fmt);   // bytes per M samples
	return M * std::max<size_t>(1, (size_t)RXB200_SDR_MIX_SCRATCH_BYTES / per);
}

// rxb200_sdr_mix_create (w the channels' NCO words, ddc the filter), rxb200_sdr_mix_create_two_stage (ts planned,
// ddc the coarse filter, fine the fine one) and rxb200_sdr_mix_create_raster (raster planned, ddc the filter), after
// every refusal
int mix_create(const std::vector<uint32_t> &w, int n_channels, const rxb200_ddc *ddc, bool wide, const TwoStage *ts,
               const rxb200_ddc *fine, const RasterPlan *raster, int device, rxb200_sdr_mix **out)
{
	rxb200_sdr_mix *m = new (std::nothrow) rxb200_sdr_mix();
	if (!m) { return RXB200_ENOMEM; }
	m->device = device;
	m->n_ch = n_channels;
	RXB_CUDA_OR(cudaSetDevice(device), delete m);
	RXB_CUDA_OR(cudaStreamCreateWithFlags(&m->st, cudaStreamNonBlocking), delete m);
	RXB_CUDA_OR(cudaEventCreate(&m->ev0), rxb200_sdr_mix_destroy(m));
	RXB_CUDA_OR(cudaEventCreate(&m->ev1), rxb200_sdr_mix_destroy(m));
	int rc = m->f.create(ddc, wide);
	if (rc != RXB200_OK) { rxb200_sdr_mix_destroy(m); return rc; }
	if (ts) {
		m->ts = new (std::nothrow) TwoStage(*ts);
		if (!m->ts) { rxb200_sdr_mix_destroy(m); return RXB200_ENOMEM; }
		rc = m->ts->upload(fine, m->st);
		if (rc != RXB200_OK) { rxb200_sdr_mix_destroy(m); return rc; }
		RXB_CUDA_OR(cudaStreamSynchronize(m->st), rxb200_sdr_mix_destroy(m));
	} else if (raster) {
		m->r = *raster;
		m->r.wt.clear();
		RXB_CUDA_OR(cudaMalloc(&m->d_wt, raster->w_bytes()), rxb200_sdr_mix_destroy(m));
		RXB_CUDA_OR(cudaMemcpy(m->d_wt, raster->wt.data(), raster->w_bytes(), cudaMemcpyHostToDevice),
		            rxb200_sdr_mix_destroy(m));
	} else {
		std::vector<int32_t> nco(2 * NCO_ENTRIES);
		rxb200_nco_table(nco.data());
		RXB_CUDA_OR(cudaMalloc(&m->d_w, w.size() * sizeof(uint32_t)), rxb200_sdr_mix_destroy(m));
		RXB_CUDA_OR(cudaMalloc(&m->d_nco, nco.size() * sizeof(int32_t)), rxb200_sdr_mix_destroy(m));
		RXB_CUDA_OR(cudaMemcpy(m->d_w, w.data(), w.size() * sizeof(uint32_t), cudaMemcpyHostToDevice), rxb200_sdr_mix_destroy(m));
		RXB_CUDA_OR(cudaMemcpy(m->d_nco, nco.data(), nco.size() * sizeof(int32_t), cudaMemcpyHostToDevice), rxb200_sdr_mix_destroy(m));
	}
	*out = m;
	return RXB200_OK;
}

}  // namespace

extern "C" void rxb200_sdr_mix_destroy(rxb200_sdr_mix *m)
{
	if (!m) { return; }
	cudaSetDevice(m->device);
	if (m->st) { cudaStreamSynchronize(m->st); }
	if (m->ts) { m->ts->release(m->st); delete m->ts; }
	if (m->st) { cudaStreamSynchronize(m->st); }
	m->f.release();
	cudaFree(m->d_w); cudaFree(m->d_nco); cudaFree(m->d_wt); cudaFree(m->d_v); cudaFree(m->d_y); cudaFree(m->d_cap); cudaFree(m->d_out);
	if (m->ev0) { cudaEventDestroy(m->ev0); }
	if (m->ev1) { cudaEventDestroy(m->ev1); }
	if (m->st) { cudaStreamDestroy(m->st); }
	delete m;
}

extern "C" int rxb200_sdr_mix_create(int capture_rate, const int *offsets_hz, int n_channels, const rxb200_ddc *ddc,
                                     int device, rxb200_sdr_mix **out)
{
	if (!offsets_hz || !out || n_channels < 1) { set_error("bad sdr mix arguments (NULL, or n_channels < 1)"); return RXB200_EINVAL; }
	*out = nullptr;
	std::vector<uint32_t> w;
	int rc = nco_words(capture_rate, offsets_hz, n_channels, w);     // the offsets before the ddc, as rx_power's
	if (rc != RXB200_OK) { return rc; }
	bool wide = false;
	rc = ddc_check(ddc, &wide);
	if (rc != RXB200_OK) { return rc; }
	return mix_create(w, n_channels, ddc, wide, nullptr, nullptr, nullptr, device, out);
}

extern "C" int rxb200_sdr_mix_create_two_stage(int capture_rate, int n_bins, const int *offsets_hz, int n_channels,
                                               const rxb200_ddc *coarse, const rxb200_ddc *fine, int device,
                                               rxb200_sdr_mix **out)
{
	if (!out) { set_error("null argument"); return RXB200_EINVAL; }
	*out = nullptr;
	int rc = ddc_check(fine, nullptr);
	if (rc != RXB200_OK) { return rc; }
	rc = ddc_check(coarse, nullptr);
	if (rc != RXB200_OK) { return rc; }
	TwoStage t;
	rc = t.plan(capture_rate, n_bins, offsets_hz, n_channels, coarse, fine);
	if (rc != RXB200_OK) { return rc; }
	return mix_create({}, n_channels, coarse, false, &t, fine, nullptr, device, out);
}

extern "C" int rxb200_sdr_mix_create_raster(int n_bins, const int *bins, int n_channels, const rxb200_ddc *ddc,
                                            int device, rxb200_sdr_mix **out)
{
	if (!out) { set_error("null argument"); return RXB200_EINVAL; }
	*out = nullptr;
	bool wide = false;
	int rc = ddc_check(ddc, &wide);
	if (rc != RXB200_OK) { return rc; }
	rc = raster_check(n_bins, bins, n_channels, ddc);
	if (rc != RXB200_OK) { return rc; }
	RasterPlan p;
	rc = p.plan(n_bins, bins, n_channels);
	if (rc != RXB200_OK) { return rc; }
	return mix_create({}, n_channels, ddc, wide, nullptr, nullptr, &p, device, out);
}

extern "C" int rxb200_sdr_mix_reset(rxb200_sdr_mix *m)
{
	if (!m) { set_error("null argument"); return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(m->device));
	int rc = m->f.reset(m->st);                  // behind any call still running on the handle's stream
	if (rc == RXB200_OK && m->ts) { rc = m->ts->reset(m->st); }
	if (rc != RXB200_OK) { return rc; }
	m->pos = 0;
	return RXB200_OK;
}

extern "C" int rxb200_sdr_mix_decimated_len(const rxb200_sdr_mix *m, size_t n_int16, size_t *n_out)
{
	if (!m || !n_out) { set_error("null argument"); return RXB200_EINVAL; }
	*n_out = out_len(m, n_int16 / 2);
	return RXB200_OK;
}

extern "C" int rxb200_sdr_mix_process_device(rxb200_sdr_mix *m, const int16_t *d_cs16, size_t n_int16, int format,
                                             void *d_out, size_t out_cap, size_t out_stride, size_t *n_out, int sync)
{
	size_t n = 0;
	int rc = check_call(m, d_cs16, n_int16, format, d_out, out_cap, out_stride, true, &n);
	if (rc != RXB200_OK) { return rc; }
	if (n_int16 > 0) {
		RXB_CUDA(cudaSetDevice(m->device));
		rc = device_call(m, d_cs16, n_int16 / 2, format, d_out, out_stride, n);
		if (rc != RXB200_OK) { return rc; }
		if (sync) { RXB_CUDA(cudaStreamSynchronize(m->st)); }
	}
	if (n_out) { *n_out = n; }
	return RXB200_OK;
}

extern "C" int rxb200_sdr_mix_process(rxb200_sdr_mix *m, const int16_t *cs16, size_t n_int16, int format, void *out,
                                      size_t out_cap, size_t out_stride, size_t *n_out)
{
	size_t n = 0;
	int rc = check_call(m, cs16, n_int16, format, out, out_cap, out_stride, false, &n);
	if (rc != RXB200_OK) { return rc; }
	if (n_int16 > 0) {
		RXB_CUDA(cudaSetDevice(m->device));
		const size_t E = (size_t)sdr_elem_bytes(format), g = host_group(m, format), c = n_int16 / 2;
		const size_t gn = g / decim(m) + 1;                   // outputs per channel of a group at any phase
		RXB_CUDA(reserve(m->d_cap, m->cap_cap, 2 * std::min(g, c)));
		RXB_CUDA(reserve(m->d_out, m->out_cap, (size_t)m->n_ch * gn * E));
		size_t done = 0;                                      // outputs per channel written so far
		for (size_t s = 0; s < c; s += g) {
			const size_t cg = std::min(g, c - s), ng = out_len(m, cg);
			RXB_CUDA(cudaMemcpyAsync(m->d_cap, cs16 + 2 * s, cg * 2 * sizeof(int16_t), cudaMemcpyHostToDevice, m->st));
			rc = device_call(m, m->d_cap, cg, format, m->d_out, gn, ng);
			if (rc != RXB200_OK) { return rc; }
			if (ng) {
				RXB_CUDA(cudaMemcpy2DAsync(static_cast<unsigned char *>(out) + done * E, out_stride * E, m->d_out, gn * E,
				                           ng * E, (size_t)m->n_ch, cudaMemcpyDeviceToHost, m->st));
			}
			done += ng;
		}
		RXB_CUDA(cudaStreamSynchronize(m->st));
	}
	if (n_out) { *n_out = n; }
	return RXB200_OK;
}

extern "C" int rxb200_sdr_mix_kernel_ms(rxb200_sdr_mix *m, float *ms)
{
	if (!m || !ms) { set_error("null argument"); return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(m->device));
	RXB_CUDA(cudaEventSynchronize(m->ev1));
	RXB_CUDA(cudaEventElapsedTime(ms, m->ev0, m->ev1));
	return RXB200_OK;
}

extern "C" void *rxb200_sdr_mix_stream(rxb200_sdr_mix *m) { return m ? (void *)m->st : nullptr; }
