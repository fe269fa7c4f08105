// sdr_mix.cu — rx_sdr I/Q down-converter handles (include/rxb200.h, "rx_sdr channels of one capture"): several
// channels of one wideband capture, each down-converted and decimated and written in the recorded format, with the
// capture count and the filter histories carried between calls so that a recording made of many calls is one stream.
// The front stage, with the count and the histories, is a CaptureFront (capture_front.cuh) of any of its kinds, writing
// the format.  A single-stage handle's launch is here: sdr_nco_kernel, ddc.cuh's down-converter with power_mix.cu's NCO
// mixer (NcoMix, its pass length set to the row stride so that every channel's outputs form one row) and the rx_sdr
// output store (SdrOut).
#include <algorithm>
#include <new>
#include <vector>
#include "common.cuh"
#include "capture_front.cuh"

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
	CaptureFront fr;                             // the front stage (its events: around the kernels of the last group)
	NcoBank nco;                                 // single stage: the NCO table and each channel's word
	int16_t *d_cap = nullptr; size_t cap_cap = 0;         // host calls: the capture in its format (int16 elements)
	unsigned char *d_out = nullptr; size_t out_cap = 0;   // host calls: the output rows (bytes)
};

namespace {

bool good_format(int fmt) { return sdr_elem_bytes(fmt) != 0; }

// Every refusal of a process call, in the order the call reports them; *n receives the outputs per channel.
int check_call(const rxb200_sdr_mix *m, const int16_t *cs16, size_t n_int16, int fmt, const void *out, size_t out_cap,
               size_t stride, bool device, size_t *n)
{
	if (!m || !cs16 || !out) { set_error("null argument"); return RXB200_EINVAL; }
	if (!good_format(fmt)) { set_error("output format %d: need RXB200_SDR_OUT_CS16 or RXB200_CVT_CS16_CS8/CU8/CF32", fmt); return RXB200_EINVAL; }
	if (n_int16 % 2 != 0) { set_error("n_int16=%zu must be even", n_int16); return RXB200_EINVAL; }
	const size_t E = (size_t)sdr_elem_bytes(fmt), align = std::min<size_t>(E, 4);
	// a CS8, CU8 or CS12 capture may sit at any byte address
	if (device && ((((uintptr_t)cs16 & 3u) && !m->fr.in.on()) || ((uintptr_t)out & (align - 1)))) {
		set_error("d_cs16 must be 4-byte aligned and d_out %zu-byte aligned", align);
		return RXB200_EINVAL;
	}
	if (stride > RXB200_SDR_MIX_MAX_STRIDE) {
		set_error("out_stride %zu above %u elements", stride, (unsigned)RXB200_SDR_MIX_MAX_STRIDE);
		return RXB200_EINVAL;
	}
	*n = m->fr.out_len(n_int16 / 2);
	if (stride < *n || (size_t)(m->n_ch - 1) * stride + *n > out_cap) {
		set_error("%zu outputs per channel need out_stride >= %zu and out_cap >= %zu elements (have %zu, %zu)", *n, *n,
		          (size_t)(m->n_ch - 1) * stride + *n, stride, out_cap);
		return RXB200_ECAPACITY;
	}
	return RXB200_OK;
}

// One checked call on device pointers: the front stage from the c capture samples at src (a device pointer) to the
// outputs per channel at dst (rows stride elements apart), then the histories and the count; nothing becomes live
// unless everything was enqueued.
int device_call(rxb200_sdr_mix *m, const int16_t *src, size_t c, int fmt, void *dst, size_t stride)
{
	const int rc = m->fr.call<NcoMix>(src, c, dst, (long long)stride, fmt, m->n_ch, m->st, [&](DdcArgs<NcoMix> &a) {
		// one "pass" of stride outputs: channel c's output u goes to element c * stride + u (stride >= n)
		a.mix = NcoMix{m->nco.nco, m->nco.w, (int)std::max<size_t>(stride, 1)};
		const bool wide = m->fr.f.wide;
		return fmt == RXB200_CVT_CS16_CS8  ? nco_launch<RXB200_CVT_CS16_CS8>(a, wide, m->st)
		     : fmt == RXB200_CVT_CS16_CU8  ? nco_launch<RXB200_CVT_CS16_CU8>(a, wide, m->st)
		     : fmt == RXB200_CVT_CS16_CF32 ? nco_launch<RXB200_CVT_CS16_CF32>(a, wide, m->st)
		                                   : nco_launch<RXB200_SDR_OUT_CS16>(a, wide, m->st);
	});
	if (rc != RXB200_OK) { return rc; }
	m->fr.commit(c);
	return RXB200_OK;
}

// device samples per group of a host call: what a group stages fits RXB200_SDR_MIX_SCRATCH_BYTES.  Without a
// resampler that is the capture and the output rows, a multiple of M and at least M; with one, the device-rate upload,
// the resampled capture (4 bytes per capture sample, L/N of them) and the output rows, at least one device sample.  The
// upload is b bytes per device sample: 4 for CS16, else the format's bytes and the 4 of its widening.  Each group is a
// device_call, which commits when it succeeds, as rx_power's groups do
// (DdcFilter): the next group reads the history the last one left.  *gn: a bound on a group's outputs per channel at
// any phase.
size_t host_group(const rxb200_sdr_mix *m, int fmt, size_t *gn)
{
	const size_t M = m->fr.decim(), rows = (size_t)m->n_ch * (size_t)sdr_elem_bytes(fmt);   // row bytes per M samples
	const ResampleStage &rs = m->fr.rs;
	const size_t b = m->fr.in.on() ? m->fr.in.bytes(1) + 4 : 4;
	size_t g = M * std::max<size_t>(1, (size_t)RXB200_SDR_MIX_SCRATCH_BYTES / (b * M + rows));
	if (rs.on()) {
		// gd device samples take gd (b + (4 M + rows) L / (N M)) bytes
		typedef unsigned __int128 u128;
		const u128 S = RXB200_SDR_MIX_SCRATCH_BYTES, L = (u128)rs.L, N = (u128)rs.N, Mw = (u128)M;
		g = std::max<size_t>(1, (size_t)(S * N * Mw / ((u128)b * N * Mw + (4 * Mw + (u128)rows) * L)));
	}
	*gn = rs.max_out(g) / M + 1;
	return g;
}

// rxb200_sdr_mix_create (w the channels' NCO words, ddc the filter), rxb200_sdr_mix_create_two_stage (fine the fine
// filter) and rxb200_sdr_mix_create_raster, after every refusal: fr planned, ddc its filter (the coarse one for two
// stages)
int mix_create(CaptureFront &fr, const std::vector<uint32_t> &w, int n_channels, const rxb200_ddc *ddc,
               const rxb200_ddc *fine, int device, rxb200_sdr_mix **out)
{
	rxb200_sdr_mix *m = new (std::nothrow) rxb200_sdr_mix();
	if (!m) { return RXB200_ENOMEM; }
	m->device = device;
	m->n_ch = n_channels;
	m->fr = std::move(fr);
	RXB_CUDA_OR(cudaSetDevice(device), delete m);
	RXB_CUDA_OR(cudaStreamCreateWithFlags(&m->st, cudaStreamNonBlocking), delete m);
	int rc = m->fr.create(ddc, fine, m->st);
	if (rc == RXB200_OK && m->fr.kind == CaptureFront::SINGLE) { rc = m->nco.upload(w); }
	if (rc != RXB200_OK) { rxb200_sdr_mix_destroy(m); return rc; }
	RXB_CUDA_OR(cudaStreamSynchronize(m->st), rxb200_sdr_mix_destroy(m));   // the uploads ordered on st are done
	*out = m;
	return RXB200_OK;
}

}  // namespace

extern "C" void rxb200_sdr_mix_destroy(rxb200_sdr_mix *m)
{
	if (!m) { return; }
	cudaSetDevice(m->device);
	if (m->st) { cudaStreamSynchronize(m->st); }
	m->fr.release(m->st);
	if (m->st) { cudaStreamSynchronize(m->st); }
	m->nco.release();
	cudaFree(m->d_cap); cudaFree(m->d_out);
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
	CaptureFront fr;
	rc = fr.plan_single(ddc);
	if (rc != RXB200_OK) { return rc; }
	return mix_create(fr, w, n_channels, ddc, nullptr, device, out);
}

extern "C" int rxb200_sdr_mix_create_two_stage(int capture_rate, int n_bins, const int *offsets_hz, int n_channels,
                                               const rxb200_ddc *coarse, const rxb200_ddc *fine, int device,
                                               rxb200_sdr_mix **out)
{
	if (!out) { set_error("null argument"); return RXB200_EINVAL; }
	*out = nullptr;
	CaptureFront fr;
	const int rc = fr.plan_two_stage(capture_rate, n_bins, offsets_hz, n_channels, coarse, fine);
	if (rc != RXB200_OK) { return rc; }
	return mix_create(fr, {}, n_channels, coarse, fine, device, out);
}

extern "C" int rxb200_sdr_mix_create_raster(int n_bins, const int *bins, int n_channels, const rxb200_ddc *ddc,
                                            int device, rxb200_sdr_mix **out)
{
	if (!out) { set_error("null argument"); return RXB200_EINVAL; }
	*out = nullptr;
	CaptureFront fr;
	const int rc = fr.plan_raster(n_bins, bins, n_channels, ddc);
	if (rc != RXB200_OK) { return rc; }
	return mix_create(fr, {}, n_channels, ddc, nullptr, device, out);
}

extern "C" int rxb200_sdr_mix_reset(rxb200_sdr_mix *m)
{
	if (!m) { set_error("null argument"); return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(m->device));
	return m->fr.reset(m->st);                   // behind any call still running on the handle's stream
}

extern "C" int rxb200_sdr_mix_set_device_rate(rxb200_sdr_mix *m, const rxb200_resampler *rs)
{
	if (!m) { set_error("null argument"); return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(m->device));
	return m->fr.set_device_rate(rs);
}

extern "C" int rxb200_sdr_mix_set_input_format(rxb200_sdr_mix *m, int fmt)
{
	if (!m) { set_error("null argument"); return RXB200_EINVAL; }
	return m->fr.set_input_format(fmt);
}

extern "C" int rxb200_sdr_mix_decimated_len(const rxb200_sdr_mix *m, size_t n_int16, size_t *n_out)
{
	if (!m || !n_out) { set_error("null argument"); return RXB200_EINVAL; }
	*n_out = m->fr.out_len(n_int16 / 2);
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
		rc = device_call(m, d_cs16, n_int16 / 2, format, d_out, out_stride);
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
		size_t gn = 0;                                             // outputs per channel of a group at any phase
		const size_t E = (size_t)sdr_elem_bytes(format), g = host_group(m, format, &gn), c = n_int16 / 2;
		const InputStage &in = m->fr.in;
		RXB_CUDA(reserve(m->d_cap, m->cap_cap, (in.bytes(std::min(g, c)) + 1) / 2));
		RXB_CUDA(reserve(m->d_out, m->out_cap, (size_t)m->n_ch * gn * E));
		size_t done = 0;                                      // outputs per channel written so far
		for (size_t s = 0; s < c; s += g) {
			const size_t cg = std::min(g, c - s), ng = m->fr.out_len(cg);
			RXB_CUDA(cudaMemcpyAsync(m->d_cap, reinterpret_cast<const unsigned char *>(cs16) + in.bytes(s), in.bytes(cg),
			                         cudaMemcpyHostToDevice, m->st));
			rc = device_call(m, m->d_cap, cg, format, m->d_out, gn);
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
	return m->fr.kernel_ms(ms);
}

extern "C" void *rxb200_sdr_mix_stream(rxb200_sdr_mix *m) { return m ? (void *)m->st : nullptr; }
