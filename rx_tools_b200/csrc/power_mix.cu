// power_mix.cu — every hop of an rx_power sweep from one wideband capture (include/rxb200.h, "rx_power hops of one
// capture").  power_ddc_kernel mixes the capture to baseband once per hop with a phase-accumulator NCO, filters and
// decimates it, and writes each hop's outputs straight into the pass-major hop buffers ([pass][hop][buf_len]) that
// rxb200_power_accumulate_device reads; the member rxb200_power handle then accumulates them on its own stream.  The
// kernel is ddc.cuh's down-converter with its NCO mixer (NcoMix).  The handle carries the sample count (the NCO phases)
// and its filter state (DdcFilter) between calls.  A burst (a fresh capture after a retune, for a tile of a wide sweep)
// runs the same kernel on a subset of the hops, with its history read from the burst's own lead and its phases counted
// from its first sample, and leaves the carried state alone.  A handle whose input format is not CS16 (input_stage.cuh)
// widens each call's elements, stream or burst, to CS16 first.
#include <math.h>
#include <algorithm>
#include <cstring>
#include <new>
#include <vector>
#include "common.cuh"
#include "input_stage.cuh"
#include "resample_stage.cuh"

namespace rxb {

template <typename Acc>
__global__ void __launch_bounds__(DDC_THREADS) power_ddc_kernel(const DdcArgs<NcoMix> a) { ddc_body<Acc>(a); }

// w = floor((f 2^32 + floor(R/2)) / R) mod 2^32, exactly: |f| < R/2 <= 2^30, so the numerator fits 63 bits
int nco_words(int capture_rate, const int *offsets_hz, int n, std::vector<uint32_t> &w)
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
	DdcFilter f;                                 // M, T, S and the filter history
	NcoBank nco;                                 // the shared NCO table and each hop's frequency word
	unsigned long long pos = 0;                  // capture samples since create or reset (whole passes)
	ResampleStage rs;                            // from the device rate, once attached
	bool burst_rate = false;                     // rs resamples bursts only (set_burst_device_rate), statelessly
	InputStage in;                               // the input format, widened to CS16 ahead of rs
	bool taken = false;                          // a call (stream or burst) has taken samples since create or reset
	int16_t *d_cap = nullptr; size_t cap_cap = 0;     // host calls: the capture (int16 elements)
	int16_t *d_bufs = nullptr; size_t bufs_cap = 0;   // the hop buffers of one group of passes, [P][he - hb][buf_len]
	std::vector<cudaEvent_t> ev;                 // pairs around each DDC launch of the last call
	int n_ev = 0;                                // pairs recorded by the last call
};

extern "C" void rxb200_power_mix_destroy(rxb200_power_mix *m)
{
	if (!m) { return; }
	rxb200_power_destroy(m->h);                  // synchronises the stream the DDC runs on
	cudaSetDevice(m->device);
	m->f.release();
	m->rs.release();
	m->in.release();
	m->nco.release();
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
	RXB_CUDA_OR(cudaSetDevice(device), rxb200_power_mix_destroy(m));
	rc = m->nco.upload(w);
	if (rc == RXB200_OK) { rc = m->f.create(ddc, wide); }
	if (rc != RXB200_OK) { rxb200_power_mix_destroy(m); return rc; }
	*out = m;
	return RXB200_OK;
}

extern "C" rxb200_power *rxb200_power_mix_member(rxb200_power_mix *m) { return m ? m->h : nullptr; }

extern "C" int rxb200_power_mix_reset(rxb200_power_mix *m)
{
	if (!m) { return RXB200_EINVAL; }
	int rc = rxb200_power_reset(m->h);
	if (rc != RXB200_OK) { return rc; }
	RXB_CUDA(cudaSetDevice(m->device));
	rc = m->f.reset((cudaStream_t)rxb200_power_stream(m->h));   // behind any call still running on the member's stream
	if (rc == RXB200_OK) { rc = m->rs.reset((cudaStream_t)rxb200_power_stream(m->h)); }
	if (rc != RXB200_OK) { return rc; }
	m->pos = 0;
	m->taken = false;                            // the input format stays
	return RXB200_OK;
}

extern "C" int rxb200_power_mix_set_device_rate(rxb200_power_mix *m, const rxb200_resampler *rs)
{
	if (!m) { set_error("null argument"); return RXB200_EINVAL; }
	if (m->pos != 0 || m->rs.pos != 0 || m->rs.on()) {
		set_error("a device rate is set once, right after create or reset, before any sample");
		return RXB200_EINVAL;
	}
	RXB_CUDA(cudaSetDevice(m->device));
	return m->rs.attach(rs);
}

extern "C" int rxb200_power_mix_set_input_format(rxb200_power_mix *m, int fmt)
{
	if (!m) { set_error("null argument"); return RXB200_EINVAL; }
	if (m->taken) { set_error("an input format is set right after create or reset, before any sample"); return RXB200_EINVAL; }
	return m->in.set(fmt);
}

extern "C" int rxb200_power_mix_set_burst_device_rate(rxb200_power_mix *m, const rxb200_resampler *rs)
{
	if (!m) { set_error("null argument"); return RXB200_EINVAL; }
	if (m->pos != 0 || m->rs.on()) {
		set_error("a burst device rate is set once, right after create or reset, on a handle without a device rate");
		return RXB200_EINVAL;
	}
	RXB_CUDA(cudaSetDevice(m->device));
	const int rc = m->rs.attach(rs);
	if (rc == RXB200_OK) { m->burst_rate = true; }
	return rc;
}

namespace {

// G = M ceil((T - 1) / M): the lead of a burst, in complex samples
size_t burst_lead(const DdcFilter &f) { return (size_t)f.M * (((size_t)f.T - 1 + (size_t)f.M - 1) / (size_t)f.M); }

// E = ceil((J - 1) L / N): the outputs of a device-rate burst whose resampler window reaches before the burst
size_t burst_skip(const ResampleStage &rs) { return (size_t)((rs.f.T - 1) * rs.L + rs.N - 1) / (size_t)rs.N; }

// One call of any entry point: the passes of hops [hb, he) in groups of at most RXB200_POWER_MIX_SCRATCH_BYTES of hop
// buffers, each group one DDC launch into the scratch buffer ([P][he - hb][buf_len]) and one accumulate of the member.
// device: cs16 is a device pointer, else a host pointer staged through the handle's buffer.  burst: cs16 is a burst
// (its lead, then whole passes), whose groups read their history from the burst itself at positions counted from its
// first sample; else cs16 continues the handle's stream, whose history and sample count each group carries on.
int power_mix_call(rxb200_power_mix *m, int hb, int he, const int16_t *cs16, size_t n_int16, bool device, int sync,
                   bool burst)
{
	if (!m || !cs16) { set_error("null argument"); return RXB200_EINVAL; }
	if (hb < 0 || hb >= he || he > m->n_hops) {
		set_error("hop range [%d, %d) needs 0 <= hop_begin < hop_end <= n_hops = %d", hb, he, m->n_hops);
		return RXB200_EINVAL;
	}
	// a CS8, CU8 or CS12 capture may sit at any byte address
	if (device && ((uintptr_t)cs16 & 3u) != 0 && !m->in.on()) { set_error("d_cs16 must be 4-byte aligned"); return RXB200_EINVAL; }
	// rs: this call is resampled, a stream call on a handle with a device rate or a burst on one with a burst device
	// rate; a burst is resampled statelessly, so its first `skip` outputs (E) are dropped
	const bool rs = m->rs.on() && burst == m->burst_rate;
	if (m->rs.on() && burst && !rs) { set_error("a burst is a capture-rate capture: a handle with a device rate takes none"); return RXB200_EUNSUPPORTED; }
	if ((rs || m->in.on()) && n_int16 % 2 != 0) { set_error("n_int16=%zu must be even", n_int16); return RXB200_EUNSUPPORTED; }
	const size_t dev16 = n_int16;                  // with a resampler, the call's device int16; n_int16 its capture's
	const size_t skip = rs && burst ? burst_skip(m->rs) : 0;
	if (rs) {
		const size_t n_out = m->rs.out_len(dev16 / 2);
		n_int16 = n_out > skip ? 2 * (n_out - skip) : 0;
	}
	const size_t M = (size_t)m->f.M, L = (size_t)m->buf_len, pass16 = M * L;
	const size_t lead16 = burst ? 2 * burst_lead(m->f) : 0;
	if (burst && (n_int16 < lead16 + pass16 || (n_int16 - lead16) % pass16 != 0)) {
		set_error("n_int16=%zu must be the lead 2G = %zu plus a positive multiple of decim * buf_len = %zu", n_int16,
		          lead16, pass16);
		return RXB200_EUNSUPPORTED;
	}
	if (n_int16 % pass16 != 0 && !burst) {
		set_error("n_int16=%zu must be a multiple of decim * buf_len = %zu (whole passes)", n_int16, pass16);
		return RXB200_EUNSUPPORTED;
	}
	if (dev16 == 0) { return RXB200_OK; }
	const size_t n_pass = (n_int16 - lead16) / pass16, hops = (size_t)(he - hb);
	const size_t per_pass = hops * L * sizeof(int16_t);
	const size_t group = std::max<size_t>(1, std::min<size_t>(n_pass, RXB200_POWER_MIX_SCRATCH_BYTES / per_pass));
	RXB_CUDA(cudaSetDevice(m->device));
	const cudaStream_t st = (cudaStream_t)rxb200_power_stream(m->h);
	RXB_CUDA(reserve(m->d_bufs, m->bufs_cap, group * hops * L));
	// and a pair around the widening and one around the resampler
	const size_t n_groups = (n_pass + group - 1) / group + (m->in.on() ? 1 : 0) + (rs ? 1 : 0);
	while (m->ev.size() < 2 * n_groups) {
		cudaEvent_t e = nullptr;
		RXB_CUDA(cudaEventCreate(&e));
		m->ev.push_back(e);
	}
	const int16_t *src = cs16;
	if (!device) {
		RXB_CUDA(reserve(m->d_cap, m->cap_cap, dev16));
		const size_t bytes = m->in.on() ? m->in.bytes(dev16 / 2) : dev16 * sizeof(int16_t);   // the format's bytes
		RXB_CUDA(cudaMemcpyAsync(m->d_cap, cs16, bytes, cudaMemcpyHostToDevice, st));
		src = m->d_cap;
	}
	m->n_ev = 0;
	m->taken = true;
	if (m->in.on()) {                              // the whole call to CS16, ahead of everything that reads it
		const uint32_t *w = nullptr;
		RXB_CUDA(cudaEventRecord(m->ev[0], st));
		int rc = m->in.run(src, dev16 / 2, st, &w);
		if (rc != RXB200_OK) { return rc; }
		RXB_CUDA(cudaEventRecord(m->ev[1], st));
		m->n_ev++;
		src = reinterpret_cast<const int16_t *>(w);
	}
	if (rs) {                                      // the whole call to the capture, ahead of the groups that read it
		const uint32_t *x = nullptr;
		RXB_CUDA(cudaEventRecord(m->ev[(size_t)2 * m->n_ev], st));
		int rc = m->rs.run(reinterpret_cast<const uint32_t *>(src), dev16 / 2, st, &x);
		if (rc != RXB200_OK) { return rc; }
		RXB_CUDA(cudaEventRecord(m->ev[(size_t)2 * m->n_ev + 1], st));
		m->n_ev++;
		if (!burst) { m->rs.commit(dev16 / 2); }    // a burst leaves the stage at count 0 with its zero history
		src = reinterpret_cast<const int16_t *>(x + skip);
	}
	DdcFilter &f = m->f;
	for (size_t p0 = 0; p0 < n_pass; p0 += group) {
		const size_t P = std::min(group, n_pass - p0);
		DdcArgs<NcoMix> a{};
		a.src = reinterpret_cast<const uint32_t *>(src + lead16 + p0 * pass16);
		// a burst's lead is at least T - 1 samples, so its history is the samples just before src in the burst
		a.hist = burst ? a.src - (f.T - 1) : f.hist[f.cur];
		a.n_out = (long long)(P * L / 2);
		a.r0 = (long long)M - 1;                             // pos is the lead plus whole passes, so a multiple of M
		a.pos = burst ? (lead16 + p0 * pass16) / 2 : m->pos;
		a.dst = reinterpret_cast<uint32_t *>(m->d_bufs);
		a.taps = f.taps;
		a.n_ch = he - hb; a.M = f.M; a.T = f.T; a.S = f.S;
		a.mix = NcoMix{m->nco.nco, m->nco.w + hb, (int)(L / 2)};
		RXB_CUDA(cudaEventRecord(m->ev[(size_t)2 * m->n_ev], st));
		int rc = ddc_launch(a, f.wide ? power_ddc_kernel<long long> : power_ddc_kernel<int>, st);
		if (rc != RXB200_OK) { return rc; }
		RXB_CUDA(cudaEventRecord(m->ev[(size_t)2 * m->n_ev + 1], st));
		m->n_ev++;
		if (!burst) {
			rc = f.carry(a.src, P * pass16 / 2, st);
			if (rc != RXB200_OK) { return rc; }
			f.commit();
			m->pos += P * pass16 / 2;
		}
		rc = rxb200_power_accumulate_device(m->h, m->d_bufs, (int)P, hb, he, 0);
		if (rc != RXB200_OK) { return rc; }
	}
	if (!device || sync) { RXB_CUDA(cudaStreamSynchronize(st)); }
	return RXB200_OK;
}

}  // namespace

extern "C" int rxb200_power_mix_accumulate(rxb200_power_mix *m, const int16_t *cs16, size_t n_int16)
{
	return power_mix_call(m, 0, m ? m->n_hops : 1, cs16, n_int16, false, 1, false);
}

extern "C" int rxb200_power_mix_accumulate_device(rxb200_power_mix *m, const int16_t *d_cs16, size_t n_int16, int sync)
{
	return power_mix_call(m, 0, m ? m->n_hops : 1, d_cs16, n_int16, true, sync, false);
}

extern "C" int rxb200_power_mix_lead(const rxb200_power_mix *m)
{
	if (!m) { set_error("null argument"); return RXB200_EINVAL; }
	return (int)burst_lead(m->f);
}

extern "C" int rxb200_power_mix_accumulate_burst(rxb200_power_mix *m, int hop_begin, int hop_end, const int16_t *cs16,
                                                 size_t n_int16)
{
	return power_mix_call(m, hop_begin, hop_end, cs16, n_int16, false, 1, true);
}

extern "C" int rxb200_power_mix_accumulate_burst_device(rxb200_power_mix *m, int hop_begin, int hop_end,
                                                        const int16_t *d_cs16, size_t n_int16, int sync)
{
	return power_mix_call(m, hop_begin, hop_end, d_cs16, n_int16, true, sync, true);
}

extern "C" int rxb200_power_mix_burst_in_len(const rxb200_power_mix *m, int passes, size_t *n_int16)
{
	if (!m || !n_int16 || passes < 1) { set_error("burst_in_len needs a handle, n_int16 and passes >= 1"); return RXB200_EINVAL; }
	const size_t capture = burst_lead(m->f) + (size_t)passes * (size_t)m->f.M * (size_t)m->buf_len / 2;
	if (!m->burst_rate) { *n_int16 = 2 * capture; return RXB200_OK; }
	size_t c = 0;
	const int rc = rxb200_resample_in_len((int)m->rs.L, (int)m->rs.N, 0, burst_skip(m->rs) + capture, &c);
	if (rc != RXB200_OK) { return rc; }
	*n_int16 = 2 * c;
	return RXB200_OK;
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
	// the table, then the word (16 bytes)
	const size_t o_w = 2 * NCO_ENTRIES * sizeof(int32_t);
	std::vector<unsigned char> h(o_w + 16, 0);
	rxb200_nco_table(reinterpret_cast<int32_t *>(h.data()));
	memcpy(h.data() + o_w, w.data(), sizeof(uint32_t));
	const cudaStream_t st = (cudaStream_t)stream;
	DdcBlock b;
	rc = ddc_upload(h, ddc, st, &b);
	if (rc != RXB200_OK) { return rc; }
	DdcArgs<NcoMix> a{};
	a.src = reinterpret_cast<const uint32_t *>(d_src);
	a.hist = b.hist;
	a.n_out = (long long)n_out;
	a.r0 = ddc->decim - 1;
	a.pos = n0;
	a.dst = reinterpret_cast<uint32_t *>(d_dst);
	a.taps = b.taps;
	a.n_ch = 1; a.M = ddc->decim; a.T = ddc->n_taps; a.S = ddc->shift;
	// one hop: any B maps output u to word u
	a.mix = NcoMix{reinterpret_cast<const int2 *>(b.d), reinterpret_cast<const uint32_t *>(b.d + o_w), 1 << 20};
	rc = ddc_launch(a, wide ? power_ddc_kernel<long long> : power_ddc_kernel<int>, st);
	cudaFreeAsync(b.d, st);
	return rc;
}
