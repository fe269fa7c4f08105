// ddc.cu — the host side of the down-converter the mixing handles share (ddc.cuh): the check of an rxb200_ddc, the
// one-shot upload of the stateless entries and the NCO bank; and the host side of the capture front (capture_front.cuh).
#include <cstring>
#include "capture_front.cuh"

// the DDC's arguments: M, T and S in range, taps given, and sum |h| * 32768 + 2^(S-1) < 2^63 (which these ranges
// already bound by 2^59 + 2^61); *wide: the sum reaches 2^31, so the kernel accumulates in 64 bits
int rxb::ddc_check(const rxb200_ddc *d, bool *wide)
{
	if (!d || !d->taps) { set_error("null ddc or taps"); return RXB200_EINVAL; }
	if (d->decim < 1 || d->decim > 4096 || d->n_taps < 1 || d->n_taps > 8192 || d->shift < 0 || d->shift > 62) {
		set_error("ddc decim %d, n_taps %d, shift %d: need 1 <= decim <= 4096, 1 <= n_taps <= 8192, 0 <= shift <= 62",
		          d->decim, d->n_taps, d->shift);
		return RXB200_EINVAL;
	}
	unsigned long long sum = 0;
	for (int j = 0; j < d->n_taps; j++) {
		const long long h = d->taps[j];
		sum += (unsigned long long)(h < 0 ? -h : h);
	}
	const unsigned long long g = sum * 32768ull + (d->shift ? 1ull << (d->shift - 1) : 0ull);
	if (g >= (1ull << 63)) { set_error("sum |taps| * 32768 + 2^(shift-1) >= 2^63"); return RXB200_EINVAL; }
	if (wide) { *wide = g >= (1ull << 31); }
	return RXB200_OK;
}

namespace rxb {

int ddc_upload(std::vector<unsigned char> &h, const rxb200_ddc *ddc, cudaStream_t st, DdcBlock *b)
{
	const size_t T = ddc ? (size_t)ddc->n_taps : 0, o_taps = h.size(), o_hist = o_taps + T * sizeof(int32_t);
	h.resize(o_hist + (ddc ? std::max<size_t>(1, T - 1) * sizeof(uint32_t) : 0), 0);
	for (size_t j = 0; j < T; j++) { memcpy(h.data() + o_taps + j * sizeof(int32_t), ddc->taps + (T - 1 - j), sizeof(int32_t)); }
	RXB_CUDA(cudaMallocAsync((void **)&b->d, h.size(), st));
	// from pageable memory: the copy has read its source when it returns
	if (cudaMemcpyAsync(b->d, h.data(), h.size(), cudaMemcpyHostToDevice, st) != cudaSuccess) {
		set_error("%s upload failed: %s", ddc ? "ddc" : "table", cudaGetErrorString(cudaGetLastError()));
		cudaFreeAsync(b->d, st);
		b->d = nullptr;
		return RXB200_ECUDA;
	}
	b->taps = reinterpret_cast<const int32_t *>(b->d + o_taps);
	b->hist = reinterpret_cast<const uint32_t *>(b->d + o_hist);
	return RXB200_OK;
}

}  // namespace rxb

namespace rxb {

int NcoBank::upload(const std::vector<uint32_t> &words)
{
	std::vector<int32_t> tab(2 * NCO_ENTRIES);
	rxb200_nco_table(tab.data());
	RXB_CUDA(cudaMalloc(&w, words.size() * sizeof(uint32_t)));
	RXB_CUDA(cudaMalloc(&nco, tab.size() * sizeof(int32_t)));
	RXB_CUDA(cudaMemcpy(w, words.data(), words.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
	RXB_CUDA(cudaMemcpy(nco, tab.data(), tab.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
	return RXB200_OK;
}

int CaptureFront::plan_raster(int n_bins, const int *bins, int n_channels, const rxb200_ddc *ddc)
{
	int rc = ddc_check(ddc, &f.wide);
	if (rc != RXB200_OK) { return rc; }
	rc = raster_check(n_bins, bins, n_channels, ddc);
	if (rc != RXB200_OK) { return rc; }
	rc = r.plan(n_bins, bins, n_channels);
	if (rc != RXB200_OK) { return rc; }
	kind = RASTER;
	return RXB200_OK;
}

int CaptureFront::plan_two_stage(int capture_rate, int n_bins, const int *offsets_hz, int n_channels,
                                 const rxb200_ddc *coarse, const rxb200_ddc *fine)
{
	int rc = ddc_check(fine, nullptr);
	if (rc != RXB200_OK) { return rc; }
	rc = ddc_check(coarse, nullptr);
	if (rc != RXB200_OK) { return rc; }
	rc = ts.plan(capture_rate, n_bins, offsets_hz, n_channels, coarse, fine);
	if (rc != RXB200_OK) { return rc; }
	kind = TWO_STAGE;
	return RXB200_OK;
}

int CaptureFront::create(const rxb200_ddc *ddc, const rxb200_ddc *fine, cudaStream_t st)
{
	RXB_CUDA(cudaEventCreate(&ev0));
	RXB_CUDA(cudaEventCreate(&ev1));
	if (ddc) {
		const int rc = f.create(ddc, f.wide);
		if (rc != RXB200_OK) { return rc; }
	}
	if (kind == RASTER) {
		RXB_CUDA(cudaMalloc(&d_wt, r.w_bytes()));
		RXB_CUDA(cudaMemcpy(d_wt, r.wt.data(), r.w_bytes(), cudaMemcpyHostToDevice));
		r.wt = std::vector<double>();
	} else if (kind == TWO_STAGE) {
		return ts.upload(fine, st);
	}
	return RXB200_OK;
}

int CaptureFront::set_device_rate(const rxb200_resampler *r)
{
	if (pos != 0 || rs.pos != 0 || rs.on()) {
		set_error("a device rate is set once, right after create or reset, before any sample");
		return RXB200_EINVAL;
	}
	return rs.attach(r);
}

int CaptureFront::set_input_format(int fmt)
{
	if (pos != 0 || rs.pos != 0) {
		set_error("an input format is set right after create or reset, before any sample");
		return RXB200_EINVAL;
	}
	return in.set(fmt);
}

int CaptureFront::reset(cudaStream_t st)
{
	if (filtered()) {
		int rc = f.reset(st);
		if (rc == RXB200_OK && kind == TWO_STAGE) { rc = ts.reset(st); }
		if (rc != RXB200_OK) { return rc; }
	}
	const int rc = rs.reset(st);
	if (rc != RXB200_OK) { return rc; }
	pos = 0;                                     // the input format stays
	return RXB200_OK;
}

void CaptureFront::release(cudaStream_t st)
{
	in.release();
	rs.release();
	f.release();
	ts.release(st);
	cudaFree(d_wt); cudaFree(d_v); cudaFree(d_y);
	if (ev0) { cudaEventDestroy(ev0); }
	if (ev1) { cudaEventDestroy(ev1); }
}

int CaptureFront::kernel_ms(float *ms)
{
	RXB_CUDA(cudaEventSynchronize(ev1));
	RXB_CUDA(cudaEventElapsedTime(ms, ev0, ev1));
	return RXB200_OK;
}

}  // namespace rxb
