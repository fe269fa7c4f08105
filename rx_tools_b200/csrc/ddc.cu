// ddc.cu — the host side of the down-converter both mixing handles share (ddc.cuh): the check of an rxb200_ddc and the
// one-shot upload of the stateless entries.
#include <cstring>
#include "ddc.cuh"

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
