// fm_mix.cu — several rx_fm channels of one wideband capture (include/rxb200.h, "rx_fm channels of one capture").
// fm_mix_kernel mixes the capture to baseband once per channel with that channel's integer table, reading the capture
// once and writing one CS16 stream per channel; a plain rxb200_fm handle with one channel per stream then runs the
// chain on them through its device entry points.  A decimating handle (rxb200_fm_mix_create_ddc) runs fm_ddc_kernel
// instead (ddc.cuh's down-converter with the channels' tables), which mixes, filters and decimates.  A raster handle
// (rxb200_fm_mix_create_raster) is a decimating handle whose front stage is fm_raster.cu's polyphase channelizer
// instead, and a two-stage handle (rxb200_fm_mix_create_two_stage) one whose front stage is fm_two_stage.cu's coarse and
// fine stages.  The front stage of every kind, with the capture count and the filter state it carries between calls,
// is a CaptureFront (capture_front.cuh); the two mixers it calls back are here.  Every process entry point of every
// kind goes through mix_call, whose refusals and member shape come from fm_mix_check_host_call (which the group uses
// too).  The chain itself is not touched here.
#include <algorithm>
#include <cstring>
#include <new>
#include <vector>
#include "common.cuh"
#include "capture_front.cuh"

namespace rxb {

#define MIX_THREADS 256
#define MIX_UNIT 8                   // complex samples per thread and trip: 32 bytes of capture
#define MIX_SMEM_MAX (96 * 1024)     // the largest table range a CTA stages in shared memory; beyond, reads go through L1

struct MixChan {
	int off;         // first entry of the channel's table in the concatenated tables
	int L;           // period
	unsigned m;      // floor((2^32 - 1) / L): t mod L for t < 2^21 with one multiply-high and one correction
	int pad;
};

// Grid-stride over units of MIX_UNIT complex samples: each thread loads its unit once, then writes it mixed with every
// channel of its group.  Stream row c of dst is dst + c*dst_stride; sample n of the call uses entry (pos + n) mod L of
// its channel.  VEC: src, dst and the row stride are 16-byte aligned, a whole unit moves as two 16-byte vectors (the
// call's last, partial unit and every unit otherwise move 4 bytes at a time).  SMEM: the group's tables are staged in
// shared memory.
template <bool VEC, bool SMEM>
__global__ void __launch_bounds__(MIX_THREADS) fm_mix_kernel(const int16_t *__restrict__ src, long long n,
                                                            int16_t *__restrict__ dst, long long dst_stride,
                                                            const int2 *__restrict__ tab, const MixChan *__restrict__ chan,
                                                            int n_ch, unsigned long long pos)
{
	__shared__ MixChan s_ch[MIX_GROUP];
	__shared__ int s_q[MIX_GROUP];          // each channel's table entry at the trip's first sample
	extern __shared__ int2 s_tab[];
	const int c0 = (int)blockIdx.y * MIX_GROUP;
	const int nc = min(MIX_GROUP, n_ch - c0);
	for (int c = threadIdx.x; c < nc; c += blockDim.x) { s_ch[c] = chan[c0 + c]; }
	__syncthreads();
	const int lo = s_ch[0].off;             // the group's tables are one range of the concatenated tables
	if (SMEM) {
		const int hi = s_ch[nc - 1].off + s_ch[nc - 1].L;
		for (int e = threadIdx.x; e < hi - lo; e += blockDim.x) { s_tab[e] = tab[lo + e]; }
	}
	const long long units = (n + MIX_UNIT - 1) / MIX_UNIT;
	for (long long u0 = (long long)blockIdx.x * blockDim.x; u0 < units; u0 += (long long)gridDim.x * blockDim.x) {
		__syncthreads();                    // the previous trip is done with s_q (and the first trip sees the tables)
		const unsigned long long first = pos + (unsigned long long)u0 * MIX_UNIT;
		for (int c = threadIdx.x; c < nc; c += blockDim.x) { s_q[c] = (int)(first % (unsigned long long)s_ch[c].L); }
		__syncthreads();
		const long long u = u0 + threadIdx.x;
		if (u >= units) { continue; }
		const long long s = u * MIX_UNIT;
		const int cnt = n - s < MIX_UNIT ? (int)(n - s) : MIX_UNIT;
		const bool vec = VEC && cnt == MIX_UNIT;
		const uint32_t *in = reinterpret_cast<const uint32_t *>(src) + s;
		uint32_t w[MIX_UNIT];
		if (vec) {
			const uint4 a = __ldg(reinterpret_cast<const uint4 *>(in)), b = __ldg(reinterpret_cast<const uint4 *>(in) + 1);
			w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
		} else {
#pragma unroll
			for (int j = 0; j < MIX_UNIT; j++) { w[j] = j < cnt ? __ldg(in + j) : 0u; }
		}
		for (int c = 0; c < nc; c++) {
			const MixChan ch = s_ch[c];
			const unsigned L = (unsigned)ch.L;
			const unsigned t = (unsigned)s_q[c] + (unsigned)threadIdx.x * MIX_UNIT;   // < 2^20 + 2^11
			unsigned p = t - __umulhi(t, ch.m) * L;                                    // the quotient is low by at most 1
			if (p >= L) { p -= L; }
			const int base = SMEM ? ch.off - lo : ch.off;
			uint32_t o[MIX_UNIT];
#pragma unroll
			for (int j = 0; j < MIX_UNIT; j++) {
				const int2 cs = SMEM ? s_tab[base + (int)p] : __ldg(tab + base + (int)p);
				o[j] = mix_one(w[j], cs);
				if (++p == L) { p = 0; }
			}
			uint32_t *row = reinterpret_cast<uint32_t *>(dst + (long long)(c0 + c) * dst_stride) + s;
			if (vec) {
				reinterpret_cast<uint4 *>(row)[0] = make_uint4(o[0], o[1], o[2], o[3]);
				reinterpret_cast<uint4 *>(row)[1] = make_uint4(o[4], o[5], o[6], o[7]);
			} else {
#pragma unroll
				for (int j = 0; j < MIX_UNIT; j++) { if (j < cnt) { row[j] = o[j]; } }
			}
		}
	}
}

typedef void (*mix_kernel_fn)(const int16_t *, long long, int16_t *, long long, const int2 *, const MixChan *, int,
                              unsigned long long);

// Launches fm_mix_kernel on the current device: n complex samples of src to n_ch rows of dst, dst_stride int16 apart.
// chan is the host copy of d_chan (for the table range each group stages).
static int mix_launch(const int16_t *src, long long n, int16_t *dst, long long dst_stride, const int2 *d_tab,
                      const MixChan *d_chan, const std::vector<MixChan> &chan, unsigned long long pos, cudaStream_t st)
{
	const int n_ch = (int)chan.size();
	const int groups = (n_ch + MIX_GROUP - 1) / MIX_GROUP;
	size_t smem = 0;
	for (int g = 0; g < groups; g++) {
		const MixChan &a = chan[(size_t)g * MIX_GROUP], &b = chan[(size_t)std::min(n_ch, (g + 1) * MIX_GROUP) - 1];
		const size_t bytes = (size_t)(b.off + b.L - a.off) * sizeof(int2);
		if (bytes > smem) { smem = bytes; }
	}
	const bool use_smem = smem <= MIX_SMEM_MAX;
	if (!use_smem) { smem = 0; }
	const bool vec = ((uintptr_t)src & 15u) == 0 && ((uintptr_t)dst & 15u) == 0 && ((size_t)dst_stride * 2) % 16 == 0;
	const mix_kernel_fn kern = vec ? (use_smem ? fm_mix_kernel<true, true> : fm_mix_kernel<true, false>)
	                               : (use_smem ? fm_mix_kernel<false, true> : fm_mix_kernel<false, false>);
	if (use_smem) { RXB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, MIX_SMEM_MAX)); }
	int dev = 0, n_sm = 0, per_sm = 0;
	RXB_CUDA(cudaGetDevice(&dev));
	RXB_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
	RXB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, MIX_THREADS, smem));
	const long long units = (n + MIX_UNIT - 1) / MIX_UNIT;
	long long bx = (units + MIX_THREADS - 1) / MIX_THREADS;
	const long long fill = (long long)n_sm * (per_sm > 0 ? per_sm : 1) / groups;
	if (bx > fill) { bx = fill > 0 ? fill : 1; }
	kern<<<dim3((unsigned)bx, (unsigned)groups), MIX_THREADS, smem, st>>>(src, n, dst, dst_stride, d_tab, d_chan, n_ch, pos);
	RXB_CUDA(cudaGetLastError());
	return RXB200_OK;
}

static MixChan mix_chan(int off, size_t L)
{
	return MixChan{off, (int)L, (unsigned)(0xffffffffu / (unsigned)L), 0};
}

// the table of (R, f) into a vector; *period receives its length
static int mix_table(int capture_rate, int offset_hz, std::vector<int32_t> &t, size_t *period)
{
	int rc = rxb200_fm_mix_table(capture_rate, offset_hz, nullptr, 0, period);
	if (rc != RXB200_ECAPACITY) { return rc; }
	t.resize(2 * *period);
	return rxb200_fm_mix_table(capture_rate, offset_hz, t.data(), t.size(), period);
}

// ---- the decimating down-converter (rxb200_fm_mix_create_ddc, rxb200_ddc_device): ddc_body with channel c's mixer
// its own table (src[i] uses entry (pos + i) mod L) and its outputs in row c of dst, dst_stride words apart
struct TabMix {
	const int2 *tab;
	const MixChan *chan;
	long long dst_stride;
	struct Row {
		const DdcArgs<TabMix> &a;
		int c0, c;
		long long u0;
		MixChan *s_ch, ch;               // the grid row's channel records in shared memory, and channel c's
		unsigned *s_base, base;          // their table entries at the CTA's first staged sample, and channel c's
		__device__ Row(const DdcArgs<TabMix> &a, int c0, int nc, long long u0, long long g0) : a(a), c0(c0), u0(u0)
		{
			__shared__ MixChan sc[MIX_GROUP];
			__shared__ unsigned sb[MIX_GROUP];
			for (int c = threadIdx.x; c < nc; c += blockDim.x) {
				const MixChan m = a.mix.chan[c0 + c];
				long long q = g0 % m.L;
				sb[c] = (unsigned)(q < 0 ? q + m.L : q);
				sc[c] = m;
			}
			s_ch = sc; s_base = sb;
		}
		__device__ void chan(int k) { c = k; ch = s_ch[k]; base = s_base[k]; }
		__device__ const int2 *entry(int off) const
		{
			const unsigned L = (unsigned)ch.L, t = base + (unsigned)off;      // < 2^20 + DDC_REACH
			unsigned p = t - __umulhi(t, ch.m) * L;                         // the quotient is low by at most 1
			if (p >= L) { p -= L; }
			return a.mix.tab + ch.off + (int)p;
		}
		__device__ uint32_t *out(int u) const { return a.dst + (long long)(c0 + c) * a.mix.dst_stride + u0 + u; }
	};
};

template <typename Acc>
__global__ void __launch_bounds__(DDC_THREADS) fm_ddc_kernel(const DdcArgs<TabMix> a) { ddc_body<Acc>(a); }

}  // namespace rxb

using namespace rxb;

struct rxb200_fm_mix {
	rxb200_fm *h = nullptr;                      // the member: one channel per mixed stream
	int device = 0;
	int n_channels = 0;
	std::vector<MixChan> chan;                   // host copy of d_chan
	int2 *d_tab = nullptr;                       // every channel's table, concatenated
	MixChan *d_chan = nullptr;
	int16_t *d_cap = nullptr; size_t cap_cap = 0;   // host calls: the capture (int16 elements)
	int16_t *d_mix = nullptr; size_t mix_cap = 0;   // the mixed streams, [n_channels][n_int16]
	int16_t *d_out = nullptr; size_t out_cap = 0;   // host calls: the PCM rows, total + 8 apart
	// the front stage: a plain handle's has no filter, and channel k's mixer phase is fr.pos mod L_k; a decimating
	// handle's (any with a filter) writes the decimated streams to d_mix ([n_channels][n_dec_int16]) and the member runs
	// on those
	CaptureFront fr;
};

// Every refusal of a mixing handle's call of n_int16 capture int16 (with a resampler, those its device samples emit), in
// the order the call reports them, without enqueuing anything; *total
// receives the PCM count per channel, *n16 and *chunk16 the member's call (n16 == 0: no member call).  A plain handle's
// member sees the call's own shape.  A decimating handle's member sees the decimated one: a read with no output reports
// what an empty call of the member reports (no PCM, no level chunks), and chunk_result_len entries of capture chunks
// past the member's chunks are 0.
int rxb::fm_mix_check_host_call(rxb200_fm_mix *m, const int16_t *cs16, size_t n_int16, size_t chunk_int16, int16_t *pcm,
                                size_t pcm_stride, int *chunk_result_len, size_t *n_pcm, bool read, size_t *total,
                                size_t *n16, size_t *chunk16)
{
	if (!m) { set_error("null argument"); return RXB200_EINVAL; }
	if (!m->fr.filtered()) {
		*n16 = n_int16;
		*chunk16 = chunk_int16;
		return rxb::fm_check_host_call(m->h, cs16, n_int16, chunk_int16, pcm, pcm_stride, chunk_result_len, n_pcm, read,
		                               total);
	}
	if (!cs16 || !pcm) { set_error("null argument"); return RXB200_EINVAL; }
	const size_t M = m->fr.decim();
	if (n_int16 % 2 != 0) { set_error("n_int16=%zu must be even", n_int16); return RXB200_EUNSUPPORTED; }
	if (!read && (chunk_int16 == 0 || chunk_int16 % (2 * M) != 0)) {
		set_error("chunk_int16=%zu must be a multiple of 2 * decim = %zu", chunk_int16, 2 * M);
		return RXB200_EUNSUPPORTED;
	}
	*n16 = 2 * m->fr.dec_len(n_int16 / 2);
	*chunk16 = read ? *n16 : chunk_int16 / M;
	if (read && *n16 == 0 && n_int16 > 0) {
		return rxb::fm_check_host_call(m->h, cs16, 0, 262144, pcm, pcm_stride, nullptr, n_pcm, false, total);
	}
	const int rc = rxb::fm_check_host_call(m->h, cs16, *n16, *chunk16, pcm, pcm_stride, chunk_result_len, n_pcm, read,
	                                       total);
	if (rc == RXB200_OK && !read && chunk_result_len) {
		const size_t caps = (n_int16 + chunk_int16 - 1) / chunk_int16, decs = (*n16 + *chunk16 - 1) / *chunk16;
		for (size_t c = decs; c < caps; c++) { chunk_result_len[c] = 0; }
	}
	return rc;
}

namespace {

// One call of any process entry point.  device: cs16 and pcm are device pointers (the member's device entry point
// writes pcm), else host pointers staged through the handle's buffers.  read: one read (chunk_int16 == n_int16).  The
// front stage (fm_mix_kernel for a plain handle, fm_ddc_kernel for a decimating one, the raster kernels for a raster
// handle, both stages for a two-stage handle) writes the member's input to d_mix; when it has no output (n16 == 0) the
// member does not run, but the phases and the histories still advance.  The front commits once, after the member's
// call, so a failed call leaves the old histories live.
int mix_call(rxb200_fm_mix *m, const int16_t *cs16, size_t n_int16, size_t chunk_int16, int16_t *pcm, size_t pcm_stride,
             size_t *n_pcm, int *chunk_result_len, bool read, bool device, int sync)
{
	if (!m) { set_error("null argument"); return RXB200_EINVAL; }
	// a CS8, CU8 or CS12 capture may sit at any byte address
	if (device && ((uintptr_t)cs16 & 3u) != 0 && !m->fr.in.on()) { set_error("d_cs16 must be 4-byte aligned"); return RXB200_EINVAL; }
	// with a resampler, the call's shape is that of its capture-rate output: one read of those samples, or its chunks
	const bool rs = m->fr.rs.on();
	if (rs && n_int16 % 2 != 0) { set_error("n_int16=%zu must be even", n_int16); return RXB200_EUNSUPPORTED; }
	const size_t cap16 = rs ? 2 * m->fr.rs.out_len(n_int16 / 2) : n_int16;
	size_t total = 0, n16 = 0, chunk16 = 0;
	// a call whose device samples emit no capture sample reports what an empty call of the member reports
	int rc = rs && cap16 == 0 && n_int16 > 0
	             ? rxb::fm_check_host_call(m->h, cs16, 0, 262144, pcm, pcm_stride, nullptr, n_pcm, false, &total)
	             : rxb::fm_mix_check_host_call(m, cs16, cap16, read ? cap16 : chunk_int16, pcm, pcm_stride,
	                                           chunk_result_len, n_pcm, read, &total, &n16, &chunk16);
	if (rc != RXB200_OK || n_int16 == 0) { return rc; }
	RXB_CUDA(cudaSetDevice(m->device));
	const cudaStream_t st = (cudaStream_t)rxb200_fm_stream(m->h);
	const size_t K = (size_t)m->n_channels, c = n_int16 / 2;
	if (n16) { RXB_CUDA(reserve(m->d_mix, m->mix_cap, n16 * K)); }
	const int16_t *src = cs16;
	if (!device) {
		RXB_CUDA(reserve(m->d_cap, m->cap_cap, n_int16));
		if (n16) { RXB_CUDA(reserve(m->d_out, m->out_cap, (total + 8) * K)); }
		const size_t bytes = m->fr.in.on() ? m->fr.in.bytes(c) : n_int16 * sizeof(int16_t);   // the format's bytes
		RXB_CUDA(cudaMemcpyAsync(m->d_cap, cs16, bytes, cudaMemcpyHostToDevice, st));
		src = m->d_cap;
	}
	rc = m->fr.call<TabMix>(src, c, m->d_mix, (long long)(n16 / 2), RXB200_SDR_OUT_CS16, m->n_channels, st,
	                        [&](DdcArgs<TabMix> &a) {
		if (!m->fr.filtered()) {
			return mix_launch(reinterpret_cast<const int16_t *>(a.src), a.n_out, m->d_mix, (long long)n16, m->d_tab,
			                  m->d_chan, m->chan, a.pos, st);
		}
		a.mix = TabMix{m->d_tab, m->d_chan, (long long)(n16 / 2)};
		return ddc_launch(a, m->fr.f.wide ? fm_ddc_kernel<long long> : fm_ddc_kernel<int>, st);
	});
	if (rc != RXB200_OK) { return rc; }
	rxb::fm_unchain(m->h);                       // the member's input was just written on its stream
	if (n16) {
		int16_t *out = device ? pcm : m->d_out;
		const size_t stride = device ? pcm_stride : total + 8;
		size_t n = 0;
		rc = read ? rxb200_fm_process_read_device(m->h, m->d_mix, n16, out, stride, &n, device ? sync : 0)
		          : rxb200_fm_process_device(m->h, m->d_mix, n16, chunk16, out, stride, &n, device ? sync : 0);
		if (rc != RXB200_OK) { return rc; }
	}
	if (!device) {
		if (total) {
			RXB_CUDA(cudaMemcpy2DAsync(pcm, pcm_stride * sizeof(int16_t), m->d_out, (total + 8) * sizeof(int16_t),
			                           total * sizeof(int16_t), K, cudaMemcpyDeviceToHost, st));
		}
		RXB_CUDA(cudaStreamSynchronize(st));
	} else if (sync && n16 == 0) {
		RXB_CUDA(cudaStreamSynchronize(st));    // with output, the member's call has synchronised
	}
	m->fr.commit(c);
	if (n_pcm) { *n_pcm = total; }
	return RXB200_OK;
}

// The device block of a one-channel call of the mixer or the DDC alone: the table and the channel record, then what
// ddc_upload adds.  *tab and *chan point into it.
int upload_one(const std::vector<int32_t> &t, size_t L, const rxb200_ddc *ddc, cudaStream_t st, DdcBlock *b,
               const int2 **tab, const MixChan **chan)
{
	std::vector<unsigned char> h(L * sizeof(int2) + sizeof(MixChan));
	const MixChan ch = mix_chan(0, L);
	memcpy(h.data(), t.data(), L * sizeof(int2));
	memcpy(h.data() + L * sizeof(int2), &ch, sizeof(MixChan));
	const int rc = ddc_upload(h, ddc, st, b);
	if (rc != RXB200_OK) { return rc; }
	*tab = reinterpret_cast<const int2 *>(b->d);
	*chan = reinterpret_cast<const MixChan *>(b->d + L * sizeof(int2));
	return RXB200_OK;
}

}  // namespace

extern "C" int rxb200_mix_device(int capture_rate, int offset_hz, long long phase, const int16_t *d_src, size_t n_complex,
                                 int16_t *d_dst, void *stream)
{
	if (!d_src || !d_dst || phase < 0) { set_error("bad mix request (null pointer or negative phase)"); return RXB200_EINVAL; }
	if (((uintptr_t)d_src & 3u) || ((uintptr_t)d_dst & 3u)) { set_error("pointers must be 4-byte aligned"); return RXB200_EINVAL; }
	std::vector<int32_t> t;
	size_t L = 0;
	int rc = mix_table(capture_rate, offset_hz, t, &L);
	if (rc != RXB200_OK || n_complex == 0) { return rc; }
	const cudaStream_t st = (cudaStream_t)stream;
	DdcBlock b;
	const int2 *tab = nullptr;
	const MixChan *chan = nullptr;
	rc = upload_one(t, L, nullptr, st, &b, &tab, &chan);
	if (rc != RXB200_OK) { return rc; }
	rc = mix_launch(d_src, (long long)n_complex, d_dst, 0, tab, chan, std::vector<MixChan>(1, mix_chan(0, L)),
	                (unsigned long long)phase % L, st);
	cudaFreeAsync(b.d, st);
	return rc;
}

extern "C" void rxb200_fm_mix_destroy(rxb200_fm_mix *m)
{
	if (!m) { return; }
	rxb200_fm_destroy(m->h);   // synchronises the stream the mixer runs on
	cudaSetDevice(m->device);
	cudaFree(m->d_tab); cudaFree(m->d_chan); cudaFree(m->d_cap); cudaFree(m->d_mix); cudaFree(m->d_out);
	m->fr.release(0);
	delete m;
}

namespace {

// rxb200_fm_mix_create (fr not planned: no filter), rxb200_fm_mix_create_ddc (ddc its filter, already checked),
// rxb200_fm_mix_create_raster and rxb200_fm_mix_create_two_stage (ddc the coarse filter, fine the fine one), with fr
// planned; a single stage has offsets and tables, a raster or two stages none
int mix_create(const rxb200_fm_params *params, int capture_rate, const int *offsets_hz, int n_channels, CaptureFront &fr,
               const rxb200_ddc *ddc, const rxb200_ddc *fine, int device, rxb200_fm_mix **out)
{
	const bool tables = fr.kind == CaptureFront::SINGLE;
	*out = nullptr;
	// every table first: a refused offset fails before any device work
	std::vector<int32_t> all, t;
	std::vector<MixChan> chan;
	for (int k = 0; tables && k < n_channels; k++) {
		size_t L = 0;
		const int rc = mix_table(capture_rate, offsets_hz[k], t, &L);
		if (rc != RXB200_OK) { return rc; }
		if (all.size() / 2 + L > (size_t)INT32_MAX) { set_error("mixer tables beyond 2^31 entries"); return RXB200_EUNSUPPORTED; }
		chan.push_back(mix_chan((int)(all.size() / 2), L));
		all.insert(all.end(), t.begin(), t.end());
	}
	rxb200_fm_mix *m = new (std::nothrow) rxb200_fm_mix();
	if (!m) { return RXB200_ENOMEM; }
	m->device = device;
	m->n_channels = n_channels;
	m->chan = chan;
	m->fr = std::move(fr);
	int rc = rxb200_fm_create(params, device, n_channels, &m->h);
	if (rc != RXB200_OK) { delete m; return rc; }
	RXB_CUDA_OR(cudaSetDevice(device), rxb200_fm_mix_destroy(m));
	if (tables) {
		RXB_CUDA_OR(cudaMalloc(&m->d_tab, all.size() * sizeof(int32_t)), rxb200_fm_mix_destroy(m));
		RXB_CUDA_OR(cudaMalloc(&m->d_chan, chan.size() * sizeof(MixChan)), rxb200_fm_mix_destroy(m));
		RXB_CUDA_OR(cudaMemcpy(m->d_tab, all.data(), all.size() * sizeof(int32_t), cudaMemcpyHostToDevice), rxb200_fm_mix_destroy(m));
		RXB_CUDA_OR(cudaMemcpy(m->d_chan, chan.data(), chan.size() * sizeof(MixChan), cudaMemcpyHostToDevice), rxb200_fm_mix_destroy(m));
	}
	rc = m->fr.create(ddc, fine, (cudaStream_t)rxb200_fm_stream(m->h));
	if (rc != RXB200_OK) { rxb200_fm_mix_destroy(m); return rc; }
	*out = m;
	return RXB200_OK;
}

}  // namespace

extern "C" int rxb200_fm_mix_create(const rxb200_fm_params *params, int capture_rate, const int *offsets_hz,
                                    int n_channels, int device, rxb200_fm_mix **out)
{
	if (!params || !offsets_hz || !out || n_channels < 1) { set_error("bad mix arguments (n_channels >= 1)"); return RXB200_EINVAL; }
	CaptureFront fr;
	return mix_create(params, capture_rate, offsets_hz, n_channels, fr, nullptr, nullptr, device, out);
}

extern "C" int rxb200_fm_mix_create_ddc(const rxb200_fm_params *params, int capture_rate, const int *offsets_hz,
                                        int n_channels, const rxb200_ddc *ddc, int device, rxb200_fm_mix **out)
{
	if (!params || !offsets_hz || !out || n_channels < 1) { set_error("bad mix arguments (n_channels >= 1)"); return RXB200_EINVAL; }
	*out = nullptr;
	CaptureFront fr;
	const int rc = fr.plan_single(ddc);
	if (rc != RXB200_OK) { return rc; }
	return mix_create(params, capture_rate, offsets_hz, n_channels, fr, ddc, nullptr, device, out);
}

extern "C" int rxb200_fm_mix_create_raster(const rxb200_fm_params *params, int n_bins, const int *bins, int n_channels,
                                           const rxb200_ddc *ddc, int device, rxb200_fm_mix **out)
{
	if (!params || !out) { set_error("null argument"); return RXB200_EINVAL; }
	*out = nullptr;
	CaptureFront fr;
	const int rc = fr.plan_raster(n_bins, bins, n_channels, ddc);
	if (rc != RXB200_OK) { return rc; }
	return mix_create(params, 0, nullptr, n_channels, fr, ddc, nullptr, device, out);
}

extern "C" int rxb200_fm_mix_create_two_stage(const rxb200_fm_params *params, int capture_rate, int n_bins,
                                              const int *offsets_hz, int n_channels, const rxb200_ddc *coarse,
                                              const rxb200_ddc *fine, int device, rxb200_fm_mix **out)
{
	if (!params || !out) { set_error("null argument"); return RXB200_EINVAL; }
	*out = nullptr;
	CaptureFront fr;
	const int rc = fr.plan_two_stage(capture_rate, n_bins, offsets_hz, n_channels, coarse, fine);
	if (rc != RXB200_OK) { return rc; }
	return mix_create(params, 0, nullptr, n_channels, fr, coarse, fine, device, out);
}

extern "C" int rxb200_fm_mix_set_device_rate(rxb200_fm_mix *m, const rxb200_resampler *rs)
{
	if (!m) { set_error("null argument"); return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(m->device));
	return m->fr.set_device_rate(rs);
}

extern "C" int rxb200_fm_mix_set_input_format(rxb200_fm_mix *m, int fmt)
{
	if (!m) { set_error("null argument"); return RXB200_EINVAL; }
	return m->fr.set_input_format(fmt);
}

extern "C" int rxb200_fm_mix_decimated_len(const rxb200_fm_mix *m, size_t n_int16, size_t *n_dec_int16)
{
	if (!m || !n_dec_int16) { set_error("null argument"); return RXB200_EINVAL; }
	*n_dec_int16 = m->fr.filtered() || m->fr.rs.on() ? 2 * m->fr.out_len(n_int16 / 2) : n_int16;
	return RXB200_OK;
}

extern "C" size_t rxb200_fm_mix_max_output(const rxb200_fm_mix *m, size_t n_int16, size_t chunk_int16)
{
	if (!m || chunk_int16 == 0) { return 0; }
	const size_t c = m->fr.rs.max_out(n_int16 / 2);             // the capture samples at any resampler count
	if (!m->fr.filtered()) { return rxb200_fm_max_output(m->h, m->fr.rs.on() ? 2 * c : n_int16, chunk_int16); }
	// floor((p + c) / M) - floor(p / M) <= ceil(c / M) at any phase p
	const size_t M = m->fr.decim(), n16 = 2 * ((c + M - 1) / M);
	return rxb200_fm_max_output(m->h, n16, chunk_int16 / M ? chunk_int16 / M : 2);
}

extern "C" int rxb200_ddc_device(int capture_rate, int offset_hz, long long phase, const rxb200_ddc *ddc,
                                 const int16_t *d_src, size_t n_complex, int16_t *d_dst, void *stream)
{
	if (!d_src || !d_dst || phase < 0) { set_error("bad ddc request (null pointer or negative phase)"); return RXB200_EINVAL; }
	if (((uintptr_t)d_src & 3u) || ((uintptr_t)d_dst & 3u)) { set_error("pointers must be 4-byte aligned"); return RXB200_EINVAL; }
	bool wide = false;
	int rc = rxb::ddc_check(ddc, &wide);
	if (rc != RXB200_OK) { return rc; }
	std::vector<int32_t> t;
	size_t L = 0;
	rc = mix_table(capture_rate, offset_hz, t, &L);
	const size_t n_out = n_complex / (size_t)ddc->decim;
	if (rc != RXB200_OK || n_out == 0) { return rc; }
	const cudaStream_t st = (cudaStream_t)stream;
	DdcBlock b;
	DdcArgs<TabMix> a{};
	rc = upload_one(t, L, ddc, st, &b, &a.mix.tab, &a.mix.chan);
	if (rc != RXB200_OK) { return rc; }
	a.src = reinterpret_cast<const uint32_t *>(d_src);
	a.hist = b.hist;
	a.n_out = (long long)n_out;
	a.r0 = ddc->decim - 1;
	a.pos = (unsigned long long)phase % L;
	a.dst = reinterpret_cast<uint32_t *>(d_dst);
	a.taps = b.taps;
	a.n_ch = 1; a.M = ddc->decim; a.T = ddc->n_taps; a.S = ddc->shift;
	rc = ddc_launch(a, wide ? fm_ddc_kernel<long long> : fm_ddc_kernel<int>, st);
	cudaFreeAsync(b.d, st);
	return rc;
}

extern "C" int rxb200_fm_mix_reset(rxb200_fm_mix *m)
{
	if (!m) { return RXB200_EINVAL; }
	const int rc = rxb200_fm_reset(m->h);
	if (rc != RXB200_OK) { return rc; }
	RXB_CUDA(cudaSetDevice(m->device));
	return m->fr.reset((cudaStream_t)rxb200_fm_stream(m->h));   // behind any call still running on the member's stream
}

extern "C" rxb200_fm *rxb200_fm_mix_member(rxb200_fm_mix *m) { return m ? m->h : nullptr; }

extern "C" int rxb200_fm_mix_process(rxb200_fm_mix *m, const int16_t *cs16, size_t n_int16, size_t chunk_int16,
                                     int16_t *pcm, size_t pcm_stride, size_t *n_pcm, int *chunk_result_len)
{
	return mix_call(m, cs16, n_int16, chunk_int16, pcm, pcm_stride, n_pcm, chunk_result_len, false, false, 1);
}

extern "C" int rxb200_fm_mix_process_device(rxb200_fm_mix *m, const int16_t *d_cs16, size_t n_int16, size_t chunk_int16,
                                            int16_t *d_pcm, size_t pcm_stride, size_t *n_pcm, int sync)
{
	return mix_call(m, d_cs16, n_int16, chunk_int16, d_pcm, pcm_stride, n_pcm, nullptr, false, true, sync);
}

extern "C" int rxb200_fm_mix_process_read(rxb200_fm_mix *m, const int16_t *cs16, size_t n_int16, int16_t *pcm,
                                          size_t pcm_stride, size_t *n_pcm)
{
	return mix_call(m, cs16, n_int16, n_int16, pcm, pcm_stride, n_pcm, nullptr, true, false, 1);
}

extern "C" int rxb200_fm_mix_process_read_device(rxb200_fm_mix *m, const int16_t *d_cs16, size_t n_int16, int16_t *d_pcm,
                                                 size_t pcm_stride, size_t *n_pcm, int sync)
{
	return mix_call(m, d_cs16, n_int16, n_int16, d_pcm, pcm_stride, n_pcm, nullptr, true, true, sync);
}

extern "C" int rxb200_fm_mix_squelch_hits(rxb200_fm_mix *m, int *hits)
{
	return m ? rxb200_fm_squelch_hits(m->h, hits) : RXB200_EINVAL;
}

extern "C" int rxb200_fm_mix_levels(rxb200_fm_mix *m, int *levels, size_t cap, size_t *n_chunks)
{
	return m ? rxb200_fm_levels(m->h, levels, cap, n_chunks) : RXB200_EINVAL;
}

extern "C" int rxb200_fm_mix_kernel_ms(rxb200_fm_mix *m, float *ms)
{
	if (!m || !ms) { return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(m->device));
	return m->fr.kernel_ms(ms);
}
