// fm_group.cpp — rx_fm on several GPUs in one process (include/rxb200.h, rxb200_fm_group_*): n_dev rxb200_fm handles,
// each owning a contiguous block of the channels.  Host code only: every member runs the single-handle device entry
// points on its own stream, so the group adds copies and bookkeeping, no kernel.
#include <new>
#include <vector>
#include "common.cuh"

using rxb::set_error;

struct rxb200_fm_group {
	int n_channels = 0;
	int n_dev = 0;
	std::vector<rxb200_fm *> h;              // NULL for a member that owns no channel
	std::vector<int> device, ch_begin, ch_end;
	// each member's staging buffers on its device: its channels' input, and its PCM at a row stride of total + 8
	std::vector<int16_t *> d_in, d_out;
	std::vector<size_t> in_cap, out_cap;     // int16 elements
};

namespace {

// puts the caller's current device back when an entry point returns, whichever way it returns
struct DeviceGuard {
	int dev = -1;
	DeviceGuard() { if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = -1; } }
	~DeviceGuard() { if (dev >= 0) { cudaSetDevice(dev); } }
};

// grows a member's staging buffer to at least `need` int16 (the contents are not kept)
cudaError_t reserve(int16_t *&buf, size_t &cap, size_t need)
{
	if (need <= cap) { return cudaSuccess; }
	cudaFree(buf); buf = nullptr; cap = 0;
	const cudaError_t e = cudaMalloc(&buf, need * sizeof(int16_t));
	if (e == cudaSuccess) { cap = need; }
	return e;
}

// Member i's input half of a call: its block of channels to its device, then the device entry point without a sync, on
// its own stream.  *started is set once anything was enqueued.
int enqueue_in(rxb200_fm_group *g, int i, const int16_t *cs16, size_t n_int16, size_t chunk_int16, size_t total,
               bool read, bool *started)
{
	rxb200_fm *h = g->h[(size_t)i];
	const size_t b = (size_t)g->ch_begin[(size_t)i], nch = (size_t)(g->ch_end[(size_t)i] - g->ch_begin[(size_t)i]);
	const size_t out_stride = total + 8;
	RXB_CUDA(cudaSetDevice(g->device[(size_t)i]));
	RXB_CUDA(reserve(g->d_in[(size_t)i], g->in_cap[(size_t)i], n_int16 * nch));
	RXB_CUDA(reserve(g->d_out[(size_t)i], g->out_cap[(size_t)i], out_stride * nch));
	int16_t *d_in = g->d_in[(size_t)i], *d_out = g->d_out[(size_t)i];
	*started = true;
	RXB_CUDA(cudaMemcpyAsync(d_in, cs16 + b * n_int16, n_int16 * nch * sizeof(int16_t), cudaMemcpyHostToDevice,
	                         (cudaStream_t)rxb200_fm_stream(h)));
	size_t n = 0;
	return read ? rxb200_fm_process_read_device(h, d_in, n_int16, d_out, total + 8, &n, 0)
	            : rxb200_fm_process_device(h, d_in, n_int16, chunk_int16, d_out, total + 8, &n, 0);
}

// Member i's output half: its PCM rows into the caller's pcm, on its stream behind its kernels
int enqueue_out(rxb200_fm_group *g, int i, int16_t *pcm, size_t pcm_stride, size_t total)
{
	const size_t b = (size_t)g->ch_begin[(size_t)i], nch = (size_t)(g->ch_end[(size_t)i] - g->ch_begin[(size_t)i]);
	if (total == 0) { return RXB200_OK; }
	RXB_CUDA(cudaSetDevice(g->device[(size_t)i]));
	RXB_CUDA(cudaMemcpy2DAsync(pcm + b * pcm_stride, pcm_stride * sizeof(int16_t), g->d_out[(size_t)i],
	                           (total + 8) * sizeof(int16_t), total * sizeof(int16_t), nch, cudaMemcpyDeviceToHost,
	                           (cudaStream_t)rxb200_fm_stream(g->h[(size_t)i])));
	return RXB200_OK;
}

int group_process(rxb200_fm_group *g, const int16_t *cs16, size_t n_int16, size_t chunk_int16, int16_t *pcm,
                  size_t pcm_stride, size_t *n_pcm, int *chunk_result_len, bool read)
{
	if (!g || !cs16 || !pcm) { set_error("null argument"); return RXB200_EINVAL; }
	DeviceGuard guard;
	// every refusal first, on every member, so that a refused call starts none of them
	size_t total = 0;
	for (int i = 0; i < g->n_dev; i++) {
		if (!g->h[(size_t)i]) { continue; }
		const int rc = rxb::fm_check_host_call(g->h[(size_t)i], cs16, n_int16, chunk_int16, pcm, pcm_stride, chunk_result_len,
		                                       n_pcm, read, &total);
		if (rc != RXB200_OK) { return rc; }
	}
	if (n_int16 == 0) { return RXB200_OK; }
	int rc = RXB200_OK;
	std::vector<char> started((size_t)g->n_dev, 0);
	// every member's input and kernels before any output copy: a copy to or from pageable memory holds this thread until
	// it is done, and an output copy waits for its member's kernels, which then overlap the later members' input copies
	for (int i = 0; i < g->n_dev && rc == RXB200_OK; i++) {
		if (!g->h[(size_t)i]) { continue; }
		bool st = false;
		rc = enqueue_in(g, i, cs16, n_int16, chunk_int16, total, read, &st);
		started[(size_t)i] = st ? 1 : 0;
	}
	for (int i = 0; i < g->n_dev && rc == RXB200_OK; i++) {
		if (g->h[(size_t)i]) { rc = enqueue_out(g, i, pcm, pcm_stride, total); }
	}
	// wait for every member that started, also after a failure: its copies still read cs16 and write pcm
	for (int i = 0; i < g->n_dev; i++) {
		if (!started[(size_t)i]) { continue; }
		cudaError_t e = cudaSetDevice(g->device[(size_t)i]);
		if (e == cudaSuccess) { e = cudaStreamSynchronize((cudaStream_t)rxb200_fm_stream(g->h[(size_t)i])); }
		if (e != cudaSuccess && rc == RXB200_OK) {
			set_error("member %d: cudaStreamSynchronize failed: %s", i, cudaGetErrorString(e));
			rc = RXB200_ECUDA;
		}
	}
	if (rc == RXB200_OK && n_pcm) { *n_pcm = total; }
	return rc;
}

}  // namespace

extern "C" void rxb200_fm_group_destroy(rxb200_fm_group *g)
{
	if (!g) { return; }
	DeviceGuard guard;
	for (int i = 0; i < g->n_dev; i++) {
		rxb200_fm_destroy(g->h[(size_t)i]);   // synchronises the member's stream
		if (g->d_in[(size_t)i] || g->d_out[(size_t)i]) {
			cudaSetDevice(g->device[(size_t)i]);
			cudaFree(g->d_in[(size_t)i]);
			cudaFree(g->d_out[(size_t)i]);
		}
	}
	delete g;
}

extern "C" int rxb200_fm_group_create(const rxb200_fm_params *params, int n_channels, int n_dev, const int *devices,
                                      rxb200_fm_group **out)
{
	if (!params || !out || n_channels < 1 || n_dev < 1) { set_error("bad group arguments (n_channels >= 1, n_dev >= 1)"); return RXB200_EINVAL; }
	*out = nullptr;
	DeviceGuard guard;
	rxb200_fm_group *g = new (std::nothrow) rxb200_fm_group();
	if (!g) { return RXB200_ENOMEM; }
	g->n_channels = n_channels;
	g->n_dev = n_dev;
	const size_t n = (size_t)n_dev;
	g->h.assign(n, nullptr);
	g->device.assign(n, 0); g->ch_begin.assign(n, 0); g->ch_end.assign(n, 0);
	g->d_in.assign(n, nullptr); g->d_out.assign(n, nullptr);
	g->in_cap.assign(n, 0); g->out_cap.assign(n, 0);
	for (int i = 0; i < n_dev; i++) {
		g->device[(size_t)i] = devices ? devices[i] : i;
		rxb200_power_shard(n_channels, n_dev, i, &g->ch_begin[(size_t)i], &g->ch_end[(size_t)i]);
		const int nch = g->ch_end[(size_t)i] - g->ch_begin[(size_t)i];
		if (nch < 1) { continue; }
		const int rc = rxb200_fm_create(params, g->device[(size_t)i], nch, &g->h[(size_t)i]);
		if (rc != RXB200_OK) { rxb200_fm_group_destroy(g); return rc; }
	}
	*out = g;
	return RXB200_OK;
}

extern "C" int rxb200_fm_group_size(const rxb200_fm_group *g) { return g ? g->n_dev : 0; }

extern "C" rxb200_fm *rxb200_fm_group_member(rxb200_fm_group *g, int i)
{
	return (g && i >= 0 && i < g->n_dev) ? g->h[(size_t)i] : nullptr;
}

extern "C" int rxb200_fm_group_process(rxb200_fm_group *g, const int16_t *cs16, size_t n_int16, size_t chunk_int16,
                                       int16_t *pcm, size_t pcm_stride, size_t *n_pcm, int *chunk_result_len)
{
	return group_process(g, cs16, n_int16, chunk_int16, pcm, pcm_stride, n_pcm, chunk_result_len, false);
}

extern "C" int rxb200_fm_group_process_read(rxb200_fm_group *g, const int16_t *cs16, size_t n_int16, int16_t *pcm,
                                            size_t pcm_stride, size_t *n_pcm)
{
	return group_process(g, cs16, n_int16, n_int16, pcm, pcm_stride, n_pcm, nullptr, true);
}

extern "C" int rxb200_fm_group_squelch_hits(rxb200_fm_group *g, int *hits)
{
	if (!g || !hits) { return RXB200_EINVAL; }
	DeviceGuard guard;
	for (int i = 0; i < g->n_dev; i++) {
		if (!g->h[(size_t)i]) { continue; }
		const int rc = rxb200_fm_squelch_hits(g->h[(size_t)i], hits + g->ch_begin[(size_t)i]);
		if (rc != RXB200_OK) { return rc; }
	}
	return RXB200_OK;
}

extern "C" int rxb200_fm_group_levels(rxb200_fm_group *g, int *levels, size_t cap, size_t *n_chunks)
{
	if (!g || !levels || !n_chunks) { set_error("null argument"); return RXB200_EINVAL; }
	DeviceGuard guard;
	// every member holds the same chunk count; member 0 always owns a channel.  A zero capacity only asks for the count
	size_t nc = 0;
	int rc = rxb200_fm_levels(g->h[0], levels, 0, &nc);
	if (rc != RXB200_OK && rc != RXB200_ECAPACITY) { return rc; }
	*n_chunks = nc;
	const size_t cells = nc * (size_t)g->n_channels;
	if (cap < cells) { set_error("levels capacity %zu < %zu", cap, cells); return RXB200_ECAPACITY; }
	for (int i = 0; i < g->n_dev && cells; i++) {
		if (!g->h[(size_t)i]) { continue; }
		const size_t b = (size_t)g->ch_begin[(size_t)i], e = (size_t)g->ch_end[(size_t)i];
		size_t member_chunks = 0;
		rc = rxb200_fm_levels(g->h[(size_t)i], levels + b * nc, (e - b) * nc, &member_chunks);
		if (rc != RXB200_OK) { return rc; }
	}
	return RXB200_OK;
}

extern "C" int rxb200_fm_group_reset(rxb200_fm_group *g)
{
	if (!g) { return RXB200_EINVAL; }
	DeviceGuard guard;
	for (auto *h : g->h) {
		if (!h) { continue; }
		const int rc = rxb200_fm_reset(h);
		if (rc != RXB200_OK) { return rc; }
	}
	return RXB200_OK;
}
