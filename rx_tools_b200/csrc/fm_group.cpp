// fm_group.cpp — rx_fm on several GPUs in one process (include/rxb200.h): rxb200_fm_group_* splits channel streams over
// n_dev rxb200_fm handles, rxb200_fm_mix_group_* splits the channels of one capture over n_dev rxb200_fm_mix handles.
// Each member owns a contiguous block of the channels.  Host code only: every member runs the single-handle device
// entry points on its own stream, so a group adds copies and bookkeeping, no kernel.  Both kinds share every step of a
// call; a member record tells them apart where they differ (how a member is made, reset and destroyed, what its input
// copy takes and which device entry point it calls).
#include <new>
#include <vector>
#include "common.cuh"

using rxb::reserve;
using rxb::set_error;

namespace {

struct Member {
	rxb200_fm *h = nullptr;          // the inner handle: refusals, stream, levels, squelch hits.  NULL: no channel
	rxb200_fm_mix *m = nullptr;      // a mixing group's member (h is its inner handle); NULL in a plain group
	int device = 0, ch_begin = 0, ch_end = 0;
	// staging buffers on the member's device: its input, and its PCM at a row stride of total + 8
	int16_t *d_in = nullptr, *d_out = nullptr;
	size_t in_cap = 0, out_cap = 0;  // int16 elements
};

struct Group {
	int n_channels = 0;
	std::vector<Member> mb;
};

}  // namespace

struct rxb200_fm_group : Group {};
struct rxb200_fm_mix_group : Group {};

namespace {

// puts the caller's current device back when an entry point returns, whichever way it returns
struct DeviceGuard {
	int dev = -1;
	DeviceGuard() { if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = -1; } }
	~DeviceGuard() { if (dev >= 0) { cudaSetDevice(dev); } }
};

template <typename G>
void group_destroy(G *g)
{
	if (!g) { return; }
	DeviceGuard guard;
	for (Member &mb : g->mb) {
		if (mb.m) { rxb200_fm_mix_destroy(mb.m); } else { rxb200_fm_destroy(mb.h); }   // synchronises the member's stream
		if (mb.d_in || mb.d_out) {
			cudaSetDevice(mb.device);
			cudaFree(mb.d_in);
			cudaFree(mb.d_out);
		}
	}
	delete g;
}

// the members' shard ranges and devices; make(member, nch) creates the handle of a member whose range is not empty
template <typename G, typename Make>
int group_create(int n_channels, int n_dev, const int *devices, Make make, G **out)
{
	DeviceGuard guard;
	G *g = new (std::nothrow) G();
	if (!g) { return RXB200_ENOMEM; }
	g->n_channels = n_channels;
	g->mb.resize((size_t)n_dev);
	for (int i = 0; i < n_dev; i++) {
		Member &mb = g->mb[(size_t)i];
		mb.device = devices ? devices[i] : i;
		rxb200_power_shard(n_channels, n_dev, i, &mb.ch_begin, &mb.ch_end);
		const int nch = mb.ch_end - mb.ch_begin;
		if (nch < 1) { continue; }
		const int rc = make(mb, nch);
		if (rc != RXB200_OK) { group_destroy(g); return rc; }
	}
	*out = g;
	return RXB200_OK;
}

// A member's input half of a call: its input to its device (a mixing member takes the whole capture, a plain one its
// block of channel streams), then the device entry point without a sync, on its own stream.  *started is set once
// anything was enqueued.
int enqueue_in(Member &mb, const int16_t *cs16, size_t n_int16, size_t chunk_int16, size_t total, bool read,
               bool *started)
{
	const size_t nch = (size_t)(mb.ch_end - mb.ch_begin);
	const int16_t *src = mb.m ? cs16 : cs16 + (size_t)mb.ch_begin * n_int16;
	const size_t in_elems = mb.m ? n_int16 : n_int16 * nch;
	RXB_CUDA(cudaSetDevice(mb.device));
	RXB_CUDA(reserve(mb.d_in, mb.in_cap, in_elems));
	RXB_CUDA(reserve(mb.d_out, mb.out_cap, (total + 8) * nch));
	*started = true;
	RXB_CUDA(cudaMemcpyAsync(mb.d_in, src, in_elems * sizeof(int16_t), cudaMemcpyHostToDevice,
	                         (cudaStream_t)rxb200_fm_stream(mb.h)));
	rxb::fm_unchain(mb.h);
	size_t n = 0;
	if (mb.m) {
		return read ? rxb200_fm_mix_process_read_device(mb.m, mb.d_in, n_int16, mb.d_out, total + 8, &n, 0)
		            : rxb200_fm_mix_process_device(mb.m, mb.d_in, n_int16, chunk_int16, mb.d_out, total + 8, &n, 0);
	}
	return read ? rxb200_fm_process_read_device(mb.h, mb.d_in, n_int16, mb.d_out, total + 8, &n, 0)
	            : rxb200_fm_process_device(mb.h, mb.d_in, n_int16, chunk_int16, mb.d_out, total + 8, &n, 0);
}

// A member's output half: its PCM rows into the caller's pcm, on its stream behind its kernels
int enqueue_out(const Member &mb, int16_t *pcm, size_t pcm_stride, size_t total)
{
	const size_t b = (size_t)mb.ch_begin, nch = (size_t)(mb.ch_end - mb.ch_begin);
	if (total == 0) { return RXB200_OK; }
	RXB_CUDA(cudaSetDevice(mb.device));
	RXB_CUDA(cudaMemcpy2DAsync(pcm + b * pcm_stride, pcm_stride * sizeof(int16_t), mb.d_out,
	                           (total + 8) * sizeof(int16_t), total * sizeof(int16_t), nch, cudaMemcpyDeviceToHost,
	                           (cudaStream_t)rxb200_fm_stream(mb.h)));
	return RXB200_OK;
}

int group_process(Group *g, const int16_t *cs16, size_t n_int16, size_t chunk_int16, int16_t *pcm, size_t pcm_stride,
                  size_t *n_pcm, int *chunk_result_len, bool read)
{
	if (!g || !cs16 || !pcm) { set_error("null argument"); return RXB200_EINVAL; }
	DeviceGuard guard;
	// every refusal first, on every member, so that a refused call starts none of them
	size_t total = 0, n16 = 0, chunk16 = 0;
	for (Member &mb : g->mb) {
		if (!mb.h) { continue; }
		const int rc = mb.m ? rxb::fm_mix_check_host_call(mb.m, cs16, n_int16, chunk_int16, pcm, pcm_stride,
		                                                  chunk_result_len, n_pcm, read, &total, &n16, &chunk16)
		                    : rxb::fm_check_host_call(mb.h, cs16, n_int16, chunk_int16, pcm, pcm_stride, chunk_result_len,
		                                              n_pcm, read, &total);
		if (rc != RXB200_OK) { return rc; }
	}
	if (n_int16 == 0) { return RXB200_OK; }
	int rc = RXB200_OK;
	std::vector<char> started(g->mb.size(), 0);
	// every member's input and kernels before any output copy: a copy to or from pageable memory holds this thread until
	// it is done, and an output copy waits for its member's kernels, which then overlap the later members' input copies
	for (size_t i = 0; i < g->mb.size() && rc == RXB200_OK; i++) {
		if (!g->mb[i].h) { continue; }
		bool st = false;
		rc = enqueue_in(g->mb[i], cs16, n_int16, chunk_int16, total, read, &st);
		started[i] = st ? 1 : 0;
	}
	for (size_t i = 0; i < g->mb.size() && rc == RXB200_OK; i++) {
		if (g->mb[i].h) { rc = enqueue_out(g->mb[i], pcm, pcm_stride, total); }
	}
	// wait for every member that started, also after a failure: its copies still read cs16 and write pcm
	for (size_t i = 0; i < g->mb.size(); i++) {
		if (!started[i]) { continue; }
		cudaError_t e = cudaSetDevice(g->mb[i].device);
		if (e == cudaSuccess) { e = cudaStreamSynchronize((cudaStream_t)rxb200_fm_stream(g->mb[i].h)); }
		if (e != cudaSuccess && rc == RXB200_OK) {
			set_error("member %d: cudaStreamSynchronize failed: %s", (int)i, cudaGetErrorString(e));
			rc = RXB200_ECUDA;
		}
	}
	if (rc == RXB200_OK && n_pcm) { *n_pcm = total; }
	return rc;
}

int group_squelch_hits(Group *g, int *hits)
{
	if (!g || !hits) { return RXB200_EINVAL; }
	DeviceGuard guard;
	for (const Member &mb : g->mb) {
		if (!mb.h) { continue; }
		const int rc = rxb200_fm_squelch_hits(mb.h, hits + mb.ch_begin);
		if (rc != RXB200_OK) { return rc; }
	}
	return RXB200_OK;
}

int group_levels(Group *g, int *levels, size_t cap, size_t *n_chunks)
{
	if (!g || !levels || !n_chunks) { set_error("null argument"); return RXB200_EINVAL; }
	DeviceGuard guard;
	// every member holds the same chunk count; member 0 always owns a channel.  A zero capacity only asks for the count
	size_t nc = 0;
	int rc = rxb200_fm_levels(g->mb[0].h, levels, 0, &nc);
	if (rc != RXB200_OK && rc != RXB200_ECAPACITY) { return rc; }
	*n_chunks = nc;
	const size_t cells = nc * (size_t)g->n_channels;
	if (cap < cells) { set_error("levels capacity %zu < %zu", cap, cells); return RXB200_ECAPACITY; }
	for (size_t i = 0; i < g->mb.size() && cells; i++) {
		const Member &mb = g->mb[i];
		if (!mb.h) { continue; }
		const size_t b = (size_t)mb.ch_begin, e = (size_t)mb.ch_end;
		size_t member_chunks = 0;
		rc = rxb200_fm_levels(mb.h, levels + b * nc, (e - b) * nc, &member_chunks);
		if (rc != RXB200_OK) { return rc; }
	}
	return RXB200_OK;
}

int group_reset(Group *g)
{
	if (!g) { return RXB200_EINVAL; }
	DeviceGuard guard;
	for (const Member &mb : g->mb) {
		if (!mb.h) { continue; }
		const int rc = mb.m ? rxb200_fm_mix_reset(mb.m) : rxb200_fm_reset(mb.h);
		if (rc != RXB200_OK) { return rc; }
	}
	return RXB200_OK;
}

}  // namespace

// ---- channel streams: rxb200_fm_group_*
extern "C" void rxb200_fm_group_destroy(rxb200_fm_group *g) { group_destroy(g); }

extern "C" int rxb200_fm_group_create(const rxb200_fm_params *params, int n_channels, int n_dev, const int *devices,
                                      rxb200_fm_group **out)
{
	if (!params || !out || n_channels < 1 || n_dev < 1) { set_error("bad group arguments (n_channels >= 1, n_dev >= 1)"); return RXB200_EINVAL; }
	*out = nullptr;
	return group_create(n_channels, n_dev, devices,
	                    [&](Member &mb, int nch) { return rxb200_fm_create(params, mb.device, nch, &mb.h); }, out);
}

extern "C" int rxb200_fm_group_size(const rxb200_fm_group *g) { return g ? (int)g->mb.size() : 0; }

extern "C" rxb200_fm *rxb200_fm_group_member(rxb200_fm_group *g, int i)
{
	return (g && i >= 0 && i < (int)g->mb.size()) ? g->mb[(size_t)i].h : nullptr;
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

extern "C" int rxb200_fm_group_squelch_hits(rxb200_fm_group *g, int *hits) { return group_squelch_hits(g, hits); }

extern "C" int rxb200_fm_group_levels(rxb200_fm_group *g, int *levels, size_t cap, size_t *n_chunks)
{
	return group_levels(g, levels, cap, n_chunks);
}

extern "C" int rxb200_fm_group_reset(rxb200_fm_group *g) { return group_reset(g); }

// ---- channels of one capture: rxb200_fm_mix_group_*
extern "C" void rxb200_fm_mix_group_destroy(rxb200_fm_mix_group *g) { group_destroy(g); }

namespace {

// rxb200_fm_mix_group_create and rxb200_fm_mix_group_create_ddc (ddc != NULL: decimating members)
int mix_group_create(const rxb200_fm_params *params, int capture_rate, const int *offsets_hz, int n_channels,
                     const rxb200_ddc *ddc, int n_dev, const int *devices, rxb200_fm_mix_group **out)
{
	if (!params || !offsets_hz || !out || n_channels < 1 || n_dev < 1) {
		set_error("bad mix group arguments (n_channels >= 1, n_dev >= 1)");
		return RXB200_EINVAL;
	}
	*out = nullptr;
	if (ddc) {
		const int rc = rxb::ddc_check(ddc, nullptr);
		if (rc != RXB200_OK) { return rc; }
	}
	// every channel's table first, so that a bad offset on any member is refused before any device work
	for (int k = 0; k < n_channels; k++) {
		size_t period = 0;
		const int rc = rxb200_fm_mix_table(capture_rate, offsets_hz[k], nullptr, 0, &period);
		if (rc != RXB200_ECAPACITY) { return rc; }
	}
	return group_create(n_channels, n_dev, devices, [&](Member &mb, int nch) {
		const int *offs = offsets_hz + mb.ch_begin;
		const int rc = ddc ? rxb200_fm_mix_create_ddc(params, capture_rate, offs, nch, ddc, mb.device, &mb.m)
		                   : rxb200_fm_mix_create(params, capture_rate, offs, nch, mb.device, &mb.m);
		mb.h = rxb200_fm_mix_member(mb.m);
		return rc;
	}, out);
}

}  // namespace

extern "C" int rxb200_fm_mix_group_create(const rxb200_fm_params *params, int capture_rate, const int *offsets_hz,
                                          int n_channels, int n_dev, const int *devices, rxb200_fm_mix_group **out)
{
	return mix_group_create(params, capture_rate, offsets_hz, n_channels, nullptr, n_dev, devices, out);
}

extern "C" int rxb200_fm_mix_group_create_ddc(const rxb200_fm_params *params, int capture_rate, const int *offsets_hz,
                                              int n_channels, const rxb200_ddc *ddc, int n_dev, const int *devices,
                                              rxb200_fm_mix_group **out)
{
	if (!ddc) { set_error("null ddc"); return RXB200_EINVAL; }
	return mix_group_create(params, capture_rate, offsets_hz, n_channels, ddc, n_dev, devices, out);
}

extern "C" int rxb200_fm_mix_group_size(const rxb200_fm_mix_group *g) { return g ? (int)g->mb.size() : 0; }

extern "C" rxb200_fm_mix *rxb200_fm_mix_group_member(rxb200_fm_mix_group *g, int i)
{
	return (g && i >= 0 && i < (int)g->mb.size()) ? g->mb[(size_t)i].m : nullptr;
}

extern "C" int rxb200_fm_mix_group_process(rxb200_fm_mix_group *g, const int16_t *cs16, size_t n_int16,
                                           size_t chunk_int16, int16_t *pcm, size_t pcm_stride, size_t *n_pcm,
                                           int *chunk_result_len)
{
	return group_process(g, cs16, n_int16, chunk_int16, pcm, pcm_stride, n_pcm, chunk_result_len, false);
}

extern "C" int rxb200_fm_mix_group_process_read(rxb200_fm_mix_group *g, const int16_t *cs16, size_t n_int16,
                                                int16_t *pcm, size_t pcm_stride, size_t *n_pcm)
{
	return group_process(g, cs16, n_int16, n_int16, pcm, pcm_stride, n_pcm, nullptr, true);
}

extern "C" int rxb200_fm_mix_group_squelch_hits(rxb200_fm_mix_group *g, int *hits) { return group_squelch_hits(g, hits); }

extern "C" int rxb200_fm_mix_group_levels(rxb200_fm_mix_group *g, int *levels, size_t cap, size_t *n_chunks)
{
	return group_levels(g, levels, cap, n_chunks);
}

extern "C" int rxb200_fm_mix_group_reset(rxb200_fm_mix_group *g) { return group_reset(g); }
