// resample_stage.cuh — the rational resampler (resample.cu) as the first stage of a capture handle: rxb200_fm_mix and
// rxb200_sdr_mix through their CaptureFront (capture_front.cuh), and rxb200_power_mix.  Once a handle's
// _set_device_rate attaches it, each call's device-rate samples go through resample_kernel into a capture-rate scratch
// buffer on the handle's stream, and the handle's front runs on that buffer.  The stage carries the device-sample count
// and the last J - 1 raw device samples: a CaptureFront commits them with its own, rx_power once a call's resampling is
// enqueued, ahead of its pass groups.  So the handle's bytes are those of the resampler's handle followed by the same
// handle without one, however the device stream is cut into calls.  Its host code is in resample.cu.
#pragma once
#include "ddc.cuh"

namespace rxb {

// the resampler's arguments: every refusal of rxb200_resample_create but the out pointer; *wide: the kernel
// accumulates in 64 bits
int resample_check(const rxb200_resampler *rs, bool *wide);
// the outputs of a call over device samples [n0, n0 + c)
size_t out_count(unsigned long long n0, size_t c, long long L, long long N);
// Launches resample_kernel on st for the outputs of a call over device samples [n0, n0 + c) at src (hist: the J - 1
// samples before it), to dst; nothing when the call has no output.
int resample_launch(long long L, long long N, int J, int S, bool wide, const int32_t *taps, const uint32_t *src,
                    const uint32_t *hist, unsigned long long n0, size_t c, uint32_t *dst, cudaStream_t st);

struct ResampleStage {
	long long L = 1, N = 1;
	DdcFilter f;                                 // T = J, S; taps: the prototype phase-major (NULL: not attached)
	unsigned long long pos = 0;                  // device samples since create or reset
	uint32_t *d_y = nullptr; size_t y_cap = 0;   // the capture-rate samples of the current call (words)

	bool on() const { return f.taps != nullptr; }
	// the capture samples a call of c device samples emits at the current count (c when not attached)
	size_t out_len(size_t c) const { return on() ? out_count(pos, c, L, N) : c; }
	// a bound on out_len(c) at any count: ceil(c L / N)
	size_t max_out(size_t c) const;
	// the refusals of rxb200_resample_create, then the taps and the zeroed history on the current device; a refused or
	// failed attach leaves the stage detached
	int attach(const rxb200_resampler *rs);
	// One call's resampling on st: the c device samples at src (a device pointer) to the out_len(c) capture samples at
	// *out (d_y; src itself when not attached), then the carry of the raw history.  Nothing becomes live before commit.
	int run(const uint32_t *src, size_t c, cudaStream_t st, const uint32_t **out);
	// the history a call of c device samples wrote becomes live, and the count advances past it
	void commit(size_t c)
	{
		if (on()) { f.commit(); pos += c; }
	}
	// the history zeroed behind any call still running on st, and the count cleared; the stage stays attached
	int reset(cudaStream_t st);
	// frees the device state once no kernel of the stage's is in flight
	void release();
};

}  // namespace rxb
