// input_stage.cuh — a capture handle's input format (include/rxb200.h, "capture handles in a device's own format"):
// rxb200_fm_mix and rxb200_sdr_mix through their CaptureFront (capture_front.cuh), and rxb200_power_mix.  Once a
// handle's _set_input_format picks CS8, CU8 or CS12, each call's elements go through sdr_convert_kernel's widening kind
// into a CS16 scratch buffer on the handle's stream, ahead of everything else, and the rest of the handle (the
// resampler when attached, then the front) runs on that buffer unchanged.  The stage carries no state between calls.
// Its host code is in sdr_kernels.cu.
#pragma once
#include "common.cuh"

namespace rxb {

struct InputStage {
	int fmt = RXB200_IN_CS16;                    // RXB200_IN_*
	uint32_t *d_w = nullptr; size_t w_cap = 0;   // the widened samples of the current call (words)

	bool on() const { return fmt != RXB200_IN_CS16; }
	// bytes of c complex elements in the format
	size_t bytes(size_t c) const { return c * (fmt == RXB200_IN_CS16 ? 4 : fmt == RXB200_IN_CS12 ? 3 : 2); }
	// the format, RXB200_EINVAL for an unknown one; no device work
	int set(int in_fmt);
	// One call's widening on st: the c elements at src (a device pointer, any byte address unless CS16) to the c CS16
	// samples at *out (d_w; src itself for CS16).
	int run(const void *src, size_t c, cudaStream_t st, const uint32_t **out);
	// frees the scratch once no kernel of the stage's is in flight
	void release();
};

}  // namespace rxb
