// fm_rows.cuh — the "row" front end of the split rx_fm kernel (included by fm_kernels.cu inside namespace rxb).
//
// The segment front end (front_item) gives every THREAD its own contiguous segment: the price is a halo of
// 16 decimated samples replayed per thread (16 % of the work at 824-sample segments) and one private 32-byte
// load stream per thread.  Here a WARP owns a contiguous stretch of the stream and walks it in rows of
// ROW_LEN = 1024 input samples; lane l takes samples [32 l, 32 l + 32) of the row.  The finite-memory chain
//   scale (src/rtl_fm.c:846) -> rotate16_90 (:309) -> fifth_order x P (:411) -> generic_fir (:442) -> fm_demod (:584)
// is evaluated level by level on the lane's block; what a level needs from BEFORE the block (the last five
// inputs of that level, nine for the droop FIR, one for the discriminator) is the neighbouring lane's tail,
// handed over through a 1.8 KB per-warp exchange area in shared memory (lane 0 receives lane 31's tail of
// the previous row).  Nothing is replayed per lane; a warp rebuilds the state in front of its stretch from the last
// 128 input samples of the row before it (row_start_state: the chain's memory is shorter than that).
//
// An item's back end also needs the PCM of the `n_extra` (rows_margin) rows before the item's own rows.  Those rows
// belong to the previous items of the channel: each item's front end publishes the PCM of its last n_extra rows to a
// per-item slot in global memory (rows_publish), and the back end copies it from there (rows_collect), so no row is
// computed twice.
//
// Input: a row is 32 lines of 128 bytes, one per lane.  A per-lane 128-byte load spreads every warp-wide load
// instruction over 32 lines, 16 bytes in each (Hopper has no 256-bit load); instead each front-end warp has a ring of
// ROWS_STAGES row buffers in shared memory that a 2-D tensor copy (one box = one row, 128-byte swizzle) fills, and
// lanes read their line back with conflict-free 128-bit shared loads.
//
// Per-chunk semantics stay literal (SURVEY F7, F8): a chunk is a whole number of rows, so only lane 0 of a
// chunk's first row sees the boundary -- there every pass drops its pending odd sample (the history is taken
// one sample older) and the first discriminator output goes through atan2.
#pragma once

#define ROW_LANE 32                    // input samples per lane per row
#define ROW_LEN (32 * ROW_LANE)        // input samples per warp row
#define ROW_BYTES (4 * ROW_LEN)        // one row of CS16 input
#ifndef ROWS_STAGES
#define ROWS_STAGES 2                  // row buffers per front-end warp
#endif

template <int P>
struct RowSmem {                       // word offsets inside a warp's exchange area
	static constexpr int NV = ROW_LANE >> P;                 // decimated samples per lane per row
	static constexpr int SLOTQ = 0;                          // uint4[32]: words 0..3 of lane l's tail at index l + 1
	static constexpr int SLOTD = 128;                        // uint2[32]: words 4..5 (two arrays: no bank conflicts at 16 / 8 byte strides)
	static constexpr int CARRY = 192;                        // [3 levels][2 parities][8]: lane 31's tail of a row
	static constexpr int VRING = CARRY + 48;                 // [12 + 32 NV]: droop FIR inputs, 12 of the previous row first
	static constexpr int FPRE = VRING + 12 + 32 * NV;        // [2 parities]: last FIR output of a row (raw I/Q pair)
	static constexpr int WORDS = FPRE + 4;
};

// A warp's input ring: stage s of the warp's ROWS_STAGES row buffers (1024-byte aligned, as the 128-byte swizzle
// requires) and its mbarrier.  `line` = first 128-byte line of the row in the tensor map (channel ch, row r:
// ch * n / 32 + 32 r); only lane 0 calls this.
struct RowRing {
	const CUtensorMap *map;
	uint8_t *buf;                      // [ROWS_STAGES][ROW_BYTES]
	uint64_t *bar;                     // [ROWS_STAGES]
	uint32_t seq;                      // rows this warp has consumed so far: stage seq % S, phase (seq / S) & 1
	__device__ __forceinline__ void issue(int stage, int line)
	{
		mbar_expect_tx(&bar[stage], ROW_BYTES);
		tensor_load_2d(buf + stage * ROW_BYTES, map, 0, line, &bar[stage]);
	}
};

// a lane's 32 samples of the current row from its stage.  The copy swizzles 16-byte chunk q of line l to chunk
// q ^ (l & 7): eight consecutive lanes then read eight different bank groups.
__device__ __forceinline__ void row_read(const uint8_t *stage, int lane, uint32_t (&v)[ROW_LANE])
{
	const uint8_t *line = stage + 128 * lane;
#pragma unroll
	for (int q = 0; q < ROW_LANE / 4; q++) {
		const uint4 w = *reinterpret_cast<const uint4 *>(line + 16 * (q ^ (lane & 7)));
		v[4 * q] = w.x; v[4 * q + 1] = w.y; v[4 * q + 2] = w.z; v[4 * q + 3] = w.w;
	}
}

// hand the level's tail (its last six inputs, oldest first) to the next lane and fetch the five inputs before this
// lane's block.  cs0: lane 0 of a chunk's first row -- the pass forgot its pending odd sample, the history is one older.
// CS: the row starts a chunk (a separate instantiation of the whole row, so the common rows carry none of this).
template <bool CS>
__device__ __forceinline__ void row_exchange(uint32_t *xs, int carry_w, int carry_r, int lane,
                                             uint32_t t0, uint32_t t1, uint32_t t2, uint32_t t3, uint32_t t4, uint32_t t5,
                                             uint32_t (&h)[5])
{
	__syncwarp();                          // the slots' previous readers are done
	uint32_t *wq = (lane == 31) ? xs + carry_w : xs + 4 * (lane + 1);
	uint32_t *wd = (lane == 31) ? xs + carry_w + 4 : xs + 128 + 2 * (lane + 1);
	*reinterpret_cast<uint4 *>(wq) = make_uint4(t0, t1, t2, t3);
	*reinterpret_cast<uint2 *>(wd) = make_uint2(t4, t5);
	__syncwarp();
	const uint32_t *rq = (lane == 0) ? xs + carry_r : xs + 4 * lane;
	const uint32_t *rd = (lane == 0) ? xs + carry_r + 4 : xs + 128 + 2 * lane;
	const uint4 a = *reinterpret_cast<const uint4 *>(rq);
	const uint2 b = *reinterpret_cast<const uint2 *>(rd);
	h[0] = a.y; h[1] = a.z; h[2] = a.w; h[3] = b.x; h[4] = b.y;
	if (CS && lane == 0) { h[4] = b.x; h[3] = a.w; h[2] = a.z; h[1] = a.y; h[0] = a.x; }
}

// one fifth_order pass over the lane's M inputs -> M/2 outputs (src/rtl_fm.c:411-440); output j is the tap set over
// inputs 2j-5 .. 2j of the level's sequence
template <int M, bool CS>
__device__ __forceinline__ void row_level(uint32_t *xs, int carry_w, int carry_r, int lane,
                                          const uint32_t (&in)[M], uint32_t (&out)[M / 2])
{
	uint32_t h[5];
	row_exchange<CS>(xs, carry_w, carry_r, lane, in[M - 6], in[M - 5], in[M - 4], in[M - 3], in[M - 2], in[M - 1], h);
	// (computing the outputs that need no history first, to give the exchange time, measured 1 % slower)
	out[0] = hb_tap(h[0], h[1], h[2], h[3], h[4], in[0]);
	out[1] = hb_tap(h[2], h[3], h[4], in[0], in[1], in[2]);
	out[2] = hb_tap(h[4], in[0], in[1], in[2], in[3], in[4]);
#pragma unroll
	for (int j = 3; j < M / 2; j++) { out[j] = hb_tap(in[2 * j - 5], in[2 * j - 4], in[2 * j - 3], in[2 * j - 2], in[2 * j - 1], in[2 * j]); }
}

// generic_fir (src/rtl_fm.c:442-465) on nine explicit history words whose lanes are biased by FIR_B (see droop9_packed)
__device__ __forceinline__ void droop9_words(const int (&c)[6], int fir_bias, uint32_t h0, uint32_t h1, uint32_t h2, uint32_t h3,
                                             uint32_t h4, uint32_t h5, uint32_t h6, uint32_t h7, uint32_t h8, int &di, int &dq)
{
	const uint32_t s0 = h0 + h8, s1 = h1 + h7, s2 = h2 + h6, s3 = h3 + h5, s4 = h4;
	int ai = sub_w(mul_w((int)(s0 & 0xffffu), c[1]), fir_bias);
	int aq = sub_w(mul_w((int)(s0 >> 16), c[1]), fir_bias);
	ai = add_w(ai, mul_w((int)(s1 & 0xffffu), c[2])); aq = add_w(aq, mul_w((int)(s1 >> 16), c[2]));
	ai = add_w(ai, mul_w((int)(s2 & 0xffffu), c[3])); aq = add_w(aq, mul_w((int)(s2 >> 16), c[3]));
	ai = add_w(ai, mul_w((int)(s3 & 0xffffu), c[4])); aq = add_w(aq, mul_w((int)(s3 >> 16), c[4]));
	ai = add_w(ai, mul_w((int)(s4 & 0xffffu), c[5])); aq = add_w(aq, mul_w((int)(s4 >> 16), c[5]));
	di = wrap16(ai >> 15);
	dq = wrap16(aq >> 15);
}

// ||x| - |y|| of fast_atan2 for the conjugate product (cr, cj); its 4096 (|x| - |y|) leaves int32 from 2^19 on, where
// FP32 does not wrap with it
__device__ __forceinline__ float row_angle_n(int cr, int cj)
{
	return fabsf(__fsub_rn(fabsf(__int2float_rn(cr)), fabsf(__int2float_rn(cj))));
}

// A lane's NV discriminator outputs as the low 16 bits of angle + 1.5 * 2^23.  WRAPS: operands whose product leaves
// int32 take the integer form.
template <int NV, bool CS, bool WRAPS>
__device__ __forceinline__ void row_angles(const int *cr, const int *cj, int lane, uint32_t *ab)
{
#pragma unroll
	for (int j = 0; j < NV; j++) {
		float ang = fast_atan2_f32(__int2float_rn(cj[j]), __int2float_rn(cr[j]));
		if (WRAPS && row_angle_n(cr[j], cj[j]) >= 524288.0f) { ang = __int2float_rn(fast_atan2_i(cj[j], cr[j])); }
		if (CS && j == 0 && lane == 0) { ang = __int2float_rn(disc_std(cr[0], cj[0])); }   // F8: the first sample of a chunk goes through atan2
		ab[j] = (uint32_t)__float_as_int(__fadd_rn(ang, 12582912.0f));      // low 16 bits of angle + 1.5 * 2^23: the int16 value
	}
}

// One row of one lane, read from stage `stage` of the ring.  Once level 0 is through (its exchange has every lane's
// inputs consumed) lane 0 refills the stage with the row ROWS_STAGES ahead, at `next_line` (< 0: none left).
// par = parity of the row (which carry slot lane 31 writes); CS = the row starts a chunk;
// rel = index of the lane's first PCM sample in the item's shared PCM buffer.
template <int P, bool FIR, bool CS>
__device__ __forceinline__ void row_body(const FmDev &c, uint32_t *xs, int par, int lane,
                                         RowRing &ring, int stage, int next_line, int16_t *pcm_s, int rel)
{
	typedef RowSmem<P> RS;
	constexpr int NV = RS::NV;
	uint32_t o[NV];                        // the lane's decimated samples, lanes biased by 128 << P
	{
		uint32_t y[ROW_LANE / 2];
		{
			uint32_t x[ROW_LANE];
			{
				uint32_t v[ROW_LANE];
				row_read(ring.buf + stage * ROW_BYTES, lane, v);
#pragma unroll
				for (int j = 0; j < ROW_LANE; j++) { x[j] = scale_rot_pack(v[j], j, true); }
			}
			row_level<ROW_LANE, CS>(xs, RS::CARRY + (0 * 2 + par) * 8, RS::CARRY + (0 * 2 + (par ^ 1)) * 8, lane, x, y);
		}
		if (lane == 0 && next_line >= 0) { ring.issue(stage, next_line); }
		if constexpr (P == 1) {
#pragma unroll
			for (int j = 0; j < NV; j++) { o[j] = y[j]; }
		} else {
			uint32_t z[ROW_LANE / 4];
			row_level<ROW_LANE / 2, CS>(xs, RS::CARRY + (1 * 2 + par) * 8, RS::CARRY + (1 * 2 + (par ^ 1)) * 8, lane, y, z);
			if constexpr (P == 2) {
#pragma unroll
				for (int j = 0; j < NV; j++) { o[j] = z[j]; }
			} else {
				row_level<ROW_LANE / 4, CS>(xs, RS::CARRY + (2 * 2 + par) * 8, RS::CARRY + (2 * 2 + (par ^ 1)) * 8, lane, z, o);
			}
		}
	}
	constexpr int BO = 128 << P;
	int di[NV], dq[NV];
	if constexpr (FIR) {
		// droop FIR over the previous nine decimated samples: the row's samples sit in a linear ring, twelve of the
		// previous row in front, so lane l's history is simply the nine words before its own
		uint32_t ob[NV];
#pragma unroll
		for (int j = 0; j < NV; j++) { ob[j] = o[j] + (FIR_B - (unsigned)BO) * 0x10001u; }
		uint32_t *vr = xs + RS::VRING;
		__syncwarp();
#pragma unroll
		for (int j = 0; j < NV; j += 4) { *reinterpret_cast<uint4 *>(vr + 12 + NV * lane + j) = make_uint4(ob[j], ob[j + 1], ob[j + 2], ob[j + 3]); }
		__syncwarp();
		uint32_t s[9 + NV];
		{
			const uint4 a = *reinterpret_cast<const uint4 *>(vr + NV * lane);
			const uint4 b = *reinterpret_cast<const uint4 *>(vr + NV * lane + 4);
			const uint4 d = *reinterpret_cast<const uint4 *>(vr + NV * lane + 8);
			s[0] = a.w; s[1] = b.x; s[2] = b.y; s[3] = b.z; s[4] = b.w; s[5] = d.x; s[6] = d.y; s[7] = d.z; s[8] = d.w;
		}
#pragma unroll
		for (int j = 0; j < NV; j++) { s[9 + j] = ob[j]; }
#pragma unroll
		for (int j = 0; j < NV; j++) {
			droop9_words(c.fir, c.fir_bias, s[j], s[j + 1], s[j + 2], s[j + 3], s[j + 4], s[j + 5], s[j + 6], s[j + 7], s[j + 8], di[j], dq[j]);
		}
		__syncwarp();                      // every lane has its history: the ring's tail moves to the front for the next row
		if (lane < 12) { vr[lane] = vr[32 * NV + lane]; }
	} else {
#pragma unroll
		for (int j = 0; j < NV; j++) { di[j] = (int)(o[j] & 0xffffu) - BO; dq[j] = (int)(o[j] >> 16) - BO; }
	}
	// fm_demod (src/rtl_fm.c:584-615): x[n] * conj(x[n-1]) -> fast_atan2; the sample before the block is the neighbour's last
	const uint32_t last = pack2(di[NV - 1], dq[NV - 1]);
	uint32_t prev = __shfl_up_sync(0xffffffffu, last, 1);
	if (lane == 31) { xs[RS::FPRE + par] = last; }
	if (lane == 0) { prev = xs[RS::FPRE + (par ^ 1)]; }
	int br = lo16(prev), bj = hi16(prev);
	int cr[NV], cj[NV];
#pragma unroll
	for (int j = 0; j < NV; j++) {
		cr[j] = add_w(mul_w(di[j], br), mul_w(dq[j], bj));
		cj[j] = sub_w(mul_w(dq[j], br), mul_w(di[j], bj));
		br = di[j]; bj = dq[j];
	}
	// fast_atan2 in FP32 (fast_atan2_f32: every quantity an integer a float holds exactly).  Its operands always fit: the
	// chain from the 8-bit-range samples to here is linear with non-negative half-band taps, so |d| <= 128 * sum|g| with g
	// the combined response of the P passes and the droop FIR -- 405 / 835 / 1684 for P = 1 / 2 / 3 (1024 without the FIR),
	// plus less than 32 for the floors -- and |cr| + |cj| <= 4 d^2 < 1.2e7 < 2^24
	// (tests/test_host_logic.py::test_row_discriminator_operands_fit_fp32 recomputes the bound from the table).
	// The FP32 form issues every cycle and leaves the adder pipe, which bounds this loop, ~16 instructions per output
	// lighter than the integer form (DESIGN.md §4.1).  One case it does not reproduce: the reference's 4096 (|x| - |y|)
	// wraps in int32 once ||x| - |y|| >= 2^19 (decimated samples beyond ~724, e.g. from full-scale noise).  A row in which
	// some lane has such an operand, rare, takes row_angles<..., true>, where those operands go through the integer form,
	// which wraps the same way; every other row keeps the straight FP32 loop.
	uint32_t wpk[NV / 2];                  // PCM, two samples per word
	{
		uint32_t ab[NV];
		bool wraps = false;
#pragma unroll
		for (int j = 0; j < NV; j++) { wraps |= row_angle_n(cr[j], cj[j]) >= 524288.0f; }
		if (__any_sync(0xffffffffu, wraps)) { row_angles<NV, CS, true>(cr, cj, lane, ab); }
		else { row_angles<NV, CS, false>(cr, cj, lane, ab); }
#pragma unroll
		for (int j = 0; j < NV; j += 2) { wpk[j / 2] = __byte_perm(ab[j], ab[j + 1], 0x5410); }
	}
	int16_t *dst = pcm_s + pcm_phys<PCM_PAD_ROWS>(rel);
#pragma unroll
	for (int j = 0; j < NV; j += 4) {
		uint2 w;
		w.x = wpk[j / 2]; w.y = wpk[j / 2 + 1];
		*reinterpret_cast<uint2 *>(dst + j) = w;
	}
}

// What a row leaves behind for the next one -- lane 31's tails at every level (CARRY), the droop FIR's last inputs
// (VRING) and the last FIR output (FPRE) -- from the row's last 128 input samples `v` (4 per lane), written to the
// parity-1 slots, which the first row of a stretch (parity 0) reads.  Every pass, the droop FIR and the discriminator
// have finite memory: window output j of a pass needs its inputs 2j-5 .. 2j, so the window's y are exact from y[3] on,
// its z from z[4], its o (P = 3) from o[5].  What is written needs no more than x[122..], y[58..], z[26..] and the last
// ten o, so no word of it depends on anything before the window (tests/test_rows_reach.py pins this on the port).
// Chunks start on row boundaries, so no chunk start (F7, F8) falls inside the window.
template <int P, bool FIR>
__device__ __forceinline__ void row_start_state(const FmDev &c, uint4 v, uint32_t *xs, int lane)
{
	typedef RowSmem<P> RS;
	constexpr unsigned FULL = 0xffffffffu;
	uint32_t *cw = xs + RS::CARRY;                        // [level][parity][8]; parity 1 is at + 8
	// level 0: x[4l .. 4l+3], five inputs of history from lanes l-1 and l-2 -> y[2l], y[2l+1]
	const uint32_t x0 = scale_rot_pack(v.x, 0, true), x1 = scale_rot_pack(v.y, 1, true);
	const uint32_t x2 = scale_rot_pack(v.z, 2, true), x3 = scale_rot_pack(v.w, 3, true);
	uint32_t h0 = __shfl_up_sync(FULL, x3, 2), h1 = __shfl_up_sync(FULL, x0, 1), h2 = __shfl_up_sync(FULL, x1, 1);
	uint32_t h3 = __shfl_up_sync(FULL, x2, 1), h4 = __shfl_up_sync(FULL, x3, 1);
	const uint32_t y0 = hb_tap(h0, h1, h2, h3, h4, x0), y1 = hb_tap(h2, h3, h4, x0, x1, x2);
	if (lane == 31) {
		*reinterpret_cast<uint4 *>(cw + 8) = make_uint4(h3, h4, x0, x1);
		*reinterpret_cast<uint2 *>(cw + 8 + 4) = make_uint2(x2, x3);
	}
	uint32_t o0, o1 = 0u;                                 // the lane's decimated samples (P = 1: two, else one)
	int m0, m1 = -1;                                      // their indices among the window's M decimated samples
	constexpr int M = 128 >> P;
	if constexpr (P == 1) {
		o0 = y0; o1 = y1; m0 = 2 * lane; m1 = 2 * lane + 1;
	} else {
		// level 1: y[2l], y[2l+1], history from lanes l-1 .. l-3 -> z[l]
		h0 = __shfl_up_sync(FULL, y1, 3); h1 = __shfl_up_sync(FULL, y0, 2); h2 = __shfl_up_sync(FULL, y1, 2);
		h3 = __shfl_up_sync(FULL, y0, 1); h4 = __shfl_up_sync(FULL, y1, 1);
		const uint32_t z = hb_tap(h0, h1, h2, h3, h4, y0);
		if (lane == 31) {
			*reinterpret_cast<uint4 *>(cw + 24) = make_uint4(h1, h2, h3, h4);
			*reinterpret_cast<uint2 *>(cw + 24 + 4) = make_uint2(y0, y1);
		}
		if constexpr (P == 2) {
			o0 = z; m0 = lane;
		} else {
			// level 2: z[l-5 .. l] -> o[l / 2] on the even lanes
			h0 = __shfl_up_sync(FULL, z, 5); h1 = __shfl_up_sync(FULL, z, 4); h2 = __shfl_up_sync(FULL, z, 3);
			h3 = __shfl_up_sync(FULL, z, 2); h4 = __shfl_up_sync(FULL, z, 1);
			o0 = hb_tap(h0, h1, h2, h3, h4, z); m0 = (lane & 1) ? -1 : lane >> 1;
			if (lane == 31) {
				*reinterpret_cast<uint4 *>(cw + 40) = make_uint4(h0, h1, h2, h3);
				*reinterpret_cast<uint2 *>(cw + 40 + 4) = make_uint2(h4, z);
			}
		}
	}
	constexpr int BO = 128 << P;
	if constexpr (FIR) {
		// the last ten o, biased, go where a row leaves its last twelve (VRING[m - M + 12]); the next row reads [3, 12),
		// the last FIR output is the filter over [2, 11)
		uint32_t *vr = xs + RS::VRING;
		if (m0 >= M - 10) { vr[m0 - M + 12] = o0 + (FIR_B - (unsigned)BO) * 0x10001u; }
		if (m1 >= M - 10) { vr[m1 - M + 12] = o1 + (FIR_B - (unsigned)BO) * 0x10001u; }
		__syncwarp();
		if (lane == 0) {
			int di, dq;
			droop9_words(c.fir, c.fir_bias, vr[2], vr[3], vr[4], vr[5], vr[6], vr[7], vr[8], vr[9], vr[10], di, dq);
			xs[RS::FPRE + 1] = pack2(di, dq);
		}
	} else {
		const uint32_t last = (P == 1) ? o1 : o0;
		if (m0 == M - 1 || m1 == M - 1) { xs[RS::FPRE + 1] = pack2((int)(last & 0xffffu) - BO, (int)(last >> 16) - BO); }
	}
}

// The rows [r0, r1) of one work item that this warp owns (rows are counted from the start of the channel's call).
// The item's rows [own_lo, own_hi) split evenly over the front-end warps; the margin rows before own_lo come from
// the previous items (rows_collect).
template <int P, bool FIR>
__device__ __forceinline__ void front_rows(const FmDev &c, const FmCall &k, const Item &it, int warp, int lane,
                                           int16_t *pcm_s, uint32_t *xs, RowRing &ring)
{
	typedef RowSmem<P> RS;
	constexpr int NV = RS::NV;
	// rows fit 32 bits (a call is at most 2^31 samples per channel)
	const int rows_total = (int)(k.n / ROW_LEN);
	const int own_lo = it.b * k.n_own;
	const int own_hi = own_lo + k.n_own < rows_total ? own_lo + k.n_own : rows_total;
	const int per = (own_hi - own_lo + k.fe_warps - 1) / k.fe_warps;
	const int r0 = own_lo + warp * per;
	const int r1 = r0 + per < own_hi ? r0 + per : own_hi;
	if (r0 >= r1) { return; }
	// line walks the rows' tensor-map coordinates; rows_left counts the loop; to_cs counts down to the next chunk start.
	// Every row this warp copies it also consumes, so the ring is empty between items.
	constexpr int S = ROWS_STAGES;
	const int line0 = it.ch * (int)(k.n / 32) + 32 * r0;
	int rows_left = r1 - r0;
	if (lane == 0) {
		for (int i = 0; i < S && i < rows_left; i++) { ring.issue((int)((ring.seq + i) % S), line0 + 32 * i); }
	}
	// what the row before the first one left behind: the call's carry at the start of the stream, else rebuilt from
	// that row's last 128 samples (one coalesced 512-byte load; the input is not written during the launch)
	const uint32_t *carry = k.carry_in + (size_t)it.ch * k.state_words;
	uint4 tail = make_uint4(0u, 0u, 0u, 0u);
	if (r0 > 0) { tail = __ldg(reinterpret_cast<const uint4 *>(k.in) + ((size_t)it.ch * (size_t)k.n + (size_t)r0 * ROW_LEN - 128) / 4 + lane); }
	__syncwarp();
	if (r0 == 0) {
		if (lane < 6) {
#pragma unroll
			for (int l = 0; l < P; l++) { xs[RS::CARRY + (l * 2 + 1) * 8 + lane] = carry[ST_HDR + 6 * l + lane]; }
		}
		if (FIR && lane < 9) { xs[RS::VRING + 3 + lane] = fir_bias_lanes(carry[ST_HDR + 6 * P + lane]); }
		if (lane == 0) { xs[RS::FPRE + 1] = pack2((int)carry[ST_PRE_I], (int)carry[ST_PRE_Q]); }
	} else {
		row_start_state<P, FIR>(c, tail, xs, lane);
	}
	__syncwarp();
	const int rpc = k.chunk / ROW_LEN;              // rows per chunk
	int par = 0;
	int to_cs = r0 % rpc;                           // 0: this row starts a chunk
	int rel = (int)((((long long)r0 * ROW_LEN) >> P) - it.m_lo) + NV * lane;
	for (int i = 0; rows_left > 0; rows_left--, i++) {
		const int stage = (int)(ring.seq % S);
		mbar_wait(&ring.bar[stage], (ring.seq / S) & 1u);
		const int next_line = rows_left > S ? line0 + 32 * (i + S) : -1;
		// a chunk's first row is its own instantiation (warp-uniform branch): the common rows carry no trace of it
		if (to_cs == 0) { row_body<P, FIR, true>(c, xs, par, lane, ring, stage, next_line, pcm_s, rel); }
		else { row_body<P, FIR, false>(c, xs, par, lane, ring, stage, next_line, pcm_s, rel); }
		ring.seq++;
		par ^= 1;
		rel += ROW_LEN >> P;
		if (++to_cs == rpc) { to_cs = 0; }
	}
	if (r1 == rows_total) {
		// this warp saw the end of the stream: lane 31's tails are the next call's carry (same layout as front_store)
		__syncwarp();
		uint32_t *co = k.carry_out + (size_t)it.ch * k.state_words;
		const int pl = par ^ 1;                     // parity of the last row
		if (lane < 6) {
#pragma unroll
			for (int l = 0; l < P; l++) { co[ST_HDR + 6 * l + lane] = xs[RS::CARRY + (l * 2 + pl) * 8 + lane]; }
		}
		if (FIR && lane < 9) { co[ST_HDR + 6 * P + lane] = fir_unbias_lanes(xs[RS::VRING + 3 + lane]); }
		if (lane == 0) {
			const uint32_t f = xs[RS::FPRE + pl];
			co[ST_PRE_I] = (uint32_t)lo16(f); co[ST_PRE_Q] = (uint32_t)hi16(f);
			co[ST_BOX_I] = 0u; co[ST_BOX_Q] = 0u; co[ST_BOX_N] = 0u;
		}
	}
}

// ---- margin hand-over between the items of a channel.  Item w's slot in k.margin holds n_extra rows of PCM: row r of
// the item sits at (r - (own_hi - n_extra)) * row_pcm, and only its own rows are written.  pub[4 w + 2] = 1 says the
// slot is complete.  (PCM_PAD_ROWS is 0: the shared buffer is linear.)
#define BAR_PUB 3
__device__ __forceinline__ int ld_acquire_gpu(const int *p)
{
	int v;
	asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
}
__device__ __forceinline__ void st_release_gpu(int *p, int v) { asm volatile("st.release.gpu.global.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }

// Front end, after its own rows: the last front-end warp waits for the others' rows (the others only arrive), copies
// the item's last n_extra rows to its slot and raises the flag.  This never waits for a back end, so no item's margin
// sits behind another item's serial stages.
template <int P>
__device__ __forceinline__ void rows_publish(const FmCall &k, const Item &it, int work, const int16_t *pcm_s, int warp, int lane)
{
	if (warp != k.fe_warps - 1) { asm volatile("bar.arrive %0, %1;" ::"r"(BAR_PUB), "r"(k.fe_threads) : "memory"); return; }
	bar_sync(BAR_PUB, k.fe_threads);
	if (it.b == k.n_cta - 1) { return; }                // the channel's last item: nobody reads its margin
	constexpr int LG = 10 - P;                             // log2 of PCM samples per row
	const int own_hi = (it.b + 1) * k.n_own;             // not the last item: never clipped at the end of the call
	const int lo = it.b * k.n_own > own_hi - k.n_extra ? it.b * k.n_own : own_hi - k.n_extra;
	const uint4 *src = reinterpret_cast<const uint4 *>(pcm_s + (((long long)lo << LG) - it.m_lo));
	uint4 *dst = reinterpret_cast<uint4 *>(k.margin + ((size_t)work * k.n_extra + (lo - (own_hi - k.n_extra))) * (1 << LG));
	const int n = ((own_hi - lo) << LG) / 8;
	for (int i = lane; i < n; i += 32) { dst[i] = src[i]; }
	__syncwarp();
	if (lane == 0) { __threadfence(); st_release_gpu(k.pub + 4 * (size_t)work + 2, 1); }
}

// Back end, before pass 1: the margin rows [buf_lo, own_lo) of this item, from the slots of the older items of the
// channel that own them (up to n_extra of them when items are shorter than the margin).  Progress: these are older
// tickets, and a front end that holds a ticket waits for nothing but its own warps (it took the ticket after its
// `empty` wait), so their flags always come.  Coherent loads: the slots are written during the launch.
template <int P>
__device__ __forceinline__ void rows_collect(const FmCall &k, const Item &it, int work, int16_t *pcm_s, int q, int lanes)
{
	const int own_lo = it.b * k.n_own;
	const int buf_lo = own_lo - k.n_extra > 0 ? own_lo - k.n_extra : 0;
	if (buf_lo == own_lo) { return; }
	constexpr int LG = 10 - P;
	const int first = buf_lo / k.n_own;                  // the oldest item holding a margin row
	for (int j = first; j < it.b; j++) {
		const int *f = k.pub + 4 * (size_t)(work - (it.b - j)) + 2;
		while (ld_acquire_gpu(f) == 0) { __nanosleep(32); }
	}
	const int n = ((own_lo - buf_lo) << LG) / 8;
	uint4 *dst = reinterpret_cast<uint4 *>(pcm_s + (((long long)buf_lo << LG) - it.m_lo));
	for (int i = q; i < n; i += lanes) {
		const int r = buf_lo + ((8 * i) >> LG);
		const int j = r / k.n_own;
		const size_t e = ((size_t)(work - (it.b - j)) * k.n_extra + (r - ((j + 1) * k.n_own - k.n_extra))) * (1 << LG) + ((8 * i) & ((1 << LG) - 1));
		dst[i] = __ldcg(reinterpret_cast<const uint4 *>(k.margin + e));
	}
	bar_sync(BAR_BE, lanes);
}
