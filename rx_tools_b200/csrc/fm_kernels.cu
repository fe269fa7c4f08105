// fm_kernels.cu — rx_fm hot path on sm_90a: ONE fused kernel per call covering
//   CS16->8-bit-range scale (src/rtl_fm.c:846) -> rotate16_90 (:309) -> low_pass (:351) |
//   fifth_order x P (:411) + generic_fir (:442) -> fm_demod (:584; std/fast/lut/ale) | am/usb/lsb/raw
//   -> deemph_filter (:667) -> low_pass_real (:389)
// with no intermediate buffer in HBM (algorithmic traffic: 4 B in + 2*rate_out2/rate_capture B out
// per complex sample).
//
// Decomposition (DESIGN.md "rx_fm kernel"):
//   * A CTA (128 or 256 threads, see fm_cta_threads) owns a contiguous stretch of one channel's stream.  FRONT END: every
//     thread runs scale/rotate/decimate/FIR/discriminator over its own Sf-sample segment, all state
//     in registers, after replaying `halo` samples so the finite-memory filters are exact; the
//     demodulated PCM (one int16 per decimated sample) goes to shared memory only.
//   * BACK END: the first `be_lanes` threads run the serial stages (deemph_filter, low_pass_real)
//     over the item's PCM, one contiguous piece of OUTPUTS per lane.  deemph_filter is a rounding
//     (non-linear) IIR, so each lane replays W_dec PCM samples before its piece from BOTH extreme
//     states (-32768 / +32767): the step map is monotone in the state, the true state is
//     bracketed, and once the two trajectories meet it is exact (SURVEY.md §7 hard part 2).  A
//     bracket that stays open (quiet input: the IIR has a dead zone) is summarised per piece --
//     merged / pass-through / open -- and resolved by thread 0 plus a decoupled look-back over the
//     items' published words (items are ticketed in order, so a reader only waits for older
//     ones); those pieces then produce their outputs in a second parallel pass.  The result is
//     bit-exact for every input.
//   * The halo/warm-up PCM a CTA needs from before its stretch is recomputed by `n_extra` of its
//     own threads, so nothing but the CS16 stream is read from HBM and nothing but PCM written.
// Per-chunk semantics (rotation phase restart, fifth_order dropping the last sample of a chunk,
// first FM output of a chunk through atan2: SURVEY F7, F8) are reproduced literally: the chunk
// length is a kernel argument.
#include <math.h>
#include <string.h>
#include <stdlib.h>
#include <new>
#include <vector>
#include <cudaTypedefs.h>        // PFN_cuTensorMapEncodeTiled
#include "common.cuh"

namespace rxb {

#define FM_MAX_THREADS 256       // widest CTA; the width is a kernel template parameter (fm_cta_threads picks it)
// stream prefetch into L2 ahead of the register prefetch: every RXB_L2_MASK+1 samples, RXB_L2_AHEAD samples ahead
#define RXB_L2_MASK 31
#define RXB_L2_AHEAD 64
#define RXB_OCC 3                // resident CTAs per SM of the P <= 3 kernels, stated for 256 threads
#define FM_MAX_PACKED 3          // fifth_order passes run as packed I/Q SWAR (bias keeps lanes unsigned)
// ------------------------------------------------------------------------------ device config
struct FmDev {
	int mode, D, P, PL, fir_on, atan_mode, out_scale, post_ds;
	int deemph, a, a_half, a_even;
	unsigned a_magic; int a_K, a_use_magic;   // floor(n/a) == umulhi(n, a_magic) for the n range used
	int resample, fast, slow, lpr_div;
	int lpr_ok, lpr_m, lpr_s, lpr_add;        // acc / lpr_div (C truncation) == ((mulhi(acc, lpr_m) [+ acc]) >> lpr_s) + sign, host-verified
	int offset_tuning;
	int squelch, rdc_on, rdc_k, adc_on, adc_k;   // per-chunk reduction stages (src/rtl_fm.c:781-790, :699-721, :684-697)
	int levels;                                  // keep per-chunk rms() (-L, src/rtl_fm.c:792-806)
	int fir[6];
	int fir_bias;                                // packed droop FIR: FIR_B * (2(c1+c2+c3+c4)+c5), see droop9_packed
	const int *atan_lut;
};

struct FmCall {
	const int16_t *in;        // [n_ch][n] complex CS16
	int16_t *out;             // [n_ch][out_stride] int16
	long long n;              // complex samples per channel in this call
	long long out_stride;     // int16 per channel
	int chunk;                // complex samples per chunk
	int n_ch;
	int Sf;                   // front-end segment (complex samples per thread)
	int halo;                 // samples replayed before a segment
	int n_extra, n_own;       // thread slots: warm-up region / owned stretch
	int n_cta;                // CTAs per channel
	int W_dec;                // back-end replay length (decimated samples)
	int pcm_cap;              // int16 entries of the shared PCM buffer
	int direct_out;           // 1: no serial stage, the front end stores the output itself
	int be_lanes;             // threads of the CTA that run the back end (multiple of 32)
	int fe_threads, fe_warps; // split kernel: threads / warps of the CTA that run the front end
	int xs_words;             // split kernel, row front end: words of a warp's exchange area
	int state_words;
	const uint32_t *carry_in; // [n_ch][state_words]
	uint32_t *carry_out;      // [n_ch][state_words]
	int *ticket;              // work counter
	int *pub;                 // [n_ch*n_cta][4]  flag, avg, margin flag (row front end), -
	int16_t *margin;          // row front end: [n_ch*n_cta][n_extra * row PCM] the margin hand-over (fm_rows.cuh)
	int *fix_count;           // lanes that had to be re-run from a neighbour's state
	// per-chunk scalars of the optional reduction stages, [n_ch][n_chunks]; null when the stage is off
	const int *rdc;           // [..][2] dc_avgI, dc_avgQ subtracted in that chunk
	const int *sqz;           // 1: squelch zeroes that chunk
	const int *adc;           // audio DC average subtracted in that chunk
	long long *sums;          // [..][2] accumulators of the reduction pre-passes
	int n_chunks;
	int reduce_mode;          // 0 main pass, 1 squelch sums (t, p), 2 audio-DC sums
	int one;                  // always 1 (see front_run)
	const int16_t *pcm_g;     // fm_back_kernel: [n_ch][pcm_g_stride] PCM of the whole call in global memory (null elsewhere)
	long long pcm_g_stride;
};

// Scratch builds (-DRXB_PROF): per-warp clock64() sums of the split kernel's phases in a device array that
// tools/fm_prof.py reads back (rxb200_fm_prof_read).  Compiles to nothing by default.
#ifdef RXB_PROF
#define PROF_CTAS 1024
#define PROF_SLOTS 16
enum { PF_WARPID = 0, PF_SMID, PF_TOTAL, PF_ITEMS, PF_ROWS, PF_FRONT, PF_BAR_FE, PF_EMPTY, PF_RING, PF_PUBLISH,
       PF_FULL, PF_COLLECT, PF_PASS1, PF_CHAIN, PF_PASS2 };
__device__ unsigned long long rxb_prof[PROF_CTAS * 32 * PROF_SLOTS];
__device__ __forceinline__ unsigned long long *prof_slot(int s)
{
	return rxb_prof + ((size_t)blockIdx.x * 32 + (threadIdx.x >> 5)) * PROF_SLOTS + s;
}
#define PROF_CLK(var_) const long long var_ = clock64()
#define PROF_ADD(slot_, t_) do { if (blockIdx.x < PROF_CTAS && (threadIdx.x & 31) == 0) { *prof_slot(slot_) += (unsigned long long)(clock64() - (t_)); } } while (0)
#define PROF_SET(slot_, val_) do { if (blockIdx.x < PROF_CTAS && (threadIdx.x & 31) == 0) { *prof_slot(slot_) = (unsigned long long)(val_); } } while (0)
#define PROF_INC(slot_, val_) do { if (blockIdx.x < PROF_CTAS && (threadIdx.x & 31) == 0) { *prof_slot(slot_) += (unsigned long long)(val_); } } while (0)
#else
#define PROF_CLK(var_) do { } while (0)
#define PROF_ADD(slot_, t_) do { } while (0)
#define PROF_SET(slot_, val_) do { } while (0)
#define PROF_INC(slot_, val_) do { } while (0)
#endif

enum { ST_BOX_I = 0, ST_BOX_Q, ST_BOX_N, ST_PRE_I, ST_PRE_Q, ST_AVG, ST_LPR_ACC, ST_LPR_PHASE,
       ST_SQ_HITS, ST_ADC, ST_RDC_I, ST_RDC_Q, ST_HDR = 16 };

static inline int fm_packed_levels(int P, int wide) { return wide ? 0 : (P < FM_MAX_PACKED ? P : FM_MAX_PACKED); }
static inline int fm_state_words(int P, int wide) { int pl = fm_packed_levels(P, wide); return ST_HDR + 6 * pl + 7 * (P - pl) + 9; }

constexpr unsigned FIR_B = 16384u;
// raw int16 lanes <-> lanes biased by FIR_B (no carry between lanes while |v| <= 16383)
__device__ __forceinline__ uint32_t fir_bias_lanes(uint32_t w) { return (w ^ 0x80008000u) - 0x40004000u; }
__device__ __forceinline__ uint32_t fir_unbias_lanes(uint32_t w) { return (w + 0x40004000u) ^ 0x80008000u; }
__device__ __forceinline__ uint32_t pack2(int i, int q) { return ((uint32_t)i & 0xffffu) | ((uint32_t)q << 16); }
__device__ __forceinline__ int lo16(uint32_t w) { return (int)(int16_t)(w & 0xffffu); }
__device__ __forceinline__ int hi16(uint32_t w) { return (int)(int16_t)(w >> 16); }

// ------------------------------------------------------------------------------ front-end state
template <int P, int SPEC>
struct FrontState {
	// SPEC 2: the per-chunk reduction stages are on; values may exceed the packed head-room (raw DC
	// block) -> every pass is scalar
	static constexpr int PL = (SPEC == 2) ? 0 : (P < FM_MAX_PACKED ? P : FM_MAX_PACKED);
	static constexpr int PS = P - PL;
	// droop FIR history kept biased (lane = v + FIR_B) when |v| <= 128 << P leaves head-room for the
	// sum of two lanes: P <= 6 and no raw DC block
	static constexpr bool FIRB = (SPEC != 2) && (P >= 1) && (P <= 6);
	int box_i, box_q, box_n;
	// packed passes: the last six samples the pass has seen (oldest first), I in the low and Q in
	// the high half-word, each biased by 128<<level so both lanes stay unsigned
	uint32_t h[PL > 0 ? PL : 1][6];
	// scalar passes (level >= 3): the reference's window a..f plus the odd sample waiting for its pair
	int wi[PS > 0 ? PS : 1][6], wq[PS > 0 ? PS : 1][6], pi[PS > 0 ? PS : 1], pq[PS > 0 ? PS : 1];
	uint32_t fh[9];            // generic_fir history, I low / Q high half-word (raw int16)
	int pre_i, pre_q;
};

template <int P, int SPEC>
__device__ __forceinline__ void front_zero(FrontState<P, SPEC> &s)
{
	s.box_i = s.box_q = s.box_n = 0;
#pragma unroll
	for (int l = 0; l < FrontState<P, SPEC>::PL; l++) {
#pragma unroll
		for (int j = 0; j < 6; j++) { s.h[l][j] = 0x00010001u * (128u << l); }
	}
#pragma unroll
	for (int l = 0; l < FrontState<P, SPEC>::PS; l++) {
#pragma unroll
		for (int j = 0; j < 6; j++) { s.wi[l][j] = 0; s.wq[l][j] = 0; }
		s.pi[l] = 0; s.pq[l] = 0;
	}
#pragma unroll
	for (int j = 0; j < 9; j++) { s.fh[j] = FrontState<P, SPEC>::FIRB ? fir_bias_lanes(0u) : 0u; }
	s.pre_i = s.pre_q = 0;
}

template <int P, int SPEC>
__device__ __forceinline__ void front_load(FrontState<P, SPEC> &s, const uint32_t *g)
{
	constexpr int PL = FrontState<P, SPEC>::PL, PS = FrontState<P, SPEC>::PS;
	s.box_i = (int)g[ST_BOX_I]; s.box_q = (int)g[ST_BOX_Q]; s.box_n = (int)g[ST_BOX_N];
	s.pre_i = (int)g[ST_PRE_I]; s.pre_q = (int)g[ST_PRE_Q];
#pragma unroll
	for (int l = 0; l < PL; l++) {
#pragma unroll
		for (int j = 0; j < 6; j++) { s.h[l][j] = g[ST_HDR + 6 * l + j]; }
	}
#pragma unroll
	for (int l = 0; l < PS; l++) {
#pragma unroll
		for (int j = 0; j < 6; j++) { uint32_t w = g[ST_HDR + 6 * PL + 7 * l + j]; s.wi[l][j] = lo16(w); s.wq[l][j] = hi16(w); }
		uint32_t w = g[ST_HDR + 6 * PL + 7 * l + 6]; s.pi[l] = lo16(w); s.pq[l] = hi16(w);
	}
#pragma unroll
	for (int j = 0; j < 9; j++) { uint32_t w = g[ST_HDR + 6 * PL + 7 * PS + j]; s.fh[j] = FrontState<P, SPEC>::FIRB ? fir_bias_lanes(w) : w; }
}

template <int P, int SPEC>
__device__ __forceinline__ void front_store(const FrontState<P, SPEC> &s, uint32_t *g)
{
	constexpr int PL = FrontState<P, SPEC>::PL, PS = FrontState<P, SPEC>::PS;
	g[ST_BOX_I] = (uint32_t)s.box_i; g[ST_BOX_Q] = (uint32_t)s.box_q; g[ST_BOX_N] = (uint32_t)s.box_n;
	g[ST_PRE_I] = (uint32_t)s.pre_i; g[ST_PRE_Q] = (uint32_t)s.pre_q;
#pragma unroll
	for (int l = 0; l < PL; l++) {
#pragma unroll
		for (int j = 0; j < 6; j++) { g[ST_HDR + 6 * l + j] = s.h[l][j]; }
	}
#pragma unroll
	for (int l = 0; l < PS; l++) {
#pragma unroll
		for (int j = 0; j < 6; j++) { g[ST_HDR + 6 * PL + 7 * l + j] = pack2(s.wi[l][j], s.wq[l][j]); }
		g[ST_HDR + 6 * PL + 7 * l + 6] = pack2(s.pi[l], s.pq[l]);
	}
#pragma unroll
	for (int j = 0; j < 9; j++) { g[ST_HDR + 6 * PL + 7 * PS + j] = FrontState<P, SPEC>::FIRB ? fir_unbias_lanes(s.fh[j]) : s.fh[j]; }
}

// ------------------------------------------------------------------------------ stages
// fifth_order tap set [1 5 10 10 5 1] >> 4 on two biased 16-bit lanes at once.  With inputs biased by
// B (lane = v + B, |v| <= B) the lane sum is < 64 B <= 32768, so no carry crosses lanes, and
// (sum + 32 B) >> 4 == (sum >> 4) + 2 B exactly: the output lanes are biased by 2 B.  The int16
// store of the reference never wraps here because |v| <= 128 << level after the 8-bit-range scale.
// (Moving these adds onto the multiplier pipe did not pay: DESIGN.md §4.1, "Instruction rates".)
__device__ __forceinline__ uint32_t hb_tap(uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t e, uint32_t f)
{
	uint32_t s = a + f + (b + e) * 5u + (c + d) * 10u;
	return (s >> 4) & 0x0FFF0FFFu;
}

// Scalar fifth_order pass for levels >= 3 (values may exceed the packed head-room; int16 wrap kept).
// One input sample at in-chunk index idx of pass L (src/rtl_fm.c:411-440, :765-768): a pass emits at
// even input indices; index 0 of a chunk slides the window by one (a..e = hist[1..5], f = data[0]),
// every later even index by two; an odd-indexed sample waits and is lost if the chunk ends on it (F7).
template <int L, int P, int SPEC>
__device__ __forceinline__ bool scalar_push(FrontState<P, SPEC> &s, int xi, int xq, unsigned idx, int &oi, int &oq)
{
	constexpr int PS = FrontState<P, SPEC>::PS;
	if constexpr (L >= PS) {
		oi = xi; oq = xq;
		return true;
	} else {
		if (idx & 1u) { s.pi[L] = xi; s.pq[L] = xq; return false; }
		if (idx == 0u) {
#pragma unroll
			for (int j = 0; j < 5; j++) { s.wi[L][j] = s.wi[L][j + 1]; s.wq[L][j] = s.wq[L][j + 1]; }
		} else {
#pragma unroll
			for (int j = 0; j < 4; j++) { s.wi[L][j] = s.wi[L][j + 2]; s.wq[L][j] = s.wq[L][j + 2]; }
			s.wi[L][4] = s.pi[L]; s.wq[L][4] = s.pq[L];
		}
		s.wi[L][5] = xi; s.wq[L][5] = xq;
		int yi = wrap16((s.wi[L][0] + (s.wi[L][1] + s.wi[L][4]) * 5 + (s.wi[L][2] + s.wi[L][3]) * 10 + s.wi[L][5]) >> 4);
		int yq = wrap16((s.wq[L][0] + (s.wq[L][1] + s.wq[L][4]) * 5 + (s.wq[L][2] + s.wq[L][3]) * 10 + s.wq[L][5]) >> 4);
		return scalar_push<L + 1, P, SPEC>(s, yi, yq, idx >> 1, oi, oq);
	}
}

// generic_fir (src/rtl_fm.c:442-465) on both components: output from the PREVIOUS nine samples, then
// the current sample is shifted into the history.  int32 wrap-around preserved.
__device__ __forceinline__ void droop9(uint32_t (&h)[9], const int (&c)[6], int &di, int &dq)
{
	int ai = mul_w(lo16(h[0]) + lo16(h[8]), c[1]);
	int aq = mul_w(hi16(h[0]) + hi16(h[8]), c[1]);
	ai = add_w(ai, mul_w(lo16(h[1]) + lo16(h[7]), c[2]));
	aq = add_w(aq, mul_w(hi16(h[1]) + hi16(h[7]), c[2]));
	ai = add_w(ai, mul_w(lo16(h[2]) + lo16(h[6]), c[3]));
	aq = add_w(aq, mul_w(hi16(h[2]) + hi16(h[6]), c[3]));
	ai = add_w(ai, mul_w(lo16(h[3]) + lo16(h[5]), c[4]));
	aq = add_w(aq, mul_w(hi16(h[3]) + hi16(h[5]), c[4]));
	ai = add_w(ai, mul_w(lo16(h[4]), c[5]));
	aq = add_w(aq, mul_w(hi16(h[4]), c[5]));
#pragma unroll
	for (int j = 0; j < 8; j++) { h[j] = h[j + 1]; }
	h[8] = pack2(di, dq);
	di = wrap16(ai >> 15);
	dq = wrap16(aq >> 15);
}

// Same filter on the biased history (lanes = v + FIR_B): the symmetric taps are added two lanes at a
// time (lane sums <= 2 (FIR_B + 8192) < 65536, no carry), the bias leaves through one constant,
//   sum c_k (v_k + v_k' + 2 FIR_B) = sum c_k (v_k + v_k') + fir_bias   (all in wrapping int32).
__device__ __forceinline__ void droop9_packed(uint32_t (&h)[9], const int (&c)[6], int fir_bias, int &di, int &dq)
{
	const uint32_t s0 = h[0] + h[8], s1 = h[1] + h[7], s2 = h[2] + h[6], s3 = h[3] + h[5], s4 = h[4];
	int ai = sub_w(mul_w((int)(s0 & 0xffffu), c[1]), fir_bias);
	int aq = sub_w(mul_w((int)(s0 >> 16), c[1]), fir_bias);
	ai = add_w(ai, mul_w((int)(s1 & 0xffffu), c[2])); aq = add_w(aq, mul_w((int)(s1 >> 16), c[2]));
	ai = add_w(ai, mul_w((int)(s2 & 0xffffu), c[3])); aq = add_w(aq, mul_w((int)(s2 >> 16), c[3]));
	ai = add_w(ai, mul_w((int)(s3 & 0xffffu), c[4])); aq = add_w(aq, mul_w((int)(s3 >> 16), c[4]));
	ai = add_w(ai, mul_w((int)(s4 & 0xffffu), c[5])); aq = add_w(aq, mul_w((int)(s4 >> 16), c[5]));
#pragma unroll
	for (int j = 0; j < 8; j++) { h[j] = h[j + 1]; }
	h[8] = ((uint32_t)dq << 16) + (uint32_t)di + (FIR_B * 0x10001u);
	di = wrap16(ai >> 15);
	dq = wrap16(aq >> 15);
}

// polar_discriminant (src/rtl_fm.c:476-483); note 3.14159.
__device__ __noinline__ int disc_std(int cr, int cj)
{
	double angle = atan2((double)cj, (double)cr);
	return (int)(angle / 3.14159 * (double)(1 << 14));
}

// polar_discriminant without libm's general-purpose atan2: the result is only needed to the integer
// below it, so a 14-term odd polynomial on [0, 1] (|error| < 7e-13 rad, i.e. < 4e-9 output units) plus a
// division by fp32 reciprocal + one Newton step decides almost every sample; values within 1e-5 of an
// integer (where the truncation could flip) go through disc_std.  Same result as disc_std otherwise.
__device__ __forceinline__ int disc_std_lean(int cr, int cj)
{
	if (cj == 0 && cr >= 0) { return 0; }                    // atan2(0, x >= 0) == 0 exactly (also x == y == 0)
	const double y = (double)cj, x = (double)cr;
	const double ay = fabs(y), ax = fabs(x);
	const double a = fmin(ax, ay), b = fmax(ax, ay);         // b >= 1 here
	float rf;
	asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rf) : "f"(__double2float_rn(b)));
	double r = (double)rf;
	r = fma(r, fma(-b, r, 1.0), r);                          // relative error ~2^-46
	const double t = a * r, u = t * t;
	double p = -0.00023006126561948349;
	p = fma(p, u, 0.001914706015773981);
	p = fma(p, u, -0.0074929064903861186);
	p = fma(p, u, 0.018612363543602756);
	p = fma(p, u, -0.03374387219298904);
	p = fma(p, u, 0.04926117444681421);
	p = fma(p, u, -0.06301031978620865);
	p = fma(p, u, 0.07589599479154154);
	p = fma(p, u, -0.09070400517070532);
	p = fma(p, u, 0.11108328001324017);
	p = fma(p, u, -0.1428547415701187);
	p = fma(p, u, 0.1999998816752856);
	p = fma(p, u, -0.33333333059437525);
	p = fma(p, u, 0.9999999999811207);
	double ang = t * p;
	if (ay > ax) { ang = 1.5707963267948966 - ang; }
	if (cr < 0) { ang = 3.141592653589793 - ang; }
	if (cj < 0) { ang = -ang; }
	const double v = ang * (16384.0 / 3.14159);
	if (fabs(v - rint(v)) < 1e-5) { return disc_std(cr, cj); }
	return (int)v;
}

// fast_atan2 (src/rtl_fm.c:485-506), int32 wrap-around preserved.  The two branches of the reference
//   x >= 0: pi/4  - pi/4 * (x - |y|) / (x + |y|)        x < 0: 3pi/4 - pi/4 * (x + |y|) / (|y| - x)
// share the divisor |x| + |y|; the quotient is bounded by 4096 whenever that divisor is positive (also
// after wrap-around of the numerator), so one fp32 reciprocal estimate plus an exact integer remainder
// correction reproduces C's truncating '/'.  A non-positive divisor (only reachable through int32
// overflow, or x == y == 0) takes the generic path.
__device__ __forceinline__ float rcp_est(float x)
{
	float r;
	asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));   // bare MUFU.RCP, <= 1 ulp; the quotient estimate stays within +-1
	return r;
}
__device__ __forceinline__ int fast_atan2_i(int y, int x)
{
	const int q1 = 1 << 12, q3 = 3 * (1 << 12);
	const int ya = y < 0 ? neg_w(y) : y;
	const bool xneg = x < 0;
	const int num = mul_w(q1, xneg ? add_w(x, ya) : sub_w(x, ya));
	const int den = xneg ? sub_w(ya, x) : add_w(x, ya);
	int q;
	if (den > 0) {
		q = __float2int_rz(__int2float_rn(num) * rcp_est(__int2float_rn(den)));
		const int r = sub_w(num, mul_w(q, den));
		const int up = num >= 0 ? (r >= den ? 1 : 0) : (r > 0 ? 1 : 0);
		const int dn = num >= 0 ? (r < 0 ? 1 : 0) : (r <= -den ? 1 : 0);
		q += up - dn;
	} else {
		if (x == 0 && y == 0) { return 0; }
		q = div_c(num, den);
	}
	const int ang = sub_w(xneg ? q3 : q1, q);
	return y < 0 ? neg_w(ang) : ang;
}

// fast_atan2 on operands that are exact in FP32 (|x|, |y| <= 2^16: the undecimated shape, where a sample is an 8-bit-range
// value and the conjugate product at most 2 * 128^2).  FP32 adds and multiply-adds issue every cycle, the integer
// adder / shifter pipe every other one (tools/experiments/op_microbench.cu), and the integer form above is mostly
// adder-pipe work.  Every quantity below is an integer held exactly in a float:
//   den = |x| + |y|,  n = |x| - |y|,  T = floor(4096 |n| / den)  (estimate from a reciprocal biased low by 2^-20 --
//   never above the true quotient, at most one below -- then one exact remainder check: fma(-T, den, 4096 |n|)),
//   x >= 0: 4096 - sgn(n) T        x < 0: 12288 + sgn(n) T        negated for y < 0        0 for x == y == 0
// which is the reference's truncating integer division on both branches (src/rtl_fm.c:485-506).  Returns the angle as
// an integer-valued float.
__device__ __forceinline__ float fast_atan2_f32(float y, float x)
{
	const float ax = fabsf(x), ay = fabsf(y);
	const float den = __fadd_rn(ax, ay);
	const float n = __fsub_rn(ax, ay);
	const float an = __fmul_rn(fabsf(n), 4096.0f);
	float te = __fmul_rn(an, rcp_est(den));
	te = __fmaf_rn(te, -9.5367431640625e-07f, te);                       // * (1 - 2^-20)
	float T = __fsub_rn(__fadd_rd(te, 12582912.0f), 12582912.0f);        // floor(te): round-down add of 1.5 * 2^23
	const float rem = __fmaf_rn(-T, den, an);                            // exact
	if (rem >= den) { T = __fadd_rn(T, 1.0f); }
	const float Ts = __int_as_float(__float_as_int(T) ^ (__float_as_int(n) & (int)0x80000000));      // sgn(n) T  (n is never -0)
	const float ang = (x >= 0.0f) ? __fsub_rn(4096.0f, Ts) : __fadd_rn(12288.0f, Ts);
	const float r = (y < 0.0f) ? -ang : ang;
	return (den == 0.0f) ? 0.0f : r;
}

// polar_discriminant in FP32 with a guard band (operands below 2^24, i.e. exact in a float: always so without decimation).
// The fp64 form above costs ~100 instructions, most of them at the fp64 pipe's rate; here the angle is estimated in
// FP32 -- t = min/max by reciprocal + one exact-remainder step, atan(t) = t + t^3 q(t^2) with a degree-8 q (6.7e-8 rad on
// [0, 1]), times 16384/3.14159 as a two-float constant -- and assembled as an INTEGER part plus a small FRACTION per octant
// (8192.0069 - v, 16384.0138 - v: the constants' integer parts in integer arithmetic), so the only error is the
// estimate's own: 4.1e-4 output units at most over 6 M operand pairs.  Whenever the fraction is within 1.5e-3 of an
// integer (0.3 % of the samples) the truncation could go either way and the fp64 form decides.  Same results as
// disc_std_lean; the algorithm restated in numpy and checked against fp64 atan2 (tests/test_host_logic.py::test_polar_disc_fp32_form).
__device__ __forceinline__ int disc_std_f32(int cr, int cj)
{
	if (cj == 0 && cr >= 0) { return 0; }
	if ((unsigned)cr + (1u << 24) >= (1u << 25) || (unsigned)cj + (1u << 24) >= (1u << 25)) { return disc_std_lean(cr, cj); }
	const float ax = fabsf(__int2float_rn(cr)), ay = fabsf(__int2float_rn(cj));
	const float a = fminf(ax, ay), b = fmaxf(ax, ay);                  // b >= 1
	const float r = rcp_est(b);
	const float t0 = __fmul_rn(a, r);
	const float t = __fmaf_rn(__fmaf_rn(-t0, b, a), r, t0);            // a / b to half an ulp
	const float u = __fmul_rn(t, t);
	float q = -0.002447017002850771f;
	q = __fmaf_rn(q, u, 0.013750223442912102f);
	q = __fmaf_rn(q, u, -0.03627006709575653f);
	q = __fmaf_rn(q, u, 0.06284350901842117f);
	q = __fmaf_rn(q, u, -0.08673165738582611f);
	q = __fmaf_rn(q, u, 0.11037992686033249f);
	q = __fmaf_rn(q, u, -0.14279110729694366f);
	q = __fmaf_rn(q, u, 0.1999976634979248f);
	q = __fmaf_rn(q, u, -0.3333333134651184f);
	const float p = __fmaf_rn(__fmul_rn(t, u), q, t);                  // atan(t), 0 <= t <= 1
	const float KHI = 5215.193359375f, KLO = 0.00022094578889664263f;  // 16384 / 3.14159 in two floats
	const float nm = __fadd_rd(__fmul_rn(p, KHI), 12582912.0f);        // 1.5 * 2^23 + floor(p * KHI)
	const float n1 = __fsub_rn(nm, 12582912.0f);
	float F = __fmaf_rn(p, KLO, __fmaf_rn(p, KHI, -n1));               // the fraction, in [-eps, 1 + eps)
	int N = __float_as_int(nm) - 0x4B400000;                           // the integer part
	if (ay > ax) { N = 8191 - N; F = __fsub_rn(1.0069195032119751f, F); }       // pi/2 - angle: 8192.00692 - v
	if (cr < 0) { N = 16383 - N; F = __fsub_rn(1.0138390064239502f, F); }       // pi - angle: 16384.01384 - v
	const float Fm = __fadd_rn(F, 12582912.0f);                        // 1.5 * 2^23 + rint(F)
	const float Fr = __fsub_rn(Fm, 12582912.0f);
	if (fabsf(__fsub_rn(F, Fr)) < 1.5e-3f) { return disc_std_lean(cr, cj); }
	const int k = N + (__float_as_int(Fm) - 0x4B400000) - (F < Fr ? 1 : 0);    // N + floor(F)
	return cj < 0 ? -k : k;
}

// polar_disc_lut (src/rtl_fm.c:528-564)
__device__ __forceinline__ int disc_lut(const int *__restrict__ lut, int cr, int cj)
{
	if (cr == 0 || cj == 0) {
		if (cr == 0 && cj == 0) { return 0; }
		if (cr == 0) { return cj > 0 ? (1 << 13) : -(1 << 13); }
		return cr > 0 ? 0 : (1 << 14);
	}
	int x = div_c((int)((unsigned)cj << 8), cr);
	int xa = x < 0 ? neg_w(x) : x;
	// |x| >= 131072, and x = INT_MIN, whose xa wraps negative (cj = 2^23 mod 2^24 over |cr| = 1: the reference reads
	// atan_lut[INT_MIN] or divides INT_MIN by -1 there; see RXB200_ATAN_LUT).  One unsigned compare: nvcc treats
	// x < 0 ? -x : x as never negative and drops a separate signed xa < 0 test, and the table would be read at INT_MIN.
	if ((unsigned)xa >= 131072u) { return cj > 0 ? (1 << 13) : -(1 << 13); }
	if (x > 0) { return cj > 0 ? __ldg(lut + x) : __ldg(lut + x) - (1 << 14); }
	return cj > 0 ? (1 << 14) - __ldg(lut + xa) : -__ldg(lut + xa);
}

// esbensen (src/rtl_fm.c:566-582)
__device__ __forceinline__ int disc_ale(int ar, int aj, int br, int bj)
{
	int dr = mul_w(sub_w(br, ar), 2), dj = mul_w(sub_w(bj, aj), 2);
	int cj = sub_w(mul_w(bj, dr), mul_w(br, dj));
	return div_c(mul_w(2608, cj), add_w(add_w(mul_w(ar, ar), mul_w(aj, aj)), 1));
}

// One deemph_filter step (src/rtl_fm.c:673-680): avg += trunc((d +- a/2)/a).
//   d > 0 : trunc((d + h)/a) = floor((d + h)/a);   d <= 0: trunc((d - h)/a) = floor((d - h + a - 1)/a)
// i.e. floor((d + c)/a) with c = h for odd a and c = h - (d <= 0) for even a (h = a/2).  With a bias of
// K*a the numerator is non-negative and the floor is one umulhi by a host-verified reciprocal.
__device__ __forceinline__ int deemph_step(const FmDev &c, int avg, int x)
{
	int d = x - avg;
	if (c.a_use_magic) {
		int n = d + c.a_half + c.a_K * c.a;
		if (c.a_even) { n -= (d <= 0) ? 1 : 0; }
		return avg + (int)__umulhi((unsigned)n, c.a_magic) - c.a_K;
	}
	return avg + ((d > 0) ? (d + c.a_half) / c.a : (d - c.a_half) / c.a);
}

// ------------------------------------------------------------------------------ bookkeeping
// Decimated samples the reference has produced after t input samples of this call.
__device__ __forceinline__ long long dec_raw(const FmDev &c, long long t, int box_n0)
{
	if (c.P > 0) { return t >> c.P; }
	return (t + box_n0) / c.D;
}
// ... and after low_pass_simple's per-chunk grouping (-o, src/rtl_fm.c:373-387): a group counts where
// its last member is produced (supported shapes make every chunk a whole number of groups).
__device__ __forceinline__ long long dec_before(const FmDev &c, long long t, int box_n0)
{
	long long m = dec_raw(c, t, box_n0);
	return c.post_ds > 1 ? m / c.post_ds : m;
}
// chunk that produced PCM sample m (index after -o grouping, counted from the start of the call)
__device__ __forceinline__ int pcm_chunk(const FmDev &c, int chunk, long long m, int box_n0)
{
	long long md = c.post_ds > 1 ? m * c.post_ds + (c.post_ds - 1) : m;
	long long pos = c.P > 0 ? (md << c.P) : ((md + 1) * (long long)c.D - box_n0 - 1);
	return (int)(pos / chunk);
}
// Output slot of the first value produced at/after decimated index m.
__device__ __forceinline__ long long out_before(const FmDev &c, long long m, int phase0)
{
	if (c.mode == RXB200_MODE_RAW) { return 2 * m; }
	if (!c.resample) { return m; }
	return ((long long)phase0 + m * (long long)c.slow) / (long long)c.fast;
}
// shared PCM buffer: PAD entries of padding per 128 so that neither the front-end stores (thread stride ~ Sf/D
// entries) nor the back-end loads (lane stride = piece) pile on one bank.  The segment front end uses 2 (4 bytes);
// the row front end 8, which keeps its 8/16-byte vector stores aligned (fm_rows.cuh)
#define PCM_PAD_SEG 2
#define PCM_PAD_ROWS 0
template <int PAD>
__device__ __forceinline__ int pcm_phys(int rel) { return rel + PAD * (rel >> 7); }

// Compile-time specialisation of the flags that sit in the per-sample path.  SPEC 0: everything is a
// (warp-uniform) run-time branch.  SPEC 1: the wbfm shape — FM discriminator with fast_atan2, fs/4
// rotation on, serial stages present — resolved at compile time.
template <int SPEC>
struct Spec {
	// SPEC 3: the multi-channel NBFM shape (BASELINE configs[4]) -- FM discriminator through the LUT, rotation on, NO serial
	// stage (the front end stores the output itself): the back end and every other mode drop out of the kernel at compile time
	// SPEC 4: the wbfm shape's front end alone -- SPEC 1's discriminator, the PCM stored to global memory through the
	// direct-output path (fm_back_kernel runs the serial stages afterwards, fm_launch's stream path)
	static __device__ __forceinline__ int mode(const FmDev &c) { return (SPEC == 1 || SPEC == 3 || SPEC == 4) ? RXB200_MODE_FM : c.mode; }
	static __device__ __forceinline__ int atan_mode(const FmDev &c) { return (SPEC == 1 || SPEC == 4) ? RXB200_ATAN_FAST : (SPEC == 3 ? RXB200_ATAN_LUT : c.atan_mode); }
	static __device__ __forceinline__ bool rotate(const FmDev &c) { return (SPEC == 1 || SPEC == 3 || SPEC == 4) ? true : !c.offset_tuning; }
	static __device__ __forceinline__ bool direct(const FmCall &k) { return SPEC == 1 ? false : ((SPEC == 3 || SPEC == 4) ? true : (k.direct_out != 0)); }
};

struct EmitCtx {
	int16_t *pcm;            // shared PCM buffer
	int16_t *out;            // channel output (direct_out only)
	long long m_lo;          // decimated index of pcm[0]
	int rel;                 // decimated index of the next sample, relative to m_lo
	int first_in_chunk;
	int chunk_idx;           // chunk the current block belongs to
	int rdc_i, rdc_q;        // raw DC block offsets of this chunk
	int sq_zero;             // squelch closed on this chunk
	int pds_acc, pds_cnt;    // -o group in progress
	long long red_t, red_p;  // squelch pre-pass accumulators of this chunk
};

// Everything between the decimator and the serial stages, for one decimated sample.  STORE: the
// sample belongs to this thread's own segment (otherwise it only advances the filter state).
template <int P, int SPEC, bool STORE>
__device__ __forceinline__ void post_decim(const FmDev &c, const FmCall &k, FrontState<P, SPEC> &s, EmitCtx &e, int di, int dq)
{
	if (c.fir_on) {
		if constexpr (FrontState<P, SPEC>::FIRB) { droop9_packed(s.fh, c.fir, c.fir_bias, di, dq); } else { droop9(s.fh, c.fir, di, dq); }
	}
	if (SPEC == 2) {
		if (k.reduce_mode == 1) {       // rms() inputs of this chunk (src/rtl_fm.c:746-751)
			if (STORE) { e.red_t += di + dq; e.red_p += (long long)di * di + (long long)dq * dq; }
			e.rel++;
			return;
		}
		if (e.sq_zero) { di = 0; dq = 0; }   // squelch zeroes lowpassed AFTER the droop FIR saw the samples (:785-787)
	}
	const int mode = Spec<SPEC>::mode(c);
	int pcm;
	if (mode == RXB200_MODE_FM) {
		const int am = Spec<SPEC>::atan_mode(c);
		int br = s.pre_i, bj = s.pre_q;
		int cr = add_w(mul_w(di, br), mul_w(dq, bj));       // x[n] * conj(x[n-1]) (src/rtl_fm.c:470-474)
		int cj = sub_w(mul_w(dq, br), mul_w(di, bj));
		if (am == RXB200_ATAN_STD) { pcm = disc_std_f32(cr, cj); }
		else if (e.first_in_chunk) { pcm = disc_std(cr, cj); }                     // F8: one sample per chunk, out of line
		else if (am == RXB200_ATAN_FAST) { pcm = fast_atan2_i(cj, cr); }
		else if (am == RXB200_ATAN_LUT) { pcm = disc_lut(c.atan_lut, cr, cj); }
		else { pcm = disc_ale(di, dq, br, bj); }
		s.pre_i = di; s.pre_q = dq;
	} else if (mode == RXB200_MODE_AM) {
		int en = add_w(mul_w(di, di), mul_w(dq, dq));
		pcm = mul_w(wrap16((int)sqrt((double)en)), c.out_scale);
	} else if (mode == RXB200_MODE_USB) {
		pcm = mul_w(wrap16(di + dq), c.out_scale);
	} else if (mode == RXB200_MODE_LSB) {
		pcm = mul_w(wrap16(di - dq), c.out_scale);
	} else {   // raw: lowpassed copied out, nothing after (src/rtl_fm.c:658-665, :809-811)
		if (STORE && (SPEC != 2 || k.reduce_mode == 0)) { long long m = e.m_lo + e.rel; e.out[2 * m] = (int16_t)di; e.out[2 * m + 1] = (int16_t)dq; }
		e.rel++;
		e.first_in_chunk = 0;
		return;
	}
	e.first_in_chunk = 0;
	if (SPEC == 2 && c.post_ds > 1) {   // low_pass_simple: sum of post_ds int16 results, stored as int16 (:373-387)
		e.pds_acc += wrap16(pcm);
		if (++e.pds_cnt < c.post_ds) { return; }
		pcm = e.pds_acc; e.pds_acc = 0; e.pds_cnt = 0;
	}
	if (STORE) {      // the int16 store is the reference's (int16_t) cast
		if (Spec<SPEC>::direct(k)) { if (SPEC != 2 || k.reduce_mode == 0) { e.out[e.m_lo + e.rel] = (int16_t)pcm; } }
		else { e.pcm[pcm_phys<PCM_PAD_SEG>(e.rel)] = (int16_t)pcm; }
	}
	e.rel++;
}

// scale + fs/4 rotation of one CS16 word (I low, Q high): rotate16_90 multiplies sample n of the chunk by
// j^n (src/rtl_fm.c:309-327); pos = n & 3 is a compile-time constant in the unrolled block.
__device__ __forceinline__ void scale_rot(uint32_t w, int pos, bool rotate, int &ri, int &rq, int dci = 0, int dcq = 0)
{
	// dc_block_raw_filter subtracts the chunk's running mean between the scale and the rotation (:850-857)
	const int wi16 = lo16(w), wq16 = hi16(w);
	int xi = wrap16(scale_cs16(wi16) - dci), xq = wrap16(scale_cs16(wq16) - dcq);
	if (!rotate) { pos = 0; }
	switch (pos & 3) {
	case 1: ri = -xq; rq = xi; break;
	case 2: ri = -xi; rq = -xq; break;
	case 3: ri = xq; rq = -xi; break;
	default: ri = xi; rq = xq; break;
	}
}
__device__ __forceinline__ uint32_t scale_rot_pack(uint32_t w, int pos, bool rotate)
{
	int ri, rq;
	scale_rot(w, pos, rotate, ri, rq);
	return (uint32_t)(ri + 128) + ((uint32_t)(rq + 128) << 16);
}

// 32 bytes per lane as two 128-bit loads (sm_90 has no 256-bit load); the L2 fetches the whole 256-byte sector group
__device__ __forceinline__ void ldg256(const int16_t *p, uint32_t (&v)[8])
{
	asm volatile("ld.global.nc.L2::256B.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
	             "ld.global.nc.L2::256B.v4.u32 {%4,%5,%6,%7}, [%8+16];"
	             : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]), "=r"(v[4]), "=r"(v[5]), "=r"(v[6]), "=r"(v[7])
	             : "l"(p));
}

// The packed passes (levels < PL) of one block whose samples are already scaled, rotated and packed.
template <int P, int SPEC, bool STORE>
__device__ __forceinline__ void front_block_packed(const FmDev &c, const FmCall &k, FrontState<P, SPEC> &s, EmitCtx &e,
                                                   const uint32_t (&x)[8], unsigned u)
{
	constexpr int PL = FrontState<P, SPEC>::PL;
		// pass 0: window for the sample at block offset 2j is s[2j-5 .. 2j] of (h[0] .. , x[0..7])
		uint32_t (&h0)[6] = s.h[0];
		uint32_t y[4];
		y[0] = hb_tap(h0[1], h0[2], h0[3], h0[4], h0[5], x[0]);
		y[1] = hb_tap(h0[3], h0[4], h0[5], x[0], x[1], x[2]);
		y[2] = hb_tap(h0[5], x[0], x[1], x[2], x[3], x[4]);
		y[3] = hb_tap(x[1], x[2], x[3], x[4], x[5], x[6]);
#pragma unroll
		for (int j = 0; j < 6; j++) { h0[j] = x[j + 2]; }
		uint32_t outw[4];
		int nout;
		if constexpr (PL == 1) {
			outw[0] = y[0]; outw[1] = y[1]; outw[2] = y[2]; outw[3] = y[3];
			nout = 4;
		} else {
			uint32_t (&h1)[6] = s.h[1];
			uint32_t z0 = hb_tap(h1[1], h1[2], h1[3], h1[4], h1[5], y[0]);
			uint32_t z1 = hb_tap(h1[3], h1[4], h1[5], y[0], y[1], y[2]);
			h1[0] = h1[4]; h1[1] = h1[5]; h1[2] = y[0]; h1[3] = y[1]; h1[4] = y[2]; h1[5] = y[3];
			if constexpr (PL == 2) {
				outw[0] = z0; outw[1] = z1;
				nout = 2;
			} else {
				uint32_t (&h2)[6] = s.h[2];
				outw[0] = hb_tap(h2[1], h2[2], h2[3], h2[4], h2[5], z0);
				h2[0] = h2[2]; h2[1] = h2[3]; h2[2] = h2[4]; h2[3] = h2[5]; h2[4] = z0; h2[5] = z1;
				nout = 1;
			}
		}
		const int bias = 128 << PL;
#pragma unroll
		for (int j = 0; j < 4; j++) {
			if (j < nout) {
				int di = (int)(outw[j] & 0xffffu) - bias, dq = (int)(outw[j] >> 16) - bias;
				if constexpr (P > PL) {
					// in-chunk index of this sample at pass PL: (u >> PL) + j
					int oi, oq;
					if (scalar_push<0, P, SPEC>(s, di, dq, (u >> PL) + (unsigned)j, oi, oq)) { post_decim<P, SPEC, STORE>(c, k, s, e, oi, oq); }
				} else {
					post_decim<P, SPEC, STORE>(c, k, s, e, di, dq);
				}
			}
		}
	}

// One block of 8 input samples at in-chunk offset u (multiple of 8).
template <int P, int SPEC, bool STORE>
__device__ __forceinline__ void front_block(const FmDev &c, const FmCall &k, FrontState<P, SPEC> &s, EmitCtx &e,
                                            const uint32_t (&v)[8], unsigned u)
{
	constexpr int PL = FrontState<P, SPEC>::PL;
	const bool rot = Spec<SPEC>::rotate(c);
	if constexpr (P == 0 && SPEC == 4) {
		if (c.D == 1) {
			// no decimation (-s at or above 1 Msps): every input sample is a PCM sample and a block is 8 consecutive entries of
			// the global PCM array, 16-byte aligned (segments and halos are multiples of 8) -- one vector store per block
			// instead of eight 2-byte stores to 32 different lines per warp.  Same results as post_decim's FM branch:
			// the discriminator in FP32 (exact: see fast_atan2_f32); the angle leaves through the low 16 bits of
			// angle + 1.5 * 2^23, two samples per byte permute
			uint32_t ab[8];
			float br = __int2float_rn(s.pre_i), bj = __int2float_rn(s.pre_q);
			int di = s.pre_i, dq = s.pre_q;
#pragma unroll
			for (int j = 0; j < 8; j++) {
				scale_rot(v[j], j, rot, di, dq);
				const float fi = __int2float_rn(di), fq = __int2float_rn(dq);
				const float cr = __fmaf_rn(fi, br, __fmul_rn(fq, bj));
				const float cj = __fmaf_rn(fq, br, -__fmul_rn(fi, bj));
				float ang = fast_atan2_f32(cj, cr);
				// F8: the chunk's first sample (chunks start on block boundaries) goes through the libm discriminator
				if (j == 0 && e.first_in_chunk) { ang = __int2float_rn(disc_std(__float2int_rn(cr), __float2int_rn(cj))); }
				ab[j] = (uint32_t)__float_as_int(__fadd_rn(ang, 12582912.0f));
				br = fi; bj = fq;
			}
			s.pre_i = di; s.pre_q = dq;
			e.first_in_chunk = 0;
			if (STORE) {
				uint4 w;
				w.x = __byte_perm(ab[0], ab[1], 0x5410); w.y = __byte_perm(ab[2], ab[3], 0x5410);
				w.z = __byte_perm(ab[4], ab[5], 0x5410); w.w = __byte_perm(ab[6], ab[7], 0x5410);
				*reinterpret_cast<uint4 *>(e.out + e.m_lo + e.rel) = w;
			}
			e.rel += 8;
			return;
		}
	}
	if constexpr (P == 0) {
		// low_pass boxcar (src/rtl_fm.c:351-371)
#pragma unroll
		for (int j = 0; j < 8; j++) {
			int xi, xq;
			scale_rot(v[j], j, rot, xi, xq, e.rdc_i, e.rdc_q);
			s.box_i += xi; s.box_q += xq;
			if (++s.box_n >= c.D) {
				int di = wrap16(s.box_i), dq = wrap16(s.box_q);
				s.box_i = 0; s.box_q = 0; s.box_n = 0;
				post_decim<P, SPEC, STORE>(c, k, s, e, di, dq);
			}
		}
	} else if constexpr (PL == 0) {
		// "wide" variant: every fifth_order pass scalar with the reference's int16 wrap
#pragma unroll
		for (int j = 0; j < 8; j++) {
			int xi, xq, oi, oq;
			scale_rot(v[j], j, rot, xi, xq, e.rdc_i, e.rdc_q);
			if (scalar_push<0, P, SPEC>(s, xi, xq, u + (unsigned)j, oi, oq)) { post_decim<P, SPEC, STORE>(c, k, s, e, oi, oq); }
		}
	} else {
		uint32_t x[8];
#pragma unroll
		for (int j = 0; j < 8; j++) { x[j] = scale_rot_pack(v[j], j, rot); }
		front_block_packed<P, SPEC, STORE>(c, k, s, e, x, u);
	}
}

// ------------------------------------------------------------------------------ back end
// First PCM index (counted from the start of the call) of the group low_pass_real sums into output o:
// the resampler adds `slow` per sample and emits when the running phase reaches `fast`
// (src/rtl_fm.c:396-407), so output o-1 is emitted by the first sample m with
// phase0 + (m+1)*slow >= o*fast.
__device__ __forceinline__ long long group_start(const FmDev &c, long long o, int phase0)
{
	if (!c.resample) { return o; }
	if (o <= 0) { return 0; }
	long long need = o * (long long)c.fast - (long long)phase0;
	return (need + c.slow - 1) / c.slow;
}

// deemph_filter step on the magic-reciprocal path with the loop-invariant part folded into xb:
//   xb = x + a/2 + K*a;   avg' = avg + umulhi(xb - avg - [a even && x <= avg], magic) - K
template <bool EVEN>
__device__ __forceinline__ int deemph_fast(int avg, int x, int xb, unsigned magic, int K)
{
	int n = xb - avg;
	if (EVEN) { n -= (x <= avg) ? 1 : 0; }
	return avg + (int)__umulhi((unsigned)n, magic) - K;
}

template <int PAD>
__device__ __forceinline__ int pcm_load(const int16_t *pcm_s, int m) { return (int)pcm_s[pcm_phys<PAD>(m)]; }

// The de-emphasis step as the replay / output loops see it: a state, a sample as loaded from the PCM buffer, a step.
// Integer form: deemph_fast above.  FP32 form (odd a): the reference's avg += trunc((d +- a/2) / a) is d / a rounded
// to the nearest integer, and an odd a has no ties.  Keep the state as the float U = 2^23 + 32768 + avg (an integer
// below 2^24, so one ulp is exactly 1) and build the sample X = 2^23 + 32768 + x straight from its 16 bits
// ((x ^ 0x8000) | 0x4B000000).  Then d = X - U is exact and fma(d, fl(1/a), U), rounded to nearest by the hardware,
// IS U + rn(d / a): the product's error (< |d| 2^-24 / a) is far below the distance of d / a from a half-integer
// (>= 1 / (2a)).  Two full-rate FP32 instructions on an 8-cycle dependency instead of subtract, 64-bit multiply-high
// and add -- the multiply-high (IMAD.HI) is what the back kernel's warps were waiting for.  Bit-exact by construction
// and by the parity suite; even a (ties round away from zero in the reference) keeps the integer form.
#define DF_BIAS 0x4B008000
template <bool EVEN, bool F32>
struct DeemphOp {
	typedef int State;
	typedef int Sample;
	int bias, K;
	unsigned magic;
	__device__ __forceinline__ DeemphOp(const FmDev &c) : bias(c.a_half + c.a_K * c.a), K(c.a_K), magic(c.a_magic) {}
	__device__ __forceinline__ State enter(int avg) const { return avg; }
	__device__ __forceinline__ int value(State s) const { return s; }
	typedef int Raw;                            // a sample as fetched (loops that fetch ahead carry these), conv() makes it a Sample
	__device__ __forceinline__ Raw fetch(const int16_t *p) const { return (int)*p; }
	__device__ __forceinline__ Sample conv(Raw r) const { return r; }
	__device__ __forceinline__ Sample load(const int16_t *p) const { return (int)*p; }
	// four samples from an 8-byte aligned address: one load
	__device__ __forceinline__ void load4(const int16_t *p, Sample &x0, Sample &x1, Sample &x2, Sample &x3) const
	{
		const uint2 w = *reinterpret_cast<const uint2 *>(p);
		x0 = lo16(w.x); x1 = hi16(w.x); x2 = lo16(w.y); x3 = hi16(w.y);
	}
	__device__ __forceinline__ State step(State s, Sample x) const { return deemph_fast<EVEN>(s, x, x + bias, magic, K); }
};
template <>
struct DeemphOp<false, true> {
	typedef float State;
	typedef float Sample;
	float inv_a;
	__device__ __forceinline__ DeemphOp(const FmDev &c) : inv_a(1.0f / (float)c.a) {}
	__device__ __forceinline__ State enter(int avg) const { return __int_as_float(DF_BIAS + avg); }
	__device__ __forceinline__ int value(State s) const { return __float_as_int(s) - DF_BIAS; }
	typedef unsigned Raw;
	__device__ __forceinline__ Raw fetch(const int16_t *p) const
	{
		unsigned v = *reinterpret_cast<const uint16_t *>(p);
		asm("" : "+r"(v));      // 32 bits from here on (left alone the compiler carries 16-bit values across loop edges two to a
		                        // register and pays a mask and a permute per sample to get them back)
		return v;
	}
	__device__ __forceinline__ Sample conv(Raw v) const { return __int_as_float((int)(v ^ 0x4B008000u)); }   // 16 bits: the xor sets the exponent too
	__device__ __forceinline__ Sample load(const int16_t *p) const
	{
		float x = __int_as_float((int)((unsigned)*reinterpret_cast<const uint16_t *>(p) ^ 0x4B008000u));
		asm("" : "+f"(x));      // a float from here on (same reason)
		return x;
	}
	__device__ __forceinline__ void load4(const int16_t *p, Sample &x0, Sample &x1, Sample &x2, Sample &x3) const
	{
		const uint2 w = *reinterpret_cast<const uint2 *>(p);
		unsigned magic = 0x4B008000u, l0, l1;
		asm("" : "+r"(magic));                 // in a register: (w & 0xffff) ^ magic is then ONE three-input logic instruction
		asm("lop3.b32 %0, %1, 0xffff, %2, 0x6a;" : "=r"(l0) : "r"(w.x), "r"(magic));
		asm("lop3.b32 %0, %1, 0xffff, %2, 0x6a;" : "=r"(l1) : "r"(w.y), "r"(magic));
		x0 = __int_as_float((int)l0); x1 = __int_as_float((int)((w.x >> 16) ^ magic));
		x2 = __int_as_float((int)l1); x3 = __int_as_float((int)((w.y >> 16) ^ magic));
	}
	__device__ __forceinline__ State step(State s, Sample x) const { return __fmaf_rn(__fsub_rn(x, s), inv_a, s); }
};
template <bool EVEN>
struct Deemph : DeemphOp<EVEN, !EVEN> {
	__device__ __forceinline__ Deemph(const FmDev &c) : DeemphOp<EVEN, !EVEN>(c) {}
};

// deemph_filter over PCM [m, m_end) of the shared buffer from BOTH bracket ends (replay before a
// piece).  The two trajectories are independent, the next sample is fetched one step ahead.
// A8: pcm_s + m is 8-byte aligned whenever m is a multiple of 4 (the back kernel's windows): a quad is ONE 8-byte load.
template <bool EVEN, int PAD, bool A8 = false>
__device__ __forceinline__ void back_replay(const FmDev &c, const int16_t *pcm_s, int m, int m_end, int &lo, int &hi)
{
	if (m >= m_end) { return; }
	if (c.a_use_magic) {
		const Deemph<EVEN> dm(c);
		typename Deemph<EVEN>::State l = dm.enter(lo), h = dm.enter(hi);
		// quads never straddle a padding step (128 is a multiple of 4): one address, four immediate offsets
		for (; (m & 3) != 0 && m < m_end; m++) {
			const typename Deemph<EVEN>::Sample x = dm.load(pcm_s + pcm_phys<PAD>(m));
			l = dm.step(l, x); h = dm.step(h, x);
		}
		// the next quad's samples are fetched before this quad's steps (the compiler does not move the loads across the loop
		// edge by itself); the last quad re-reads itself.  (Deeper read-ahead -- eight steps per trip with the next eight
		// samples in flight -- measured slower, session AA: the register shuffling costs more than the latency it hides.)
		if (m + 4 <= m_end) {
			const int16_t *q = pcm_s + pcm_phys<PAD>(m);
			typename Deemph<EVEN>::Sample x0, x1, x2, x3;
			if constexpr (A8) { dm.load4(q, x0, x1, x2, x3); } else { x0 = dm.load(q); x1 = dm.load(q + 1); x2 = dm.load(q + 2); x3 = dm.load(q + 3); }
#pragma unroll 2
			for (; m + 4 <= m_end; m += 4) {
				// (windows: the read-ahead of the last quad lands in the row's four samples of slack -- no clamp, so the
				// load's address does not hang on a compare and a select and can issue at the top of the trip)
				const int16_t *qn = A8 ? q + 4 : pcm_s + pcm_phys<PAD>(m + 8 <= m_end ? m + 4 : m);
				typename Deemph<EVEN>::Sample y0, y1, y2, y3;
				if constexpr (A8) { dm.load4(qn, y0, y1, y2, y3); } else { y0 = dm.load(qn); y1 = dm.load(qn + 1); y2 = dm.load(qn + 2); y3 = dm.load(qn + 3); }
				l = dm.step(l, x0); h = dm.step(h, x0);
				l = dm.step(l, x1); h = dm.step(h, x1);
				l = dm.step(l, x2); h = dm.step(h, x2);
				l = dm.step(l, x3); h = dm.step(h, x3);
				x0 = y0; x1 = y1; x2 = y2; x3 = y3;
				q = qn;
			}
		}
		for (; m < m_end; m++) {
			const typename Deemph<EVEN>::Sample x = dm.load(pcm_s + pcm_phys<PAD>(m));
			l = dm.step(l, x); h = dm.step(h, x);
		}
		lo = dm.value(l); hi = dm.value(h);
	} else {
		for (; m < m_end; m++) {
			const int x = pcm_load<PAD>(pcm_s, m);
			lo = deemph_step(c, lo, x);
			hi = deemph_step(c, hi, x);
		}
	}
}

// What a piece does to the states of an open bracket [lo, hi]: both ends are run through PCM [m, m_end);
// returns non-zero when either end moved at any step.
enum { PK_OPEN = 0, PK_EXACT = 1, PK_MERGED = 2, PK_IDENT = 3 };
template <bool EVEN, int PAD>
__device__ __forceinline__ int back_probe(const FmDev &c, const int16_t *pcm_s, int m, int m_end, int &lo, int &hi)
{
	const int bias = c.a_half + c.a_K * c.a, K = c.a_K;
	const unsigned magic = c.a_magic;
	int moved = 0;
	for (; m < m_end; m++) {
		const int x = pcm_load<PAD>(pcm_s, m);
		int nl, nh;
		if (c.a_use_magic) { nl = deemph_fast<EVEN>(lo, x, x + bias, magic, K); nh = deemph_fast<EVEN>(hi, x, x + bias, magic, K); }
		else { nl = deemph_step(c, lo, x); nh = deemph_step(c, hi, x); }
		moved |= (nl ^ lo) | (nh ^ hi);
		lo = nl; hi = nh;
	}
	return moved;
}

// audio DC block bookkeeping of one back-end lane (dc_block_audio_filter, src/rtl_fm.c:684-697)
struct AdcCtx {
	const int *adc;          // per-chunk average to subtract (null: stage off or pre-pass)
	long long *sums;         // pre-pass: per-chunk sum of the de-emphasised samples
	int chunk, box_n0, n_chunks;
	long long m_lo;
	int cur, sub;            // chunk of the running sample, its average
	long long acc;           // pre-pass accumulator of chunk `cur`
};
__device__ __forceinline__ void adc_flush(AdcCtx &a)
{
	if (a.sums && a.cur >= 0 && a.acc != 0) { atomicAdd(reinterpret_cast<unsigned long long *>(a.sums + 2 * a.cur), (unsigned long long)a.acc); }
	a.acc = 0;
}
__device__ __forceinline__ int adc_apply(const FmDev &c, AdcCtx &a, int m_rel, int x)
{
	const int ch = pcm_chunk(c, a.chunk, a.m_lo + m_rel, a.box_n0);
	if (ch != a.cur) {
		adc_flush(a);
		a.cur = ch;
		a.sub = a.adc ? a.adc[ch < a.n_chunks ? ch : a.n_chunks - 1] : 0;
	}
	if (a.sums) { a.acc += x; }
	return wrap16(x - a.sub);
}

// Outputs [oa, ob) of one lane from an exact state: per output, de-emphasise the group's samples,
// sum them and divide by the integer rate ratio (deemph_filter :673-680, low_pass_real :396-407).
// `phase` is the resampler phase at the first group's start; right after an emission it is < slow, so a
// group then has floor(fast/slow) samples, or one more when that does not yet reach `fast` (only the
// group a call inherits from the previous call can start with a larger phase).
// m is the running (buffer-relative) PCM index; avg the running de-emphasis state.
// The common shape of back_outputs -- de-emphasis on the reciprocal path, resampler on, every group regular (phase
// below `slow` at the first group's start), no audio DC block -- without the run-time switches: 32-bit counters, the
// group's quotient by a host-verified multiply-high, the next sample fetched one step ahead.  Same integers.
// LF: the integer rate ratio fast/slow when it is a compile-time value (a group is LF or LF + 1 samples: LF unrolled
// steps and one conditional one), 0: any ratio (loop).
template <bool EVEN, int PAD, int LF>
__device__ __forceinline__ void back_outputs_lean(const FmDev &c, const int16_t *pcm_s, int16_t *__restrict__ out, int n_out,
                                                  int &m, int &avg, int acc, int &phase_io)
{
	const Deemph<EVEN> de(c);
	typedef typename Deemph<EVEN>::Sample Smp;
	int phase = phase_io;
	const int lf = LF > 0 ? LF : c.lpr_div, slow = c.slow, fast = c.fast;
	const int dm = c.lpr_m, dsh = c.lpr_s, dadd = c.lpr_add;
	const int16_t *p = pcm_s + pcm_phys<PAD>(m);        // PAD == 0 here: consecutive samples are consecutive entries
	typename Deemph<EVEN>::State a = de.enter(avg);
	int mm = m;
	int16_t *op = out;
	for (int n = 0; n < n_out; n++) {
		int ph = phase + lf * slow;
		const bool extra = ph < fast;
		if (extra) { ph += slow; }
		phase = ph - fast;
		// (the reference's int16 store of avg changes nothing: a step moves avg towards x and never past it, so avg stays
		// inside the int16 range of the inputs and of the carried state -- no wrap16 on the accumulate)
		if constexpr (LF > 0 && PAD == 0) {
#pragma unroll
			for (int j = 0; j < LF; j++) {
				const Smp x = de.load(p + j);
				a = de.step(a, x);
				acc += de.value(a);
			}
			if (extra) {
				const Smp x = de.load(p + LF);
				a = de.step(a, x);
				acc += de.value(a);
			}
			p += LF + (extra ? 1 : 0);
			mm += LF + (extra ? 1 : 0);
		} else if constexpr (PAD == 0) {
			// any ratio (the undecimated wbfm shape has 50 samples per output): quads, then the rest
			const int len = lf + (extra ? 1 : 0);
			int j = 0;
			if (len >= 4) {
				Smp x0 = de.load(p), x1 = de.load(p + 1), x2 = de.load(p + 2), x3 = de.load(p + 3);
#pragma unroll 2
				for (; j + 4 <= len; j += 4) {
					const int16_t *pn = p + (j + 8 <= len ? 4 : 0);
					const Smp y0 = de.load(pn), y1 = de.load(pn + 1), y2 = de.load(pn + 2), y3 = de.load(pn + 3);
					a = de.step(a, x0); acc += de.value(a);
					a = de.step(a, x1); acc += de.value(a);
					a = de.step(a, x2); acc += de.value(a);
					a = de.step(a, x3); acc += de.value(a);
					x0 = y0; x1 = y1; x2 = y2; x3 = y3;
					p += 4;
				}
			}
			for (; j < len; j++) {
				const Smp x = de.load(p++);
				a = de.step(a, x); acc += de.value(a);
			}
			mm += len;
		} else {
			const int len = lf + (extra ? 1 : 0);
			for (int j = 0; j < len; j++) {
				const Smp x = de.load(pcm_s + pcm_phys<PAD>(mm));
				a = de.step(a, x);
				acc += de.value(a);
				mm++;
			}
		}
		int q = __mulhi(acc, dm);
		if (dadd) { q += acc; }
		q >>= dsh;
		q += (int)((unsigned)q >> 31);
		*op++ = (int16_t)q;
		acc = 0;
	}
	m = mm; avg = de.value(a); phase_io = phase;
}

template <bool EVEN, int PAD>
__device__ __forceinline__ void back_outputs(const FmDev &c, const int16_t *pcm_s, int16_t *__restrict__ out,
                                             long long oa, long long ob, int &m, int &avg, int acc, int phase,
                                             AdcCtx *ax, bool store)
{
	const int bias = c.a_half + c.a_K * c.a, K = c.a_K;
	const unsigned magic = c.a_magic;
	const int lf = c.resample ? c.fast / c.slow : 1;
	const bool fast_path = c.deemph && c.a_use_magic;
	if (fast_path && c.resample && c.lpr_ok && phase < c.slow && ax == nullptr && store) {
		// the two ratios the wbfm presets produce get unrolled bodies (300 k -> 48 k: 6, 170 k -> 32 k: 5)
		if (PAD == 0 && c.lpr_div == 6) { back_outputs_lean<EVEN, PAD, 6>(c, pcm_s, out + oa, (int)(ob - oa), m, avg, acc, phase); }
		else if (PAD == 0 && c.lpr_div == 5) { back_outputs_lean<EVEN, PAD, 5>(c, pcm_s, out + oa, (int)(ob - oa), m, avg, acc, phase); }
		else { back_outputs_lean<EVEN, PAD, 0>(c, pcm_s, out + oa, (int)(ob - oa), m, avg, acc, phase); }
		return;
	}
	int x = (oa < ob) ? pcm_load<PAD>(pcm_s, m) : 0;
	for (long long o = oa; o < ob; o++) {
		int len = 1;
		if (c.resample) {
			if (phase >= c.slow) { len = (c.fast - phase + c.slow - 1) / c.slow; }   // first group of a call only
			else { len = lf; if (phase + len * c.slow < c.fast) { len++; } }
			phase += len * c.slow - c.fast;
		}
		for (int j = 0; j < len; j++) {
			int xn = pcm_load<PAD>(pcm_s, m + 1);      // one entry of slack exists past the last sample
			if (fast_path) { avg = deemph_fast<EVEN>(avg, x, x + bias, magic, K); x = wrap16(avg); }
			else if (c.deemph) { avg = deemph_step(c, avg, x); x = wrap16(avg); }
			if (ax) { x = adc_apply(c, *ax, m, x); }
			acc = add_w(acc, x);
			x = xn; m++;
		}
		if (store) { out[o] = (int16_t)(c.resample ? div_small_quotient(acc, c.lpr_div) : acc); }
		acc = 0;
	}
}

// ---- per-lane windows of global PCM staged through shared memory (fm_back_kernel).
// A lane of the back kernel walks its own piece of the call's PCM: read straight from global memory that is one 2-byte
// load per step to 32 different lines per warp -- 32 trips through the L1 tag stage per step, which at one PCM sample per
// input sample (fm2a) costs more than the arithmetic.  Instead the warp copies, for each of its lanes in turn, the next
// WS samples of that lane's piece with coalesced 4-byte asynchronous copies (cp.async: global -> shared without a trip
// through registers) into a row of shared memory, and the lanes then run the unchanged replay / output loops out of
// their rows.  Two buffers per warp: the copies of the NEXT window are in flight while the lanes work through the
// current one (in a synchronous version the warps spent much of their time waiting for their own fills and idle at the
// item barriers behind them).  Where a lane's next window starts is known before the
// current one is processed: a replay consumes the whole window, and the samples n resampler groups consume depend on
// the phase alone.  Odd row stride: lanes reading the same offset of their rows hit 32 different banks.
template <int WS>
struct LaneWin {
	static constexpr int ROW = WS / 2 + 2;      // words per row: even (8-byte copies), lanes 16 apart share a bank
	static constexpr int BUF = 32 * ROW;        // words per buffer (one row per lane)
	const int16_t *g;         // the channel's PCM in global memory
	uint32_t *rows;           // this warp's two buffers
	int lane;
};
__device__ __forceinline__ void cp_async8(uint32_t dst, const void *src)
{
	asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// all 32 lanes: lane l's row of buffer `buf` <- g[base_l .. base_l + WS), base_l a multiple of 4 samples (8-byte copies:
// the copy instruction, not its bytes, is what the load/store unit charges for: 64 four-byte copies per window keep
// the unit busy most of the time); one commit group per call
#define WIN_ALIGN 3
template <int WS>
__device__ __forceinline__ void win_issue(const LaneWin<WS> &w, int buf, int base)
{
	constexpr int NV = WS / 128;
	const uint32_t dst0 = smem_u32(w.rows + buf * LaneWin<WS>::BUF + 2 * w.lane);
	// fully unrolled: the destination of every copy is dst0 plus a compile-time offset, a row costs one shuffle, one
	// address and its copies
	const char *gl = reinterpret_cast<const char *>(w.g) + 8 * w.lane;      // this lane's eight bytes of every row
#pragma unroll
	for (int l = 0; l < 32; l++) {
		const unsigned b = (unsigned)__shfl_sync(0xffffffffu, base, l);       // bases are never negative: one 32 x 32 -> 64 multiply-add
		const char *src = gl + 2ull * b;
		const uint32_t dst = dst0 + (uint32_t)(l * LaneWin<WS>::ROW * 4);
#pragma unroll
		for (int i = 0; i < NV; i++) { cp_async8(dst + 256u * i, src + 256 * i); }
	}
	cp_async_commit();
}
// back_replay over PCM [m, m_end) through windows; every lane of the warp takes part (an empty range for lanes with
// nothing to do: they keep re-reading the window they stand on)
template <bool EVEN, int WS>
__device__ __forceinline__ void win_replay(const FmDev &c, const LaneWin<WS> &w, int m, int m_end, int &lo, int &hi)
{
	if (!__any_sync(0xffffffffu, m < m_end)) { return; }
	int base = m & ~WIN_ALIGN, buf = 0;
	__syncwarp();
	win_issue(w, 0, base);
	for (;;) {
		const int e = m_end < base + WS ? m_end : base + WS;
		const int m_next = m < e ? e : m;
		const bool more = __any_sync(0xffffffffu, m_next < m_end);
		if (more) { win_issue(w, buf ^ 1, m_next & ~WIN_ALIGN); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
		__syncwarp();
		const int16_t *row = reinterpret_cast<const int16_t *>(w.rows + buf * LaneWin<WS>::BUF + w.lane * LaneWin<WS>::ROW);
		if (m < e) { back_replay<EVEN, 0, true>(c, row - base, m, e, lo, hi); }      // rows and bases are 8-byte aligned
		__syncwarp();                          // every lane is through with this buffer before the next fill but one lands in it
		if (!more) { break; }
		m = m_next; base = m_next & ~WIN_ALIGN; buf ^= 1;
	}
}
// back_probe over PCM [m, m_end) through windows (an open bracket's piece); returns the lane's `moved` word
template <bool EVEN, int WS>
__device__ __forceinline__ int win_probe(const FmDev &c, const LaneWin<WS> &w, int m, int m_end, int &lo, int &hi)
{
	int moved = 0;
	if (!__any_sync(0xffffffffu, m < m_end)) { return moved; }
	int base = m & ~WIN_ALIGN, buf = 0;
	__syncwarp();
	win_issue(w, 0, base);
	for (;;) {
		const int e = m_end < base + WS ? m_end : base + WS;
		const int m_next = m < e ? e : m;
		const bool more = __any_sync(0xffffffffu, m_next < m_end);
		if (more) { win_issue(w, buf ^ 1, m_next & ~WIN_ALIGN); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
		__syncwarp();
		const int16_t *row = reinterpret_cast<const int16_t *>(w.rows + buf * LaneWin<WS>::BUF + w.lane * LaneWin<WS>::ROW);
		if (m < e) { moved |= back_probe<EVEN, 0>(c, row - base, m, e, lo, hi); }
		__syncwarp();
		if (!more) { break; }
		m = m_next; base = m_next & ~WIN_ALIGN; buf ^= 1;
	}
	return moved;
}
// The lean output loop (back_outputs_lean: reciprocal de-emphasis, resampler on, regular groups, no audio DC block)
// through windows.  Driven by samples, not by groups: a window is used to its last sample and a resampler group may
// straddle two windows (accumulator, phase and the samples the group still needs are lane state), so the window size
// is independent of the rate ratio.  The lane stops with the sample that completes its last output -- known up front:
// n groups end with the first sample that takes the running phase to n * fast (low_pass_real, src/rtl_fm.c:396-407).
template <bool EVEN, int WS>
__device__ __forceinline__ void win_outputs(const FmDev &c, const LaneWin<WS> &w, int16_t *__restrict__ op, int remaining, int &m, int &avg,
                                            int acc, int phase)
{
	if (!__any_sync(0xffffffffu, remaining > 0)) { return; }
	const Deemph<EVEN> de(c);
	typedef typename Deemph<EVEN>::Sample Smp;
	const int lf = c.lpr_div, slow = c.slow, fast = c.fast;
	const int dm = c.lpr_m, dsh = c.lpr_s, dadd = c.lpr_add;
	typename Deemph<EVEN>::State a = de.enter(avg);
	int mm = m;
	const int m_stop = remaining > 0 ? mm + (int)(((long long)remaining * fast - phase + slow - 1) / slow) : mm;
	int g_left = 0;                            // samples the group in progress still needs
	if (remaining > 0) {
		int ph = phase + lf * slow;
		const bool extra = ph < fast;
		if (extra) { ph += slow; }
		phase = ph - fast; g_left = lf + (extra ? 1 : 0);
	}
	auto emit = [&]() {                        // the group is complete: its output, then the next group's length
		int q = __mulhi(acc, dm);
		if (dadd) { q += acc; }
		q >>= dsh;
		q += (int)((unsigned)q >> 31);
		*op++ = (int16_t)q;
		acc = 0;
		int ph = phase + lf * slow;
		const bool extra = ph < fast;
		if (extra) { ph += slow; }
		phase = ph - fast; g_left = lf + (extra ? 1 : 0);
	};
	int base = mm & ~WIN_ALIGN, buf = 0;
	__syncwarp();
	win_issue(w, 0, base);
	for (;;) {
		const int e = m_stop < base + WS ? m_stop : base + WS;
		const int m_next = mm < e ? e : mm;
		const bool more = __any_sync(0xffffffffu, m_next < m_stop);
		if (more) { win_issue(w, buf ^ 1, m_next & ~WIN_ALIGN); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
		__syncwarp();
		const int16_t *p = reinterpret_cast<const int16_t *>(w.rows + buf * LaneWin<WS>::BUF + w.lane * LaneWin<WS>::ROW) + (mm - base);
		// run by run: what is left of the group in progress, or of the window (a stream of quads fetched two ahead with a
		// per-sample path for the quads that hold a group boundary measured slower, session AA)
		while (mm < e) {
			int run = e - mm;
			if (run > g_left) { run = g_left; }
			int j = 0;
			// up to the next multiple of 4 samples (rows and bases are 8-byte aligned: the position in the row has mm's low bits)
			for (; ((mm + j) & 3) != 0 && j < run; j++) {
				const Smp x = de.load(p++);
				a = de.step(a, x); acc += de.value(a);
			}
			if (j + 4 <= run) {                    // quads, one 8-byte load each, the next quad fetched ahead (see back_replay)
				Smp x0, x1, x2, x3;
				de.load4(p, x0, x1, x2, x3);
#pragma unroll 2
				for (; j + 4 <= run; j += 4) {
					const int16_t *pn = p + 4;             // past the run's end at most into the row's slack
					Smp y0, y1, y2, y3;
					de.load4(pn, y0, y1, y2, y3);
					a = de.step(a, x0); acc += de.value(a);
					a = de.step(a, x1); acc += de.value(a);
					a = de.step(a, x2); acc += de.value(a);
					a = de.step(a, x3); acc += de.value(a);
					x0 = y0; x1 = y1; x2 = y2; x3 = y3;
					p += 4;
				}
			}
			for (; j < run; j++) {
				const Smp x = de.load(p++);
				a = de.step(a, x); acc += de.value(a);
			}
			mm += run; g_left -= run;
			if (g_left == 0) { emit(); }
		}
		__syncwarp();
		if (!more) { break; }
		base = m_next & ~WIN_ALIGN; buf ^= 1;
	}
	m = mm; avg = de.value(a);
}

// Runs blocks [t, t_end) of one segment; chunk bookkeeping shared by the replay and the owned part.
// Entering chunk `idx`: flush the reduction pre-pass sums of the chunk just left, fetch the new chunk's scalars.
template <bool STORE>
__device__ __forceinline__ void chunk_enter(const FmDev &c, const FmCall &k, EmitCtx &e, int ch, int idx)
{
	if (k.reduce_mode == 1 && STORE && (e.red_t != 0 || e.red_p != 0)) {
		long long *sm = k.sums + 2 * ((size_t)ch * k.n_chunks + e.chunk_idx);
		atomicAdd(reinterpret_cast<unsigned long long *>(sm), (unsigned long long)e.red_t);
		atomicAdd(reinterpret_cast<unsigned long long *>(sm + 1), (unsigned long long)e.red_p);
	}
	e.red_t = 0; e.red_p = 0;
	e.chunk_idx = idx;
	const size_t ci = (size_t)ch * k.n_chunks + (idx < k.n_chunks ? idx : k.n_chunks - 1);
	if (k.rdc) { e.rdc_i = k.rdc[2 * ci]; e.rdc_q = k.rdc[2 * ci + 1]; }
	if (k.sqz) { e.sq_zero = k.sqz[ci]; }
	if (c.post_ds > 1) { e.pds_acc = 0; e.pds_cnt = 0; }       // groups never span chunks
}

// chunk start inside front_run: every pass forgets the odd sample it was holding (SURVEY F7).  Without passes a chunk
// shorter than the boxcar may complete none: fm_demod then carries lowpassed[-2], lowpassed[-1] (src/rtl_fm.c:612-613),
// which the pinned reference reads as 0 (DESIGN.md §4.1).  first_in_chunk still set here means the chunk just left
// emitted nothing; only the FM discriminator reads pre.  The call's own first chunk start is not counted (front_item)
template <int P, int SPEC, bool STORE>
__device__ __forceinline__ void front_chunk_start(const FmDev &c, const FmCall &k, FrontState<P, SPEC> &s, EmitCtx &e, int ch)
{
	if constexpr (P == 0) { if (e.first_in_chunk) { s.pre_i = 0; s.pre_q = 0; } }
	e.first_in_chunk = 1;
	if (SPEC == 2) { chunk_enter<STORE>(c, k, e, ch, e.chunk_idx + 1); }
#pragma unroll
	for (int l = 0; l < FrontState<P, SPEC>::PL; l++) {
#pragma unroll
		for (int j = 5; j > 0; j--) { s.h[l][j] = s.h[l][j - 1]; }
	}
}

__device__ __forceinline__ void ldg256_after(const int16_t *p, uint32_t (&v)[8], uint32_t dep)
{
	// `dep` is not used by the instructions: it only orders the loads behind the value's producer
	asm volatile("ld.global.nc.L2::256B.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
	             "ld.global.nc.L2::256B.v4.u32 {%4,%5,%6,%7}, [%8+16];"
	             : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]), "=r"(v[4]), "=r"(v[5]), "=r"(v[6]), "=r"(v[7])
	             : "l"(p), "r"(dep));
}

template <int P, int SPEC, bool STORE>
__device__ __forceinline__ void front_run(const FmDev &c, const FmCall &k, FrontState<P, SPEC> &s, EmitCtx &e,
                                          const int16_t *__restrict__ in, int t, int t_end, int t_last, unsigned &u, int ch)
{
	if (t >= t_end) { return; }
	constexpr bool INPLACE = FrontState<P, SPEC>::PL > 0;   // packed passes: the next block is loaded into the registers the scale just freed
	uint32_t v[8], vn[8];
	ldg256(in + 2 * (size_t)t, v);
	for (; t < t_end; t += 8) {
		const int tn = t + 8 <= t_last ? t + 8 : t_last;       // next block, clamped to the segment's last one
		if constexpr (!INPLACE) { ldg256(in + 2 * (size_t)tn, vn); }
		// pull the stream into L2 well ahead of the register prefetch (each thread walks its own region)
		if ((t & RXB_L2_MASK) == 0) {
			const int tp = min(t + RXB_L2_AHEAD, t_last);               // never past the segment
			asm volatile("prefetch.global.L2 [%0];" ::"l"(in + 2 * (size_t)tp));
		}
		if (u >= (unsigned)k.chunk) { u = 0u; }
		// a lane meets a chunk start once in chunk/8 blocks.  Left alone, ptxas if-converts the bookkeeping into
		// ~16 predicated-off moves in EVERY block; a loop (trip count k.one == 1, unknown to the compiler) cannot
		// be predicated, so the common path pays one branch
		if (u == 0u) {
#pragma unroll 1
			for (int z = 0; z < k.one; z++) { front_chunk_start<P, SPEC, STORE>(c, k, s, e, ch); }
		}
		if constexpr (INPLACE) {
			// scale first; the block's registers are free from here on, so the next block is loaded
			// straight into them and has the whole rest of this block's work to arrive
			uint32_t x[8];
			const bool rot = Spec<SPEC>::rotate(c);
#pragma unroll
			for (int j = 0; j < 8; j++) { x[j] = scale_rot_pack(v[j], j, rot); }
			ldg256_after(in + 2 * (size_t)tn, v, x[7]);
			front_block_packed<P, SPEC, STORE>(c, k, s, e, x, u);
			u += 8u;
		} else {
			front_block<P, SPEC, STORE>(c, k, s, e, v, u);
			u += 8u;
			// keep the consumer of the prefetched block BEHIND this block's work: without the (empty) asm the
			// compiler copies vn right after issuing the load and every warp then waits out the full DRAM latency
			asm volatile("" : "+r"(vn[0]), "+r"(vn[1]), "+r"(vn[2]), "+r"(vn[3]), "+r"(vn[4]), "+r"(vn[5]), "+r"(vn[6]), "+r"(vn[7])
			             : "r"(e.rel), "r"(s.pre_i));
#pragma unroll
			for (int j = 0; j < 8; j++) { v[j] = vn[j]; }
		}
	}
}

// ---- the any-length front end: calls whose chunk or length is not a multiple of 8 complex samples without passes, and
// one read of any even length per call with fifth_order passes (rxb200_fm_process_read).
// With passes the call is one chunk of n complex samples.  Pass l runs over L_l = 2n >> l int16 (src/rtl_fm.c:759-776):
// ceil(L_l / 2) I and floor(L_l / 2) Q samples, so in-chunk index i is a pair while i < n >> l, and index n >> l is an I
// sample alone when L_l is odd.  A pass takes only the first samples of the previous pass's outputs; the windows of the
// passes still advanced over the rest.  Only the last 2^P samples of a read can meet such an end (tail_push); the rest
// run through scalar_push.

// generic_fir on the I lane alone (the Q component's count ends one sample earlier)
__device__ __forceinline__ int droop9_i(uint32_t (&h)[9], const int (&c)[6], int di)
{
	int ai = mul_w(lo16(h[0]) + lo16(h[8]), c[1]);
	ai = add_w(ai, mul_w(lo16(h[1]) + lo16(h[7]), c[2]));
	ai = add_w(ai, mul_w(lo16(h[2]) + lo16(h[6]), c[3]));
	ai = add_w(ai, mul_w(lo16(h[3]) + lo16(h[5]), c[4]));
	ai = add_w(ai, mul_w(lo16(h[4]), c[5]));
#pragma unroll
	for (int j = 0; j < 8; j++) { h[j] = (h[j] & 0xffff0000u) | (h[j + 1] & 0xffffu); }
	h[8] = (h[8] & 0xffff0000u) | ((uint32_t)di & 0xffffu);
	return wrap16(ai >> 15);
}

// The lone I sample left after the passes when L_P is odd (src/rtl_fm.c:770-790, :612-613): the droop FIR and rms() count
// it, the squelch zeroes it, raw mode emits it, and fm_demod's carry becomes (last pair's Q, lone I).
template <int P, bool STORE>
__device__ __forceinline__ void lone_post(const FmDev &c, const FmCall &k, FrontState<P, 2> &s, EmitCtx &e, int di)
{
	if (c.fir_on) { di = droop9_i(s.fh, c.fir, di); }
	if (k.reduce_mode == 1) {
		if (STORE) { e.red_t += di; e.red_p += (long long)di * di; }
		return;
	}
	if (e.sq_zero) { di = 0; }
	if (c.mode == RXB200_MODE_FM) { s.pre_i = s.pre_q; s.pre_q = di; }
	else if (c.mode == RXB200_MODE_RAW && STORE && k.reduce_mode == 0) { e.out[2 * (e.m_lo + e.rel)] = (int16_t)di; }
}

// scalar_push near the end of a read: the sample enters pass L (or, L == P, the stages after the passes) as a pair, as an
// I sample alone (q false), or not at all
template <int L, int P, bool STORE>
__device__ __forceinline__ void tail_push(const FmDev &c, const FmCall &k, FrontState<P, 2> &s, EmitCtx &e, int xi, int xq,
                                          unsigned idx, bool q, unsigned n)
{
	if constexpr (L > 0) {
		if (idx >= (n >> L)) {
			if (idx > (n >> L) || ((n >> (L - 1)) & 1u) == 0u) { return; }
			q = false;
		}
	}
	if constexpr (L == P) {
		if (q) { post_decim<P, 2, STORE>(c, k, s, e, xi, xq); } else { lone_post<P, STORE>(c, k, s, e, xi); }
	} else {
		if (idx & 1u) { s.pi[L] = xi; if (q) { s.pq[L] = xq; } return; }
		if (idx == 0u) {
#pragma unroll
			for (int j = 0; j < 5; j++) { s.wi[L][j] = s.wi[L][j + 1]; if (q) { s.wq[L][j] = s.wq[L][j + 1]; } }
		} else {
#pragma unroll
			for (int j = 0; j < 4; j++) { s.wi[L][j] = s.wi[L][j + 2]; if (q) { s.wq[L][j] = s.wq[L][j + 2]; } }
			s.wi[L][4] = s.pi[L]; if (q) { s.wq[L][4] = s.pq[L]; }
		}
		s.wi[L][5] = xi; if (q) { s.wq[L][5] = xq; }
		int yi = wrap16((s.wi[L][0] + (s.wi[L][1] + s.wi[L][4]) * 5 + (s.wi[L][2] + s.wi[L][3]) * 10 + s.wi[L][5]) >> 4);
		int yq = wrap16((s.wq[L][0] + (s.wq[L][1] + s.wq[L][4]) * 5 + (s.wq[L][2] + s.wq[L][3]) * 10 + s.wq[L][5]) >> 4);
		tail_push<L + 1, P, STORE>(c, k, s, e, yi, yq, idx >> 1, q, n);
	}
}

// front_run of the any-length front end: one 32-bit load per complex sample, since a channel's base, and with it every
// block, is only 4-byte aligned (the loads of a block issue together, none past t_end: the segment that ends the channel
// may end inside a block).  u is the in-chunk index of sample t.  Without passes a chunk may start between any two
// samples, so the chunk bookkeeping -- rotation phase, F8's first_in_chunk, the per-chunk scalars and sums -- runs before
// every sample and the samples on each side of a boundary see their own chunk's values; with passes the call is one
// chunk (k.chunk == k.n), and its samples from (n >> P) << P on go through tail_push.
template <int P, int SPEC, bool STORE>
__device__ __forceinline__ void front_run_any(const FmDev &c, const FmCall &k, FrontState<P, SPEC> &s, EmitCtx &e,
                                              const uint32_t *__restrict__ in, int t, int t_end, unsigned &u, int ch)
{
	const bool rot = Spec<SPEC>::rotate(c);
	const unsigned n = (unsigned)k.n;
	const unsigned tail = (n >> P) << P;              // from here on a sample may meet the end of a pass's count
	const int t_main = P == 0 ? t_end : t + (int)(u >= tail ? 0u : min(tail - u, (unsigned)(t_end - t)));
	for (; t < t_main; t += 8) {
		const int nb = t_main - t;
		uint32_t v[8];
#pragma unroll
		for (int j = 0; j < 8; j++) { v[j] = j < nb ? __ldg(in + t + j) : 0u; }
#pragma unroll
		for (int j = 0; j < 8; j++) {
			if (j < nb) {
				if constexpr (P == 0) { if (u >= (unsigned)k.chunk) { u = 0u; } }
				if (u == 0u) {
#pragma unroll 1
					for (int z = 0; z < k.one; z++) { front_chunk_start<P, SPEC, STORE>(c, k, s, e, ch); }
				}
				int xi, xq;
				scale_rot(v[j], (int)(u & 3u), rot, xi, xq, e.rdc_i, e.rdc_q);   // rotate16_90 restarts with every chunk
				if constexpr (P == 0) {
					u++;
					s.box_i += xi; s.box_q += xq;
					if (++s.box_n >= c.D) {
						int di = wrap16(s.box_i), dq = wrap16(s.box_q);
						s.box_i = 0; s.box_q = 0; s.box_n = 0;
						post_decim<0, SPEC, STORE>(c, k, s, e, di, dq);
					}
				} else {
					int oi, oq;
					if (scalar_push<0, P, SPEC>(s, xi, xq, u, oi, oq)) { post_decim<P, SPEC, STORE>(c, k, s, e, oi, oq); }
					u++;
				}
			}
		}
	}
	if constexpr (P > 0) {
		t = t_main > t_end ? t_end : t_main;
#pragma unroll 1
		for (; t < t_end; t++, u++) {                 // u >= tail > 0: no chunk starts here
			int xi, xq;
			scale_rot(__ldg(in + t), (int)(u & 3u), rot, xi, xq, e.rdc_i, e.rdc_q);
			tail_push<0, P, STORE>(c, k, s, e, xi, xq, u, true, n);
		}
	}
}

// The any-length front end keeps every pass scalar (FrontState<P, 2>); the carry keeps the handle's layout
// (fm_state_words), so that calls of every entry point can follow one another: c.PL packed levels, lanes biased by
// 128 << l, holding the pass's last six inputs -- the window a..e of the next chunk's first output, then the sample an
// even count left pending -- and the scalar levels after them.  Without passes these are front_load / front_store's words.
template <int P, int SPEC>
__device__ __forceinline__ void any_load(const FmDev &c, FrontState<P, SPEC> &s, const uint32_t *g)
{
	s.box_i = (int)g[ST_BOX_I]; s.box_q = (int)g[ST_BOX_Q]; s.box_n = (int)g[ST_BOX_N];
	s.pre_i = (int)g[ST_PRE_I]; s.pre_q = (int)g[ST_PRE_Q];
	const int PL = P == 0 ? 0 : c.PL;
#pragma unroll
	for (int l = 0; l < P; l++) {
		if (l < PL) {
			const int b = 128 << l;
			s.wi[l][0] = 0; s.wq[l][0] = 0;       // a: shifted out before the next output
#pragma unroll
			for (int j = 0; j < 5; j++) { const uint32_t w = g[ST_HDR + 6 * l + j]; s.wi[l][j + 1] = (int)(w & 0xffffu) - b; s.wq[l][j + 1] = (int)(w >> 16) - b; }
			const uint32_t w = g[ST_HDR + 6 * l + 5];
			s.pi[l] = (int)(w & 0xffffu) - b; s.pq[l] = (int)(w >> 16) - b;
		} else {
			const uint32_t *gl = g + ST_HDR + 6 * PL + 7 * (l - PL);
#pragma unroll
			for (int j = 0; j < 6; j++) { s.wi[l][j] = lo16(gl[j]); s.wq[l][j] = hi16(gl[j]); }
			s.pi[l] = lo16(gl[6]); s.pq[l] = hi16(gl[6]);
		}
	}
#pragma unroll
	for (int j = 0; j < 9; j++) { s.fh[j] = g[ST_HDR + 6 * PL + 7 * (P - PL) + j]; }
}

template <int P, int SPEC>
__device__ __forceinline__ void any_store(const FmDev &c, const FrontState<P, SPEC> &s, uint32_t *g)
{
	g[ST_BOX_I] = (uint32_t)s.box_i; g[ST_BOX_Q] = (uint32_t)s.box_q; g[ST_BOX_N] = (uint32_t)s.box_n;
	g[ST_PRE_I] = (uint32_t)s.pre_i; g[ST_PRE_Q] = (uint32_t)s.pre_q;
	const int PL = P == 0 ? 0 : c.PL;
#pragma unroll
	for (int l = 0; l < P; l++) {
		if (l < PL) {
			const int b = 128 << l;
#pragma unroll
			for (int j = 0; j < 5; j++) { g[ST_HDR + 6 * l + j] = pack2(s.wi[l][j + 1] + b, s.wq[l][j + 1] + b); }
			g[ST_HDR + 6 * l + 5] = pack2(s.pi[l] + b, s.pq[l] + b);
		} else {
			uint32_t *gl = g + ST_HDR + 6 * PL + 7 * (l - PL);
#pragma unroll
			for (int j = 0; j < 6; j++) { gl[j] = pack2(s.wi[l][j], s.wq[l][j]); }
			gl[6] = pack2(s.pi[l], s.pq[l]);
		}
	}
#pragma unroll
	for (int j = 0; j < 9; j++) { g[ST_HDR + 6 * PL + 7 * (P - PL) + j] = s.fh[j]; }
}

// geometry of one work item (one CTA stretch of one channel)
struct Item {
	int ch, b;
	long long m_lo;
	int m_own, m_hi;           // relative to m_lo
	int box_n0, phase0;
};
__device__ __forceinline__ Item make_item(const FmDev &c, const FmCall &k, int work)
{
	Item it;
	it.ch = work / k.n_cta;
	it.b = work % k.n_cta;
	const uint32_t *carry = k.carry_in + (size_t)it.ch * k.state_words;
	it.box_n0 = (int)carry[ST_BOX_N];
	it.phase0 = (int)carry[ST_LPR_PHASE];
	const long long own_lo = (long long)it.b * k.n_own * k.Sf;
	long long own_hi = own_lo + (long long)k.n_own * k.Sf;
	if (own_hi > k.n) { own_hi = k.n; }
	long long buf_lo = own_lo - (long long)k.n_extra * k.Sf;
	if (buf_lo < 0 || k.pcm_g) { buf_lo = 0; }      // global PCM: the buffer is the whole call, indices are absolute
	it.m_lo = dec_before(c, buf_lo, it.box_n0);
	it.m_own = (int)(dec_before(c, own_lo, it.box_n0) - it.m_lo);
	it.m_hi = (int)(dec_before(c, own_hi, it.box_n0) - it.m_lo);
	return it;
}

// ---- front end of one work item: one segment per thread (tid 0..T-1).  ANY: the any-length front end (front_run_any)
template <int P, int SPEC, bool ANY>
__device__ __forceinline__ void front_item(const FmDev &c, const FmCall &k, const Item &it, int tid, int16_t *pcm_s)
{
	const uint32_t *carry = k.carry_in + (size_t)it.ch * k.state_words;
	const long long g = (long long)it.b * k.n_own + (tid - k.n_extra);
	const long long start = g * k.Sf;
	if (g < 0 || start >= k.n) { return; }
	// the squelch/level pre-pass only sums: the warm-up segments belong to the previous item's sums
	if (SPEC == 2 && k.reduce_mode == 1 && tid < k.n_extra) { return; }
	const long long end = start + k.Sf < k.n ? start + k.Sf : k.n;
	long long t0 = start - k.halo;
	FrontState<P, SPEC> s;
	if (t0 <= 0) {
		t0 = 0;
		if constexpr (ANY) { any_load<P, SPEC>(c, s, carry); } else { front_load<P, SPEC>(s, carry); }
	}
	else {
		front_zero<P, SPEC>(s);
		if (P == 0) { s.box_n = (int)((t0 + it.box_n0) % c.D); }
	}
	unsigned u = (unsigned)(t0 % k.chunk);
	const long long m0 = dec_before(c, t0, it.box_n0);
	EmitCtx e;
	e.pcm = pcm_s; e.out = k.out + (size_t)it.ch * (size_t)k.out_stride; e.m_lo = it.m_lo;
	e.rel = (int)(m0 - it.m_lo);
	// whether the chunk in progress at t0 has emitted nothing yet.  At the call's start the previous call's carry already
	// holds the empty-chunk rule, so 0: the first chunk start must not apply it again
	e.first_in_chunk = 0;
	if (P == 0 && t0 > 0) { e.first_in_chunk = (dec_raw(c, t0 - u, it.box_n0) == dec_raw(c, t0, it.box_n0)) ? 1 : 0; }
	e.rdc_i = e.rdc_q = 0; e.sq_zero = 0; e.red_t = 0; e.red_p = 0;
	e.pds_acc = 0; e.pds_cnt = 0; e.chunk_idx = 0;
	if (SPEC == 2) {
		e.chunk_idx = (int)(t0 / k.chunk);
		if (u != 0u) { chunk_enter<false>(c, k, e, it.ch, e.chunk_idx); }   // mid-chunk start: fetch this chunk's scalars
		else { e.chunk_idx -= 1; }                                           // the first block enters the chunk itself
		if (c.post_ds > 1) { e.pds_cnt = (int)((dec_raw(c, t0, it.box_n0) - dec_raw(c, t0 - u, it.box_n0)) % c.post_ds); }
	}
	// offsets relative to t0 fit 32 bits (a segment plus its halo)
	const int16_t *__restrict__ in = k.in + 2 * ((size_t)it.ch * (size_t)k.n + (size_t)t0);
	if constexpr (ANY) {
		static_assert(P == 0 || SPEC == 2, "with passes the any-length front end keeps every pass scalar");
		static_assert(P > 0 || SPEC == 0 || SPEC == 2, "without passes the any-length front end is the generic boxcar one");
		const uint32_t *in_w = reinterpret_cast<const uint32_t *>(in);
		front_run_any<P, SPEC, false>(c, k, s, e, in_w, 0, (int)(start - t0), u, it.ch);
		front_run_any<P, SPEC, true>(c, k, s, e, in_w, (int)(start - t0), (int)(end - t0), u, it.ch);
	} else {
		const int t_last = (int)(end - t0) - 8;
		front_run<P, SPEC, false>(c, k, s, e, in, 0, (int)(start - t0), t_last, u, it.ch);
		front_run<P, SPEC, true>(c, k, s, e, in, (int)(start - t0), (int)(end - t0), t_last, u, it.ch);
	}
	if (SPEC == 2 && k.reduce_mode == 1) { chunk_enter<true>(c, k, e, it.ch, e.chunk_idx); }   // flush the last chunk's sums
	if (end == k.n && (SPEC != 2 || k.reduce_mode == 0)) {
		// this thread saw the end of the stream: its registers are the next call's carry, with pre = (0, 0) when the
		// call's last chunk emitted nothing (front_chunk_start)
		if constexpr (P == 0) { if (e.first_in_chunk) { s.pre_i = 0; s.pre_q = 0; } }
		if constexpr (ANY) { any_store<P, SPEC>(c, s, k.carry_out + (size_t)it.ch * k.state_words); }
		else { front_store<P, SPEC>(s, k.carry_out + (size_t)it.ch * k.state_words); }
	}
}

// ---- back end of one work item: `lanes` threads (whole warps), one contiguous run of OUTPUTS each.
// Pieces start on resampler group boundaries, so the only state a piece inherits is the de-emphasis
// average.
struct Piece { long long oa, ob; int ga, acc0, ph0; };

__device__ __forceinline__ Piece make_piece(const FmDev &c, const Item &it, const uint32_t *carry, long long o_first,
                                            long long o_end, int per, int q)
{
	Piece p;
	p.oa = o_first + (long long)q * per;
	p.ob = p.oa + per;
	if (p.oa > o_end) { p.oa = o_end; }
	if (p.ob > o_end) { p.ob = o_end; }
	p.ga = (int)(group_start(c, p.oa, it.phase0) - it.m_lo);        // buffer-relative PCM index
	const bool at_origin = (it.m_lo == 0 && p.ga == 0);               // stream start: the carry is the state
	p.acc0 = at_origin ? (int)carry[ST_LPR_ACC] : 0;
	p.ph0 = c.resample ? (int)(((long long)it.phase0 + (it.m_lo + p.ga) * (long long)c.slow - p.oa * (long long)c.fast)) : 0;
	return p;
}

template <int PAD>
__device__ __forceinline__ void run_piece(const FmDev &c, const int16_t *pcm_s, int16_t *__restrict__ out, const Piece &p,
                                          int &m_run, int &avg, AdcCtx *ax, bool store)
{
	m_run = p.ga;
	if (c.a_even) { back_outputs<true, PAD>(c, pcm_s, out, p.oa, p.ob, m_run, avg, p.acc0, p.ph0, ax, store); }
	else { back_outputs<false, PAD>(c, pcm_s, out, p.oa, p.ob, m_run, avg, p.acc0, p.ph0, ax, store); }
	if (ax) { adc_flush(*ax); }
}

// run_piece through windows (fm_back_kernel): every lane of the warp calls it, `run` says whether this lane has a piece to run
template <int WS>
__device__ __forceinline__ void run_piece_win(const FmDev &c, const LaneWin<WS> &w, int16_t *__restrict__ out, const Piece &p,
                                              int &m_run, int &avg, AdcCtx *ax, bool store, bool run)
{
	const bool lean = run && c.deemph && c.a_use_magic && c.resample && c.lpr_ok && p.ph0 < c.slow && ax == nullptr && store;
	int m = p.ga, a = avg;
	const int n_out = lean ? (int)(p.ob - p.oa) : 0;
	if (c.a_even) { win_outputs<true, WS>(c, w, out + p.oa, n_out, m, a, p.acc0, p.ph0); }
	else { win_outputs<false, WS>(c, w, out + p.oa, n_out, m, a, p.acc0, p.ph0); }
	if (lean) { m_run = m; avg = a; }
	else if (run) { run_piece<0>(c, w.g, out, p, m_run, avg, ax, store); }      // any other shape: straight from global memory
}

#define FM_BE_MAX_LANES 256
#define BAR_BE 1                 // named barrier of the back-end warps (id 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
// bar_sync that also returns whether `v` holds in every participating thread
__device__ __forceinline__ bool bar_sync_and(int id, int count, bool v)
{
	int r;
	asm volatile("{\n\t.reg .pred p, q;\n\tsetp.ne.s32 p, %1, 0;\n\tbar.red.and.pred q, %2, %3, p;\n\tselp.s32 %0, 1, 0, q;\n\t}"
	             : "=r"(r) : "r"((int)v), "r"(id), "r"(count) : "memory");
	return r != 0;
}

// WS > 0: the PCM is the call's global array and replay / outputs go through per-lane windows of WS samples in `win_rows`
// (fm_back_kernel; whole warps call, every lane takes part in the window fills)
template <int SPEC, int PAD, int WS = 0>
__device__ __forceinline__ void back_item(const FmDev &c, const FmCall &k, const Item &it, int work, int q, int lanes,
                                          const int16_t *pcm_s, int *s_avg, int *s_mrun, unsigned char *s_ok, int *s_start,
                                          uint32_t *win_rows = nullptr)
{
	constexpr bool WIN = WS > 0;
	LaneWin<WIN ? WS : 64> lw;
	lw.g = pcm_s; lw.rows = win_rows; lw.lane = q & 31;
	const uint32_t *carry = k.carry_in + (size_t)it.ch * k.state_words;
	int16_t *__restrict__ out = k.out + (size_t)it.ch * (size_t)k.out_stride;
	const bool last_cta = (it.b == k.n_cta - 1);
	const long long o_first = out_before(c, it.m_lo + it.m_own, it.phase0);
	const long long o_end = out_before(c, it.m_lo + it.m_hi, it.phase0);
	const int n_out = (int)(o_end - o_first);
	int per = (n_out + lanes - 1) / lanes;
	if (per < 1) { per = 1; }
	const int last_q = n_out > 0 ? (n_out - 1) / per : 0;
	const bool store = (SPEC != 2) || (k.reduce_mode == 0);
	PROF_CLK(tb0);
	AdcCtx axs;
	axs.adc = k.adc ? k.adc + (size_t)it.ch * k.n_chunks : nullptr;
	axs.sums = (k.reduce_mode == 2) ? k.sums + 2 * (size_t)it.ch * k.n_chunks : nullptr;
	axs.chunk = k.chunk; axs.box_n0 = it.box_n0; axs.n_chunks = k.n_chunks; axs.m_lo = it.m_lo;
	axs.cur = -1; axs.sub = 0; axs.acc = 0;
	AdcCtx *ax = (SPEC == 2 && c.adc_on && (axs.adc || axs.sums)) ? &axs : nullptr;
	// ---- pass 1: every lane brackets the state at its piece start; a closed bracket is an exact start
	const Piece p = make_piece(c, it, carry, o_first, o_end, per, q);
	const bool active = p.oa < p.ob;
	int kind = PK_EXACT;
	{
		int lo = -32768, hi = 32767, avg = 0, m_run = p.ga;
		const bool need = active || q == 0;
		int ws = p.ga - k.W_dec;
		if (ws < 0) { ws = 0; }
		ws &= ~3;           // quad-aligned start: a longer replay only tightens the bracket; every buffer entry from 0 on is exact PCM
		if (need && it.m_lo == 0 && ws == 0) { lo = hi = (int)carry[ST_AVG]; }
		bool replayed = false;
		if constexpr (WIN) {
			if (c.deemph && c.a_use_magic) {
				const int r_end = need ? p.ga : ws;
				if (c.a_even) { win_replay<true>(c, lw, ws, r_end, lo, hi); } else { win_replay<false>(c, lw, ws, r_end, lo, hi); }
				replayed = true;
			}
		}
		if (!replayed && need && c.deemph) {
			if (c.a_even) { back_replay<true, PAD>(c, pcm_s, ws, p.ga, lo, hi); } else { back_replay<false, PAD>(c, pcm_s, ws, p.ga, lo, hi); }
		}
		// Open bracket (quiet input: the rounding IIR has a dead zone).  Summarise what the piece does to
		// ANY state in [lo, hi] by running both ends through it: if they meet, the end state is exact
		// whatever the start was; if neither ever moves, no state in between moves either (the fixed
		// points of one step form an interval), so the piece passes its start state through.
		const bool open = need && c.deemph && lo != hi;
		const int ge = (open && active) ? (int)(group_start(c, p.ob, it.phase0) - it.m_lo) : p.ga;
		int moved = 0;
		bool probed = false;
		if constexpr (WIN) {
			if (c.deemph && c.a_use_magic) {       // whole warp: the lanes without an open bracket pass an empty range
				const int pe = open ? ge : p.ga;
				moved = c.a_even ? win_probe<true>(c, lw, p.ga, pe, lo, hi) : win_probe<false>(c, lw, p.ga, pe, lo, hi);
				probed = true;
			}
		}
		if (need) {
			avg = lo;
			if (open) {
				if (!probed) { moved = c.a_even ? back_probe<true, PAD>(c, pcm_s, p.ga, ge, lo, hi) : back_probe<false, PAD>(c, pcm_s, p.ga, ge, lo, hi); }
				kind = (lo == hi) ? PK_MERGED : (moved == 0 ? PK_IDENT : PK_OPEN);
				avg = lo; m_run = ge;
			}
		}
		if constexpr (WIN) { run_piece_win(c, lw, out, p, m_run, avg, ax, store, active && kind == PK_EXACT); }
		else { if (active && kind == PK_EXACT) { run_piece<PAD>(c, pcm_s, out, p, m_run, avg, ax, store); } }
		s_avg[q] = avg; s_mrun[q] = m_run; s_ok[q] = (unsigned char)kind;
	}
	const bool all_exact = bar_sync_and(BAR_BE, lanes, kind == PK_EXACT);
	PROF_ADD(PF_PASS1, tb0);
	PROF_CLK(tb1);
	// ---- chain (thread 0).  Across items the published word is a decoupled look-back: 1 = exact end state,
	// 2 = "this item passes its start state through" (the reader keeps walking back).  An item whose end state
	// is anchored by one of its own pieces publishes before it looks at anybody else.
	if (q == 0) {
		volatile int *pub = k.pub;
		auto serial_end = [&](int j, int start) -> int {          // PK_OPEN: the piece's de-emphasis from a known start
			const Piece pj = make_piece(c, it, carry, o_first, o_end, per, j);
			int l2 = start, h2 = start;
			if (pj.oa < pj.ob) {
				const int ge = (int)(group_start(c, pj.ob, it.phase0) - it.m_lo);
				if (c.a_even) { back_probe<true, PAD>(c, pcm_s, pj.ga, ge, l2, h2); } else { back_probe<false, PAD>(c, pcm_s, pj.ga, ge, l2, h2); }
			}
			return l2;
		};
		auto publish = [&](int flag, int value) {
			volatile int *mp = pub + 4 * (size_t)work;
			// flag 1: the value goes out before the flag (a release store; the reader fences after seeing the flag)
			if (flag == 1) { mp[1] = value; st_release_gpu(const_cast<int *>(mp), 1); }
			else { mp[0] = flag; }
		};
		// Every piece started exact (the common case with signal): the last piece is the anchor, nothing needs a start
		// state, and what the loops below would do is publish its end state.  A single thread walking the pieces
		// through dependent shared-memory loads is on the back end's critical path, so skip it.
		if (all_exact) {
			if (!last_cta) { publish(1, s_avg[last_q]); }
		} else {
			int anchor = -1, n_open = 0, published = 0, fixes = 0;
			for (int j = last_q; j >= 0; j--) {
				const int kj = s_ok[j];
				if (kj == PK_EXACT || kj == PK_MERGED) { anchor = j; break; }
				if (kj == PK_OPEN) { n_open++; }
			}
			if (!last_cta) {
				if (anchor >= 0) {
					int cur = s_avg[anchor];
					for (int j = anchor + 1; j <= last_q; j++) { if (s_ok[j] == PK_OPEN) { cur = serial_end(j, cur); } }
					publish(1, cur); published = 1;
				} else if (n_open == 0) { publish(2, 0); published = 2; }
			}
			// start states, left to right (piece 0: the closest older item of this channel that knows its end state)
			int cur = 0;
			for (int j = 0; j <= last_q; j++) {
				const int kj = s_ok[j];
				if (kj == PK_EXACT) { cur = s_avg[j]; continue; }
				int start;
				if (j == 0) {
					int w = work - 1;
					for (;;) {
						const int f = pub[4 * (size_t)w];
						if (f == 0) { __nanosleep(32); continue; }
						if (f == 1) { __threadfence(); start = pub[4 * (size_t)w + 1]; break; }
						w--;                                              // f == 2: that item passes its start through
					}
				} else { start = cur; }
				s_start[j] = start;
				if (kj == PK_MERGED) { cur = s_avg[j]; }
				else if (kj == PK_IDENT) { cur = start; }
				else { cur = serial_end(j, start); }
				s_avg[j] = cur;
				fixes++;
			}
			if (!last_cta && published != 1) { publish(1, s_avg[last_q]); }
			if (fixes) { atomicAdd(k.fix_count, fixes); }
		}
	}
	bar_sync(BAR_BE, lanes);
	PROF_ADD(PF_CHAIN, tb1);
	PROF_CLK(tb2);
	// ---- pass 2: the pieces that had no exact start in pass 1 now run from the state the chain gave them
	if constexpr (WIN) {
		const bool run = active && kind != PK_EXACT;
		int avg = run ? s_start[q] : 0, m_run = p.ga;
		run_piece_win(c, lw, out, p, m_run, avg, ax, store, run);
	} else {
		if (active && kind != PK_EXACT) {
			int avg = s_start[q], m_run = p.ga;
			run_piece<PAD>(c, pcm_s, out, p, m_run, avg, ax, store);
		}
	}
	if (q != 0) { return; }
	// end state of the item = state after its last piece
	int fin_avg = s_avg[last_q];
	const int fin_m = s_mrun[last_q];
	if (last_cta) {
		// tail of the stream: samples after the last emitted output stay in the accumulator
		int acc = (it.m_lo == 0 && fin_m == 0) ? (int)carry[ST_LPR_ACC] : 0;
		for (int m = fin_m; m < it.m_hi; m++) {
			int x = (int)pcm_s[pcm_phys<PAD>(m)];
			if (c.deemph) { fin_avg = deemph_step(c, fin_avg, x); x = wrap16(fin_avg); }
			if (ax) { x = adc_apply(c, *ax, m, x); }
			acc = add_w(acc, x);
		}
		if (ax) { adc_flush(*ax); }
		if (store) {
			uint32_t *co = k.carry_out + (size_t)it.ch * k.state_words;
			co[ST_AVG] = (uint32_t)fin_avg;
			co[ST_LPR_ACC] = (uint32_t)(c.resample ? acc : 0);
			co[ST_LPR_PHASE] = c.resample ? (uint32_t)(((long long)it.phase0 + (it.m_lo + it.m_hi) * (long long)c.slow) % (long long)c.fast) : 0u;
		}
	}
	PROF_ADD(PF_PASS2, tb2);
}

// Persistent CTA of T threads: all warps run the front end of a work item, then the first
// `be_lanes/32` warps run the back end out of the shared PCM buffer.  Work items are handed out by an
// atomic ticket, oldest first (the cross-item look-back only ever waits for an older ticket).
// The occupancy target is stated for 256 threads and scales with the width (same threads per SM).
// ANY: the any-length front end (front_run_any), for the calls fm_route sends there.
template <int P, int SPEC, int T, bool ANY = false>
__global__ void __launch_bounds__(T, (FM_MAX_THREADS / T) * (SPEC == 2 ? (P <= 3 ? 2 : 1) : (P <= 3 ? RXB_OCC : (P <= 6 ? 2 : 1)))) fm_fused_kernel(const FmDev c, const FmCall k)
{
	extern __shared__ __align__(16) int16_t pcm_s[];
	__shared__ int s_work;
	__shared__ int s_avg[FM_BE_MAX_LANES], s_mrun[FM_BE_MAX_LANES];
	__shared__ unsigned char s_ok[FM_BE_MAX_LANES];
	__shared__ int s_start[FM_BE_MAX_LANES];
	const int tid = threadIdx.x;
	const int total_work = k.n_ch * k.n_cta;
	const bool direct = Spec<SPEC>::direct(k);
	for (;;) {
		__syncthreads();
		if (tid == 0) { s_work = atomicAdd(k.ticket, 1); }
		__syncthreads();
		const int work = s_work;
		if (work >= total_work) { break; }
		const Item it = make_item(c, k, work);
		front_item<P, SPEC, ANY>(c, k, it, tid, pcm_s);
		if (direct || (SPEC == 2 && k.reduce_mode == 1)) {
			if (tid == 0 && it.b == k.n_cta - 1 && (SPEC != 2 || k.reduce_mode == 0)) {
				const uint32_t *carry = k.carry_in + (size_t)it.ch * k.state_words;
				uint32_t *co = k.carry_out + (size_t)it.ch * k.state_words;
				co[ST_AVG] = carry[ST_AVG]; co[ST_LPR_ACC] = carry[ST_LPR_ACC]; co[ST_LPR_PHASE] = carry[ST_LPR_PHASE];
			}
			continue;
		}
		__syncthreads();
		if (tid < k.be_lanes) { back_item<SPEC, PCM_PAD_SEG>(c, k, it, work, tid, k.be_lanes, pcm_s, s_avg, s_mrun, s_ok, s_start); }
	}
}

// ---- back end alone, over PCM in global memory (stream path: the front end of the whole call ran first).
// An item is a stretch of the call's PCM, a piece (one lane) a run of outputs in it.  With the PCM of the whole call
// at hand a piece can be as long as the launch has lanes to spare for, so the 16 a + 64 replay steps in front of every
// piece are paid once per few thousand samples, not once per shared-memory buffer share.  Same pieces, brackets,
// look-back and integers as back_item everywhere else.
// WS: samples per window (two windows per lane), T: lanes (pieces) per item.
#define BACK_T_MAX 128
template <int WS, int T>
__global__ void __launch_bounds__(T) fm_back_kernel(const FmDev c, const FmCall k)
{
	extern __shared__ __align__(16) uint32_t win_s[];      // [T / 32][2][32][WS / 2 + 2]
	__shared__ int s_work;
	__shared__ int s_avg[T], s_mrun[T], s_start[T];
	__shared__ unsigned char s_ok[T];
	const int tid = threadIdx.x;
	const int total_work = k.n_ch * k.n_cta;
	uint32_t *rows = win_s + (size_t)(tid >> 5) * 2 * LaneWin<WS>::BUF;
	for (;;) {
		__syncthreads();
		if (tid == 0) { s_work = atomicAdd(k.ticket, 1); }
		__syncthreads();
		const int work = s_work;
		if (work >= total_work) { break; }
		const Item it = make_item(c, k, work);
		back_item<1, 0, WS>(c, k, it, work, tid, T, k.pcm_g + (size_t)it.ch * (size_t)k.pcm_g_stride, s_avg, s_mrun, s_ok, s_start, rows);
	}
}
typedef void (*fm_kernel_fn)(const FmDev, const FmCall);
static fm_kernel_fn pick_back_kernel(int ws, int t)
{
	if (ws == 256) { return t == 32 ? fm_back_kernel<256, 32> : (t == 64 ? fm_back_kernel<256, 64> : fm_back_kernel<256, 128>); }
	return t == 32 ? fm_back_kernel<128, 32> : (t == 64 ? fm_back_kernel<128, 64> : fm_back_kernel<128, 128>);
}

#include "fm_rows.cuh"

// ---- split kernel: front end and back end of a CTA work on DIFFERENT items.
// In fm_fused_kernel every warp runs the front end of an item and then parks at a barrier while the first warps
// run the serial stages (22 % of the warp time on the wbfm shape, 62 % with de-emphasis at 2.4 Msps).  Here the
// CTA's last `be_lanes` threads do nothing but the back end: the front-end warps fill one of two PCM buffers and
// move on to the next item; the hand-off is a pair of mbarriers per buffer (full: front end -> back end, empty:
// back end -> front end), item tickets travel through shared memory.  An item still only ever waits for OLDER
// items (look-back in back_item), every CTA of the grid is resident, so the oldest unfinished item always advances.
// The front end is the row front end (fm_rows.cuh: a warp per stretch, input through `in_map`); FIR: with the droop FIR.
#define BAR_FE 2
#define SPLIT_BE_MAX 128
template <int P, int SPEC, bool FIR, int TMAX, int MINB>
__global__ void __launch_bounds__(TMAX, MINB) fm_split_kernel(const FmDev c, const FmCall k, const __grid_constant__ CUtensorMap in_map)
{
	// [2][pcm_cap] PCM buffers, then the row exchange areas, then (from the next 1024-byte boundary) the row input rings
	extern __shared__ __align__(16) int16_t pcm_s[];
	__shared__ __align__(8) uint64_t s_full[2], s_empty[2];
	__shared__ __align__(8) uint64_t s_ring_bar[(TMAX / 32) * ROWS_STAGES];
	__shared__ int s_ticket[2];
	__shared__ int s_avg[SPLIT_BE_MAX], s_mrun[SPLIT_BE_MAX], s_start[SPLIT_BE_MAX];
	__shared__ unsigned char s_ok[SPLIT_BE_MAX];
	const int tid = threadIdx.x;
	const int n_fe = k.fe_threads;
	int lane;
	asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));     // volatile: read once (the compiler would re-read the special register at every use)
	if (tid == 0) {
		mbar_init(&s_full[0], n_fe); mbar_init(&s_full[1], n_fe);
		mbar_init(&s_empty[0], k.be_lanes); mbar_init(&s_empty[1], k.be_lanes);
		for (int j = 0; j < k.fe_warps * ROWS_STAGES; j++) { mbar_init(&s_ring_bar[j], 1); }
	}
	__syncthreads();
	const int total_work = k.n_ch * k.n_cta;
#ifdef RXB_PROF
	{
		unsigned wid, smid;
		asm volatile("mov.u32 %0, %%warpid;" : "=r"(wid));
		asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
		PROF_SET(PF_WARPID, wid); PROF_SET(PF_SMID, smid);
	}
#endif
	PROF_CLK(t_start);
	if (tid < n_fe) {
		RowRing ring;
		uint8_t *end = reinterpret_cast<uint8_t *>(pcm_s + 2 * (size_t)k.pcm_cap) + (size_t)k.fe_warps * k.xs_words * sizeof(uint32_t);
		end += (0u - smem_u32(end)) & 1023u;
		ring.map = &in_map;
		ring.buf = end + (size_t)(tid >> 5) * ROWS_STAGES * ROW_BYTES;
		ring.bar = s_ring_bar + (tid >> 5) * ROWS_STAGES;
		ring.seq = 0;
		for (int i = 0;; i++) {
			const int b = i & 1;
			PROF_CLK(t0);
			if (i >= 2) { mbar_wait(&s_empty[b], (uint32_t)(((i >> 1) - 1) & 1)); }   // the back end is done with item i-2
			PROF_ADD(PF_EMPTY, t0);
			// one barrier per item lines the front-end warps up behind the ticket (measured: letting them run ahead on a
			// sequence number instead costs 9 % -- the early warps only reach the `empty` wait sooner and take issue
			// slots from the warp the back end is waiting for)
			if (tid == 0) { s_ticket[b] = atomicAdd(k.ticket, 1); }
			PROF_CLK(t1);
			bar_sync(BAR_FE, n_fe);
			PROF_ADD(PF_BAR_FE, t1);
			const int work = s_ticket[b];
			if (work >= total_work) { mbar_arrive(&s_full[b]); break; }                // the back end sees the sentinel
			const Item it = make_item(c, k, work);
			int16_t *buf = pcm_s + (size_t)b * k.pcm_cap;
			uint32_t *xs = reinterpret_cast<uint32_t *>(pcm_s + 2 * (size_t)k.pcm_cap) + (size_t)(tid >> 5) * k.xs_words;
			PROF_CLK(t2);
			front_rows<P, FIR>(c, k, it, tid >> 5, lane, buf, xs, ring);
			PROF_ADD(PF_FRONT, t2);
			PROF_CLK(t3);
			rows_publish<P>(k, it, work, buf, tid >> 5, lane);
			PROF_ADD(PF_PUBLISH, t3);
			PROF_INC(PF_ITEMS, 1);
			mbar_arrive(&s_full[b]);
		}
	} else {
		const int q = tid - n_fe;
		for (int i = 0;; i++) {
			const int b = i & 1;
			PROF_CLK(t0);
			mbar_wait(&s_full[b], (uint32_t)((i >> 1) & 1));
			PROF_ADD(PF_FULL, t0);
			const int work = s_ticket[b];
			if (work >= total_work) { break; }
			const Item it = make_item(c, k, work);
			PROF_CLK(t1);
			rows_collect<P>(k, it, work, pcm_s + (size_t)b * k.pcm_cap, q, k.be_lanes);
			PROF_ADD(PF_COLLECT, t1);
			back_item<SPEC, PCM_PAD_ROWS>(c, k, it, work, q, k.be_lanes, pcm_s + (size_t)b * k.pcm_cap, s_avg, s_mrun, s_ok, s_start);
			PROF_INC(PF_ITEMS, 1);
			mbar_arrive(&s_empty[b]);
		}
	}
	PROF_ADD(PF_TOTAL, t_start);
}

// ---- per-chunk reduction pre-passes: the scalar recurrences across chunks (one thread per channel)

// dc_block_raw_filter (src/rtl_fm.c:699-721): sums of the SCALED I and Q of every chunk
__global__ void __launch_bounds__(256) fm_rdc_sum_kernel(const int16_t *in, long long n, int chunk, int n_chunks, long long *sums)
{
	// grid: (slices, n_chunks, n_ch)
	const int ch = blockIdx.z, ci = blockIdx.y;
	const long long c0 = (long long)ci * chunk;
	long long c1 = c0 + chunk; if (c1 > n) { c1 = n; }
	const uint32_t *p = reinterpret_cast<const uint32_t *>(in) + (size_t)ch * (size_t)n;
	long long si = 0, sq = 0;
	for (long long t = c0 + (long long)blockIdx.x * blockDim.x + threadIdx.x; t < c1; t += (long long)gridDim.x * blockDim.x) {
		uint32_t w = __ldg(p + t);
		si += scale_cs16(lo16(w)); sq += scale_cs16(hi16(w));
	}
	for (int o = 16; o > 0; o >>= 1) { si += __shfl_down_sync(0xffffffffu, si, o); sq += __shfl_down_sync(0xffffffffu, sq, o); }
	if ((threadIdx.x & 31) == 0) {
		long long *sm = sums + 2 * ((size_t)ch * n_chunks + ci);
		atomicAdd(reinterpret_cast<unsigned long long *>(sm), (unsigned long long)si);
		atomicAdd(reinterpret_cast<unsigned long long *>(sm + 1), (unsigned long long)sq);
	}
}

__global__ void fm_rdc_recur_kernel(const long long *sums, const int *chunk_len, int n_chunks, int n_ch, int kconst,
                                    const uint32_t *carry_in, uint32_t *carry_out, int state_words, int *rdc)
{
	const int ch = blockIdx.x * blockDim.x + threadIdx.x;
	if (ch >= n_ch) { return; }
	int ai = (int)carry_in[(size_t)ch * state_words + ST_RDC_I], aq = (int)carry_in[(size_t)ch * state_words + ST_RDC_Q];
	for (int ci = 0; ci < n_chunks; ci++) {
		const long long *sm = sums + 2 * ((size_t)ch * n_chunks + ci);
		int mi = (int)(sm[0] / (long long)chunk_len[ci]);     // avgI = sumI / (len/2)
		int mq = (int)(sm[1] / (long long)chunk_len[ci]);
		ai = div_c(add_w(mi, mul_w(ai, kconst)), kconst + 1);
		aq = div_c(add_w(mq, mul_w(aq, kconst)), kconst + 1);
		rdc[2 * ((size_t)ch * n_chunks + ci)] = ai;
		rdc[2 * ((size_t)ch * n_chunks + ci) + 1] = aq;
	}
	carry_out[(size_t)ch * state_words + ST_RDC_I] = (uint32_t)ai;
	carry_out[(size_t)ch * state_words + ST_RDC_Q] = (uint32_t)aq;
}

// rms() + squelch decision (src/rtl_fm.c:739-757, :781-790); lp_len = the chunk's lowpassed int16 (fm_count_outputs)
__global__ void fm_squelch_kernel(const long long *sums, const int *lp_len, int n_chunks, int n_ch, int level,
                                  const uint32_t *carry_in, uint32_t *carry_out, int state_words, int *sqz, int *levels)
{
	const int ch = blockIdx.x * blockDim.x + threadIdx.x;
	if (ch >= n_ch) { return; }
	int hits = (int)carry_in[(size_t)ch * state_words + ST_SQ_HITS];
	for (int ci = 0; ci < n_chunks; ci++) {
		const long long *sm = sums + 2 * ((size_t)ch * n_chunks + ci);
		const long long t = sm[0], p = sm[1];
		const int len = lp_len[ci];
		// dc = (double)(t*step)/len; err = t*2*dc - dc*dc*len; (int)sqrt((p-err)/len) -- same order, no FMA
		const double dc = __ddiv_rn((double)t, (double)len);
		const double err = __dsub_rn(__dmul_rn((double)(t * 2), dc), __dmul_rn(__dmul_rn(dc, dc), (double)len));
		const int sr = (int)sqrt(__ddiv_rn(__dsub_rn((double)p, err), (double)len));
		if (levels) { levels[(size_t)ch * n_chunks + ci] = sr; }
		if (level) {                       // squelch off: squelch_hits is never touched (:781)
			const int z = sr < level ? 1 : 0;
			hits = z ? hits + 1 : 0;
			sqz[(size_t)ch * n_chunks + ci] = z;
		}
	}
	carry_out[(size_t)ch * state_words + ST_SQ_HITS] = (uint32_t)hits;
}

// dc_block_audio_filter recurrence (src/rtl_fm.c:691-696); pcm_len = result_len of the chunk before low_pass_real
__global__ void fm_adc_recur_kernel(const long long *sums, const int *pcm_len, int n_chunks, int n_ch, int kconst,
                                    const uint32_t *carry_in, uint32_t *carry_out, int state_words, int *adc)
{
	const int ch = blockIdx.x * blockDim.x + threadIdx.x;
	if (ch >= n_ch) { return; }
	int avg = (int)carry_in[(size_t)ch * state_words + ST_ADC];
	for (int ci = 0; ci < n_chunks; ci++) {
		int m = (int)(sums[2 * ((size_t)ch * n_chunks + ci)] / (long long)pcm_len[ci]);
		avg = div_c(add_w(m, mul_w(avg, kconst)), kconst + 1);
		adc[(size_t)ch * n_chunks + ci] = avg;
	}
	carry_out[(size_t)ch * state_words + ST_ADC] = (uint32_t)avg;
}

typedef void (*fm_kernel_fn)(const FmDev, const FmCall);

// CTA width.  Only the boxcar kernels (P = 0) exist in both widths; RXB200_FM_THREADS overrides the choice there (A/B
// runs).  On an H100 SXM (700 W) 256-thread CTAs are the faster boxcar shape at both ends of the decimation range:
// fm1 (D = 1) +9 %, fm5a (D = 100) +17 % over 128 (bench.py, two alternating runs each).
#define FM_WIDTH_DECIM 128
static int fm_cta_threads(int P)
{
	if (P > 0) { return FM_WIDTH_DECIM; }
	const char *e = getenv("RXB200_FM_THREADS");
	if (e && (atoi(e) == 128 || atoi(e) == 256)) { return atoi(e); }
	return 256;
}

template <int SPEC>
static fm_kernel_fn pick_kernel_p(int P, int threads)
{
#ifdef RXB_QUICK   // development builds: only the wbfm P = 3 kernel is instantiated (seconds instead of minutes)
	return (SPEC == 1 && P == 3) ? fm_fused_kernel<3, 1, FM_WIDTH_DECIM> : nullptr;
#else
	constexpr int PMAX = (SPEC == 1) ? 4 : 10;       // the wbfm specialisation is only built for the passes rx_fm can derive for it
	if (P > PMAX) { return nullptr; }
	switch (P) {
	case 0: return threads == 128 ? fm_fused_kernel<0, SPEC, 128> : fm_fused_kernel<0, SPEC, 256>;
	case 1: return fm_fused_kernel<1, SPEC, FM_WIDTH_DECIM>;
	case 2: return fm_fused_kernel<2, SPEC, FM_WIDTH_DECIM>;
	case 3: return fm_fused_kernel<3, SPEC, FM_WIDTH_DECIM>;
	case 4: return fm_fused_kernel<4, SPEC, FM_WIDTH_DECIM>;
	case 5: return fm_fused_kernel<(SPEC == 1 ? 4 : 5), SPEC, FM_WIDTH_DECIM>;
	case 6: return fm_fused_kernel<(SPEC == 1 ? 4 : 6), SPEC, FM_WIDTH_DECIM>;
	case 7: return fm_fused_kernel<(SPEC == 1 ? 4 : 7), SPEC, FM_WIDTH_DECIM>;
	case 8: return fm_fused_kernel<(SPEC == 1 ? 4 : 8), SPEC, FM_WIDTH_DECIM>;
	case 9: return fm_fused_kernel<(SPEC == 1 ? 4 : 9), SPEC, FM_WIDTH_DECIM>;
	case 10: return fm_fused_kernel<(SPEC == 1 ? 4 : 10), SPEC, FM_WIDTH_DECIM>;
	default: return nullptr;
	}
#endif
}

typedef void (*fm_split_fn)(const FmDev, const FmCall, const CUtensorMap);

// the split kernel with the row front end exists for the wbfm shape with 1..3 packed passes
// CTA shape of the split kernel (overridable for A/B builds, tools/build_variants.sh): front-end warps, back-end lanes,
// CTAs per SM the register budget is cut for
// Two CTAs of 7 + 1 warps, ROWS_STAGES = 2.  Every front-end warp's input ring takes 8 KB of shared memory.  While each
// warp replayed a whole row before its stretch, fewer front-end warps (longer stretches) won: fm2b (bench.py, 10 steps,
// two rounds alternating the builds, one H100 80GB HBM3 SXM at a 700 W power limit, SM clock 1980 MHz), Msamples/s:
//   4 + 1 warps x 3 CTAs 579 / 579    6 + 2 x 2 562 / 563    7 + 2 x 2 549 / 547    6 + 1 x 2 547 / 544
//   5 + 1 x 3 522 / 516               before the ring (8 + 2 x 2, register loads) 388 / 387
// and on a 400 W board of the same kind: 6 + 2 x 2 469 / 469, 16 + 4 x 1 416 / 414, 12 + 3 x 1 with 3 stages
// 412 / 410, before the ring 362 / 364.  Since a warp's start state costs 1/8 row and the margin rows are handed over,
// the sweep of the P = 3 kernel alone (same bench line, fm2b only, two rounds; H100 80GB HBM3 SXM, 400 W power limit,
// SM clock 1530-1680 MHz inside the kernel by clock64 against %globaltimer):
//   7 + 1 x 2 531 / 530    6 + 1 x 2 507 / 508    4 + 1 x 3 500 / 500    5 + 1 x 3 457 / 459
// and later (H100 80GB HBM3, 400 W, three rounds of 20 steps, even row split; DESIGN.md §4.1): 7 + 1 x 2 522-524,
// 6 + 2 x 2 501-504, 15 + 1 x 1 487-488.
// The P = 1 and P = 2 shapes share the choice and were not timed.
#ifndef ROWS_FE_WARPS
#define ROWS_FE_WARPS 7
#endif
#ifndef ROWS_BE_LANES
#define ROWS_BE_LANES 32
#endif
#ifndef ROWS_MINB
#define ROWS_MINB 2
#endif
#define ROWS_TMAX (ROWS_FE_WARPS * 32 + ROWS_BE_LANES)
static fm_split_fn pick_rows_kernel(int P, int fir_on)
{
#ifdef RXB_QUICK
	return (P == 3 && fir_on) ? fm_split_kernel<3, 1, true, ROWS_TMAX, ROWS_MINB> : nullptr;
#else
	switch (P) {
	case 1: return fir_on ? fm_split_kernel<1, 1, true, ROWS_TMAX, ROWS_MINB> : fm_split_kernel<1, 1, false, ROWS_TMAX, ROWS_MINB>;
	case 2: return fir_on ? fm_split_kernel<2, 1, true, ROWS_TMAX, ROWS_MINB> : fm_split_kernel<2, 1, false, ROWS_TMAX, ROWS_MINB>;
	case 3: return fir_on ? fm_split_kernel<3, 1, true, ROWS_TMAX, ROWS_MINB> : fm_split_kernel<3, 1, false, ROWS_TMAX, ROWS_MINB>;
	default: return nullptr;
	}
#endif
}

static int rows_xs_words(int P) { return P == 1 ? RowSmem<1>::WORDS : (P == 2 ? RowSmem<2>::WORDS : RowSmem<3>::WORDS); }

static fm_kernel_fn pick_kernel(int P, int spec, int threads)
{
#ifndef RXB_QUICK
	if (spec == 3) { return P == 0 ? (threads == 128 ? fm_fused_kernel<0, 3, 128> : fm_fused_kernel<0, 3, 256>) : nullptr; }
#endif
	if (spec == 4) { return P == 0 ? (threads == 128 ? fm_fused_kernel<0, 4, 128> : fm_fused_kernel<0, 4, 256>) : nullptr; }
	if (spec == 1 && P <= 4) { return pick_kernel_p<1>(P, threads); }
	if (spec == 2) { return pick_kernel_p<2>(P, threads); }
	return pick_kernel_p<0>(P, threads);
}

// The any-length kernel, in one CTA width.  Without passes the generic boxcar kernel (SPEC 0, or SPEC 2 with the per-chunk
// reduction stages): every other specialisation's shape is also a SPEC 0 shape.  With passes SPEC 2's all-scalar passes
// and stage bookkeeping serve every shape -- with no reduction stage on, that bookkeeping stays idle.
#define FM_ANY_THREADS 256
static fm_kernel_fn pick_any_kernel(int P, int spec)
{
#ifdef RXB_QUICK
	(void)P; (void)spec;
	return nullptr;
#else
	switch (P) {
	case 0: return spec == 2 ? fm_fused_kernel<0, 2, FM_ANY_THREADS, true> : fm_fused_kernel<0, 0, FM_ANY_THREADS, true>;
	case 1: return fm_fused_kernel<1, 2, FM_ANY_THREADS, true>;
	case 2: return fm_fused_kernel<2, 2, FM_ANY_THREADS, true>;
	case 3: return fm_fused_kernel<3, 2, FM_ANY_THREADS, true>;
	case 4: return fm_fused_kernel<4, 2, FM_ANY_THREADS, true>;
	case 5: return fm_fused_kernel<5, 2, FM_ANY_THREADS, true>;
	case 6: return fm_fused_kernel<6, 2, FM_ANY_THREADS, true>;
	case 7: return fm_fused_kernel<7, 2, FM_ANY_THREADS, true>;
	case 8: return fm_fused_kernel<8, 2, FM_ANY_THREADS, true>;
	case 9: return fm_fused_kernel<9, 2, FM_ANY_THREADS, true>;
	case 10: return fm_fused_kernel<10, 2, FM_ANY_THREADS, true>;
	default: return nullptr;
	}
#endif
}

// ---- the discriminators alone (rxb200_fm_disc_device): element i is the quad (ar, aj, br, bj) = x[n], x[n-1], whose
// conjugate product the chains form with the same wrapping expression; every form calls the very device function the
// kernels above inline, so a test can hold each one to the reference at operands a chain only rarely reaches
__global__ void fm_disc_kernel(int form, const int4 *__restrict__ quads, long long n, const int *__restrict__ lut,
                               int32_t *__restrict__ out)
{
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
		const int4 q = quads[i];
		const int ar = q.x, aj = q.y, br = q.z, bj = q.w;
		const int cr = add_w(mul_w(ar, br), mul_w(aj, bj));
		const int cj = sub_w(mul_w(aj, br), mul_w(ar, bj));
		int r = 0;
		switch (form) {
		case RXB200_DISC_STD: r = disc_std_f32(cr, cj); break;
		case RXB200_DISC_FAST: r = fast_atan2_i(cj, cr); break;
		case RXB200_DISC_LUT: r = disc_lut(lut, cr, cj); break;
		case RXB200_DISC_ALE: r = disc_ale(ar, aj, br, bj); break;
		case RXB200_DISC_ATAN2: r = disc_std(cr, cj); break;
		case RXB200_DISC_STD_FP64: r = disc_std_lean(cr, cj); break;
		case RXB200_DISC_ROWS: {
			uint32_t ab;
			row_angles<1, false, true>(&cr, &cj, 0, &ab);
			r = wrap16((int)ab);
			break;
		}
		case RXB200_DISC_STREAM: {      // front_block's undecimated loop, one sample
			const float fi = __int2float_rn(ar), fq = __int2float_rn(aj), fbr = __int2float_rn(br), fbj = __int2float_rn(bj);
			const float fcr = __fmaf_rn(fi, fbr, __fmul_rn(fq, fbj));
			const float fcj = __fmaf_rn(fq, fbr, -__fmul_rn(fi, fbj));
			r = wrap16(__float_as_int(__fadd_rn(fast_atan2_f32(fcj, fcr), 12582912.0f)));
			break;
		}
		case RXB200_DISC_AM: r = wrap16((int)sqrt((double)add_w(mul_w(ar, ar), mul_w(aj, aj)))); break;
		default: break;
		}
		out[i] = r;
	}
}

}  // namespace rxb

// ================================================================================ host side
using namespace rxb;

static const int k_droop9_host[11][10] = {
	// droop-compensation FIR rows (cic_9_tables, src/rtl_fm.c:287-300): {taps, c1..c9} x 2^15
	{0, 0, 0, 0, 0, 0, 0, 0, 0, 0},
	{9, -156,  -97, 2798, -15489, 61019, -15489, 2798,  -97, -156},
	{9, -128, -568, 5593, -24125, 74126, -24125, 5593, -568, -128},
	{9, -129, -639, 6187, -26281, 77511, -26281, 6187, -639, -129},
	{9, -122, -612, 6082, -26353, 77818, -26353, 6082, -612, -122},
	{9, -120, -602, 6015, -26269, 77757, -26269, 6015, -602, -120},
	{9, -120, -582, 5951, -26128, 77542, -26128, 5951, -582, -120},
	{9, -119, -580, 5931, -26094, 77505, -26094, 5931, -580, -119},
	{9, -119, -578, 5921, -26077, 77484, -26077, 5921, -578, -119},
	{9, -119, -577, 5917, -26067, 77473, -26067, 5917, -577, -119},
	{9, -199, -362, 5303, -25505, 77489, -25505, 5303, -362, -199},
};

// atan_lut_init (src/rtl_fm.c:515-526): host libm; rxb200_fm_create uploads it once per -A lut handle
static std::vector<int> atan_lut_host()
{
	std::vector<int> lut(131072);
	for (int i = 0; i < 131072; i++) { lut[i] = (int)(atan((double)i / (double)(1 << 8)) / 3.14159 * (double)(1 << 14)); }
	return lut;
}

struct rxb200_fm {
	rxb200_fm_params p{};
	int device = 0;
	int n_channels = 0;
	int n_sm = 0;
	FmDev dev{};
	int state_words = 0;
	cudaStream_t stream = nullptr;
	uint32_t *d_carry[2] = {nullptr, nullptr};
	int cur = 0;                   // which carry buffer holds the current state
	int *d_sync = nullptr; size_t sync_cap = 0;  // [0] ticket, [1] fix_count, [4..] pub[n_ch*n_cta][4]
	int16_t *d_margin = nullptr; size_t margin_cap = 0;   // row front end: margin hand-over slots (int16 entries)
	int *d_atan_lut = nullptr;
	int16_t *d_in = nullptr; size_t d_in_cap = 0;         // int16 elements
	int16_t *d_out = nullptr; size_t d_out_cap = 0;
	// host mirror of the closed-form counters
	int h_box_n = 0;               // demod.prev_index
	int h_lpr_phase = 0;           // demod.prev_lpr_index
	int tune_seg = 0, tune_warm = 0;
	rxb200_fm_stats stats{};
	fm_kernel_fn kern = nullptr;
	fm_split_fn kern_rows = nullptr;     // split kernel with the row front end (null: shape not covered)
	fm_kernel_fn kern_front = nullptr;   // stream path: front end alone (SPEC 4), PCM to global memory; fm_back_kernel follows
	int16_t *d_pcm = nullptr; size_t d_pcm_cap = 0;       // its PCM scratch, int16 elements
	fm_kernel_fn kern_any = nullptr;     // the any-length kernel (the calls fm_route sends there), FM_ANY_THREADS wide
	size_t stream_min = 0; int stream_piece = 0, stream_win = 0, stream_t = 0;
	int threads = 0;               // CTA width of kern
	int wide = 0;                  // all-scalar fifth_order passes (raw DC block on)
	int smem_optin = 0, smem_per_sm = 0, smem_reserved = 0;
	// per-chunk reduction stages, capacities in elements
	long long *d_sums = nullptr; int *d_rdc = nullptr, *d_sqz = nullptr, *d_adc = nullptr, *d_lens = nullptr, *d_levels = nullptr;
	size_t sums_cap = 0, rdc_cap = 0, sqz_cap = 0, adc_cap = 0, lens_cap = 0, levels_cap = 0; int level_chunks = 0;
	std::vector<int> h_lens;       // host side of d_lens
	cudaEvent_t ev0 = nullptr, ev1 = nullptr;
};

static int fm_validate(const rxb200_fm_params *p)
{
	if (p->mode < RXB200_MODE_FM || p->mode > RXB200_MODE_RAW) { set_error("mode %d", p->mode); return RXB200_EINVAL; }
	if (p->downsample_passes < 0 || p->downsample_passes > 10) { set_error("downsample_passes %d", p->downsample_passes); return RXB200_EINVAL; }
	if (p->downsample_passes == 0 && (p->downsample < 1 || p->downsample > 4096)) { set_error("downsample %d", p->downsample); return RXB200_EINVAL; }
	if (p->custom_atan < 0 || p->custom_atan > 3) { set_error("custom_atan %d", p->custom_atan); return RXB200_EINVAL; }
	if (p->deemph && p->deemph_a < 1) { set_error("deemph_a %d", p->deemph_a); return RXB200_EINVAL; }
	if (p->rate_out2 > 0 && (p->rate_out < p->rate_out2 || p->rate_out <= 0)) {
		set_error("low_pass_real needs rate_out >= rate_out2 > 0 (the reference divides by rate_out/rate_out2)");
		return RXB200_EINVAL;
	}
	if (p->post_downsample < 1 || p->post_downsample > 16) { set_error("post_downsample %d", p->post_downsample); return RXB200_EINVAL; }
	return RXB200_OK;
}

static void fm_fill_dev(rxb200_fm *h)
{
	const rxb200_fm_params &p = h->p;
	FmDev &d = h->dev;
	memset(&d, 0, sizeof d);
	d.mode = p.mode; d.P = p.downsample_passes; d.PL = fm_packed_levels(d.P, h->wide);
	d.squelch = p.squelch_level; d.rdc_on = p.dc_block_raw ? 1 : 0; d.rdc_k = p.rdc_block_const;
	d.levels = p.report_levels ? 1 : 0;
	d.adc_on = (p.dc_block_audio && p.mode != RXB200_MODE_RAW) ? 1 : 0; d.adc_k = p.adc_block_const;
	d.D = p.downsample_passes ? (1 << p.downsample_passes) : p.downsample;
	d.fir_on = (p.downsample_passes > 0 && p.comp_fir_size == 9) ? 1 : 0;
	d.atan_mode = p.custom_atan; d.out_scale = p.output_scale;
	d.post_ds = (p.mode != RXB200_MODE_RAW && p.post_downsample > 1) ? p.post_downsample : 1;   // raw_demod returns before -o (:809-811)
	d.deemph = (p.deemph && p.mode != RXB200_MODE_RAW) ? 1 : 0;
	d.a = p.deemph ? p.deemph_a : 1; d.a_half = d.a / 2; d.a_even = (d.a % 2 == 0) ? 1 : 0;
	// reciprocal for floor(n/a) over the numerator range used: verified exhaustively, else fall back to '/'
	d.a_use_magic = 0;
	if (d.a >= 1 && d.a < 16384) {
		unsigned magic = (unsigned)(0x100000000ULL / (unsigned)d.a) + 1u;
		int K = (65536 + 32768 + d.a) / d.a + 1;
		bool ok = true;
		unsigned nmax = (unsigned)(K * d.a + 65536 + 32768 + d.a);
		for (unsigned n = 0; n <= nmax && ok; n++) {
			if ((unsigned)(((unsigned long long)n * magic) >> 32) != n / (unsigned)d.a) { ok = false; }
		}
		if (ok) { d.a_use_magic = 1; d.a_magic = magic; d.a_K = K; }
	}
	d.resample = (p.rate_out2 > 0 && p.mode != RXB200_MODE_RAW) ? 1 : 0;
	d.fast = p.rate_out; d.slow = p.rate_out2; d.lpr_div = d.resample ? (p.rate_out / p.rate_out2) : 1;
	d.lpr_ok = 0;
	if (d.resample && d.lpr_div >= 2 && d.lpr_div <= 4096) {
		// signed division by a constant (Hacker's Delight 10-1), then checked for every sum a group can reach
		const unsigned two31 = 0x80000000u, ad = (unsigned)d.lpr_div;
		const unsigned anc = two31 - 1 - (two31 % ad);
		int pw = 31;
		unsigned q1 = two31 / anc, r1 = two31 - q1 * anc, q2 = two31 / ad, r2 = two31 - q2 * ad, delta;
		do {
			pw++;
			q1 = 2 * q1; r1 = 2 * r1; if (r1 >= anc) { q1++; r1 -= anc; }
			q2 = 2 * q2; r2 = 2 * r2; if (r2 >= ad) { q2++; r2 -= ad; }
			delta = ad - r2;
		} while (q1 < delta || (q1 == delta && r1 == 0));
		d.lpr_m = (int)(q2 + 1); d.lpr_s = pw - 32; d.lpr_add = d.lpr_m < 0 ? 1 : 0;
		bool ok = true;
		const long long lim = (long long)(d.lpr_div + 2) * 32768;
		for (long long n = -lim; n <= lim && ok; n++) {
			long long q = ((long long)(int)n * (long long)d.lpr_m) >> 32;
			if (d.lpr_add) { q += n; }
			q >>= d.lpr_s;
			q += (long long)((unsigned)(int)q >> 31);
			if ((int)q != (int)n / d.lpr_div) { ok = false; }
		}
		d.lpr_ok = ok ? 1 : 0;
	}
	d.offset_tuning = p.offset_tuning;
	for (int j = 0; j < 6; j++) { d.fir[j] = k_droop9_host[d.P][j]; }
	d.fir_bias = (int)((unsigned)FIR_B * (2u * (unsigned)(d.fir[1] + d.fir[2] + d.fir[3] + d.fir[4]) + (unsigned)d.fir[5]));
	d.atan_lut = h->d_atan_lut;
}

extern "C" int rxb200_fm_create(const rxb200_fm_params *params, int device, int n_channels, rxb200_fm **out)
{
	if (!params || !out || n_channels < 1) { set_error("null argument"); return RXB200_EINVAL; }
	*out = nullptr;
	int rc = fm_validate(params);
	if (rc != RXB200_OK) { return rc; }
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { set_error("no CUDA device: librxb200 has no CPU fallback"); return RXB200_ENODEV; }
	if (device < 0 || device >= ndev) { set_error("device %d out of range (%d)", device, ndev); return RXB200_ENODEV; }
	RXB_CUDA(cudaSetDevice(device));
	rxb200_fm *h = new (std::nothrow) rxb200_fm();
	if (!h) { return RXB200_ENOMEM; }
	h->p = *params; h->device = device; h->n_channels = n_channels;
	// any per-chunk reduction stage selects the SPEC 2 kernel (all-scalar passes + stage bookkeeping)
	h->wide = (params->dc_block_raw || params->squelch_level || params->dc_block_audio || params->post_downsample > 1 ||
	           params->report_levels) ? 1 : 0;
	h->state_words = fm_state_words(params->downsample_passes, h->wide);
	{
		// wbfm shape: FM + fast_atan2 + rotation, with a serial stage (de-emphasis or resampler)
		const bool serial = (params->deemph != 0) || (params->rate_out2 > 0);
		const bool plain = !params->squelch_level && !params->dc_block_audio && !params->dc_block_raw && params->post_downsample <= 1;
		int spec = h->wide ? 2 : ((params->mode == RXB200_MODE_FM && params->custom_atan == RXB200_ATAN_FAST &&
		                           !params->offset_tuning && serial && plain) ? 1 : 0);
		if (!h->wide && params->mode == RXB200_MODE_FM && params->custom_atan == RXB200_ATAN_LUT && !params->offset_tuning &&
		    !serial && plain && params->downsample_passes == 0) { spec = 3; }
		h->threads = fm_cta_threads(params->downsample_passes);
		h->kern = pick_kernel(params->downsample_passes, spec, h->threads);
		const int fir_on = (params->downsample_passes > 0 && params->comp_fir_size == 9) ? 1 : 0;
		h->kern_rows = spec == 1 ? pick_rows_kernel(params->downsample_passes, fir_on) : nullptr;
		h->kern_any = pick_any_kernel(params->downsample_passes, spec);
		// stream path (front kernel + back kernel): the wbfm shape without decimating passes, de-emphasis on
#ifndef RXB_QUICK
		h->kern_front = (spec == 1 && params->downsample_passes == 0 && params->deemph) ? pick_kernel(0, 4, h->threads) : nullptr;
#endif
		// stream path shape, read once (the tests reach shapes with them that a test-sized call would not pick)
		h->stream_min = getenv("RXB200_FM_STREAM_MIN") ? (size_t)atoll(getenv("RXB200_FM_STREAM_MIN")) : (size_t)-1;   // -1: derived per call
		h->stream_piece = getenv("RXB200_FM_STREAM_PIECE") ? atoi(getenv("RXB200_FM_STREAM_PIECE")) : 0;
		{
			const int ws = getenv("RXB200_FM_STREAM_WIN") ? atoi(getenv("RXB200_FM_STREAM_WIN")) : 0;
			h->stream_win = (ws == 128 || ws == 256) ? ws : 128;
			const int t = getenv("RXB200_FM_STREAM_T") ? atoi(getenv("RXB200_FM_STREAM_T")) : 0;
			h->stream_t = (t == 32 || t == 64 || t == 128) ? t : 32;
		}
	}
	if (!h->kern) { set_error("no kernel for downsample_passes %d in this build", params->downsample_passes); delete h; return RXB200_EUNSUPPORTED; }
	cudaDeviceProp prop;
	RXB_CUDA_OR(cudaGetDeviceProperties(&prop, device), rxb200_fm_destroy(h));
	h->n_sm = prop.multiProcessorCount;
	h->smem_optin = (int)prop.sharedMemPerBlockOptin;
	h->smem_per_sm = (int)prop.sharedMemPerMultiprocessor;
	h->smem_reserved = (int)prop.reservedSharedMemPerBlock;
	RXB_CUDA_OR(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking), rxb200_fm_destroy(h));
	RXB_CUDA_OR(cudaEventCreate(&h->ev0), rxb200_fm_destroy(h));
	RXB_CUDA_OR(cudaEventCreate(&h->ev1), rxb200_fm_destroy(h));
	size_t cbytes = (size_t)n_channels * h->state_words * sizeof(uint32_t);
	RXB_CUDA_OR(cudaMalloc(&h->d_carry[0], cbytes), rxb200_fm_destroy(h));
	RXB_CUDA_OR(cudaMalloc(&h->d_carry[1], cbytes), rxb200_fm_destroy(h));
	if (params->custom_atan == RXB200_ATAN_LUT && params->mode == RXB200_MODE_FM) {
		const std::vector<int> lut = atan_lut_host();
		RXB_CUDA_OR(cudaMalloc(&h->d_atan_lut, lut.size() * sizeof(int)), rxb200_fm_destroy(h));
		RXB_CUDA_OR(cudaMemcpy(h->d_atan_lut, lut.data(), lut.size() * sizeof(int), cudaMemcpyHostToDevice), rxb200_fm_destroy(h));
	}
	fm_fill_dev(h);
	rc = rxb200_fm_reset(h);
	if (rc != RXB200_OK) { rxb200_fm_destroy(h); return rc; }
	*out = h;
	return RXB200_OK;
}

extern "C" int rxb200_fm_reset(rxb200_fm *h)
{
	if (!h) { return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(h->device));
	size_t cbytes = (size_t)h->n_channels * h->state_words * sizeof(uint32_t);
	// demod_init (src/rtl_fm.c:1084-1115): everything zero, squelch_hits 11.  A zero sample in a
	// packed fifth_order history is its bias.
	std::vector<uint32_t> init((size_t)h->n_channels * h->state_words, 0u);
	const int PL = fm_packed_levels(h->p.downsample_passes, h->wide);
	for (int c = 0; c < h->n_channels; c++) {
		uint32_t *s = &init[(size_t)c * h->state_words];
		s[ST_SQ_HITS] = 11u;
		for (int l = 0; l < PL; l++) {
			for (int j = 0; j < 6; j++) { s[ST_HDR + 6 * l + j] = 0x00010001u * (128u << l); }
		}
	}
	RXB_CUDA(cudaMemcpyAsync(h->d_carry[0], init.data(), cbytes, cudaMemcpyHostToDevice, h->stream));
	RXB_CUDA(cudaMemcpyAsync(h->d_carry[1], init.data(), cbytes, cudaMemcpyHostToDevice, h->stream));
	RXB_CUDA(cudaStreamSynchronize(h->stream));
	h->cur = 0; h->h_box_n = 0; h->h_lpr_phase = 0;
	return RXB200_OK;
}

extern "C" void rxb200_fm_destroy(rxb200_fm *h)
{
	if (!h) { return; }
	cudaSetDevice(h->device);
	if (h->stream) { cudaStreamSynchronize(h->stream); }
	cudaFree(h->d_carry[0]); cudaFree(h->d_carry[1]); cudaFree(h->d_sync); cudaFree(h->d_margin);
	cudaFree(h->d_atan_lut); cudaFree(h->d_in); cudaFree(h->d_out); cudaFree(h->d_pcm);
	cudaFree(h->d_sums); cudaFree(h->d_rdc); cudaFree(h->d_sqz); cudaFree(h->d_adc); cudaFree(h->d_lens); cudaFree(h->d_levels);
	if (h->ev0) { cudaEventDestroy(h->ev0); }
	if (h->ev1) { cudaEventDestroy(h->ev1); }
	if (h->stream) { cudaStreamDestroy(h->stream); }
	delete h;
}

extern "C" int rxb200_fm_kernel_ms(rxb200_fm *h, float *ms)
{
	if (!h || !ms) { return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(h->device));
	RXB_CUDA(cudaEventSynchronize(h->ev1));
	RXB_CUDA(cudaEventElapsedTime(ms, h->ev0, h->ev1));
	return RXB200_OK;
}

// closed-form per-chunk result_len, and the pre-passes' chunk table when `lens` is given; advances the host mirrors when commit is set
static size_t fm_count_outputs(rxb200_fm *h, size_t n_int16, size_t chunk_int16, int *chunk_result_len, int *lens, bool commit)
{
	const rxb200_fm_params &p = h->p;
	const size_t n_chunks = (n_int16 + chunk_int16 - 1) / chunk_int16;
	long long box_n = h->h_box_n, phase = h->h_lpr_phase;
	size_t total = 0, pos = 0, c = 0;
	while (pos < n_int16) {
		size_t len16 = n_int16 - pos < chunk_int16 ? n_int16 - pos : chunk_int16;
		long long L = (long long)(len16 / 2), dec;
		if (p.downsample_passes) { dec = L >> p.downsample_passes; }
		else { dec = (box_n + L) / p.downsample; box_n = (box_n + L) % p.downsample; }
		// low_pass_simple needs a whole number of groups per chunk (otherwise the reference reads stale data)
		if (dec % h->dev.post_ds != 0) { return (size_t)-1; }
		// lowpassed int16 after the passes, what rms() divides by: odd when a read's L_P is (rxb200_fm_process_read).
		// For every chunk rxb200_fm_process takes lp == 2 * dec: without passes by construction, and with them every
		// chunk is a multiple of 2 << P int16, so len16 >> P == 2 * ((len16 / 2) >> P)
		const long long lp = p.downsample_passes ? (long long)(len16 >> p.downsample_passes) : 2 * dec;
		if (lens) {
			lens[c] = (int)L; lens[n_chunks + c] = (int)dec; lens[2 * n_chunks + c] = (int)(dec / h->dev.post_ds);
			lens[3 * n_chunks + c] = (int)lp;
		}
		dec /= h->dev.post_ds;
		long long res;
		if (p.mode == RXB200_MODE_RAW) { res = lp; }
		else if (p.rate_out2 > 0) {
			long long tot = phase + dec * (long long)p.rate_out2;
			res = tot / p.rate_out; phase = tot % p.rate_out;
		} else { res = dec; }
		if (chunk_result_len) { chunk_result_len[c] = (int)res; }
		total += (size_t)res; pos += len16; c++;
	}
	if (commit) { h->h_box_n = (int)box_n; h->h_lpr_phase = (int)phase; }
	return total;
}

extern "C" size_t rxb200_fm_max_output(const rxb200_fm *h, size_t n_int16, size_t chunk_int16)
{
	if (!h || chunk_int16 == 0) { return 0; }
	const rxb200_fm_params &p = h->p;
	size_t L = n_int16 / 2;
	size_t D = p.downsample_passes ? ((size_t)1 << p.downsample_passes) : (size_t)p.downsample;
	size_t dec = L / D + 2;
	if (p.mode == RXB200_MODE_RAW) { return 2 * dec; }
	if (p.rate_out2 > 0) { return (size_t)(((unsigned long long)dec * (unsigned)p.rate_out2) / (unsigned)p.rate_out) + 2; }
	return dec;
}

// Whether a call's shape is taken (else EUNSUPPORTED), and *any: whether it runs on the any-length kernel; every other
// call keeps the kernels and plans of the vector kernels' granule, 8 complex samples per block and 2^P per chunk
// (DESIGN.md section 6).  *any is set for a refused shape too: a device input's alignment follows from it and is
// reported first.  aligned32: the input is 32-byte aligned.
// - rxb200_fm_process without passes: any even chunk of at most 262144 int16 and any even call, on the any-length
//   kernel when the chunk or the call is not a multiple of 16 int16;
// - rxb200_fm_process with passes: chunk and call multiples of the granule;
// - rxb200_fm_process_read: one read of any even length from 2 << P int16 (fm_demod reads lowpassed[-1] below that; 2
//   without passes) to 262144, on whatever rxb200_fm_process(h, x, n, n) runs when that call takes it and the input is
//   32-byte aligned, else on the any-length kernel.
static int fm_route(const rxb200_fm *h, size_t n_int16, size_t chunk_int16, bool read, bool aligned32, bool *any)
{
	const int P = h->p.downsample_passes;
	const size_t p16 = (size_t)2 << P, g16 = p16 > 16 ? p16 : 16;   // 2^P complex; the granule
	if (read) {
		*any = !aligned32 || n_int16 % g16 != 0;
		const size_t lo = P ? p16 : 2;
		if (n_int16 < lo || n_int16 > 262144 || n_int16 % 2 != 0) {
			set_error("a read of n_int16=%zu must be even, at least %zu and at most 262144", n_int16, lo);
			return RXB200_EUNSUPPORTED;
		}
		return RXB200_OK;
	}
	*any = P == 0 && (chunk_int16 % 16 != 0 || n_int16 % 16 != 0);
	const size_t m16 = P ? g16 : 2;
	if (chunk_int16 == 0 || chunk_int16 > 262144 || chunk_int16 % m16 != 0) {
		set_error("chunk_int16=%zu must be a multiple of %zu and <= 262144", chunk_int16, m16);
		return RXB200_EUNSUPPORTED;
	}
	if (n_int16 % m16 != 0) {
		set_error("n_int16=%zu must be a multiple of %zu (last chunk included)", n_int16, m16);
		return RXB200_EUNSUPPORTED;
	}
	return RXB200_OK;
}

static long long round_up_ll(long long v, long long g) { return ((v + g - 1) / g) * g; }

// grows a device scratch buffer of the handle to at least `need` elements (the contents are not kept)
template <typename T>
static cudaError_t fm_reserve(T *&buf, size_t &cap, size_t need)
{
	if (need <= cap) { return cudaSuccess; }
	cudaFree(buf); buf = nullptr; cap = 0;
	const cudaError_t e = cudaMalloc(&buf, need * sizeof(T));
	if (e == cudaSuccess) { cap = need; }
	return e;
}

// Back-end replay in decimated samples: the de-emphasis bracket in front of a piece, 0 without de-emphasis.  The bracket
// closes in two phases: the gap contracts by (1 - 1/a) per step (to 1 within ~11 a steps from the full int16 range), then
// the two trajectories sit one apart until a sample lands on the one residue mod a that merges them -- a geometric wait
// with mean a.  16 a + 64 steps leave a fraction of a percent of the pieces open, each of which costs its item a probe and
// a second pass; with the stream path's long pieces four more a's of replay (e^-4: ~0.01 %) are cheaper than those
// stragglers.
static long long fm_replay(const rxb200_fm *h, bool stream)
{
	if (!h->dev.deemph) { return 0; }
	if (h->tune_warm > 0) { return h->tune_warm; }
	return (stream ? 20LL : 16LL) * h->p.deemph_a + 64;
}

// PCM a back end needs from before its stretch (decimated samples): the replay plus the resampler group in progress
static long long fm_margin(const rxb200_fm *h, long long W_dec)
{
	return W_dec + (h->dev.resample ? (h->p.rate_out / h->p.rate_out2 + 2) : 0) + 2;
}

// sets a kernel's dynamic shared memory to `smem` and returns how many of its CTAs fit an SM
template <typename K>
static cudaError_t fm_occupancy(K kern, int threads, size_t smem, int *per_sm)
{
	const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
	return e != cudaSuccess ? e : cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, kern, threads, smem);
}

struct FmGrid { int threads, per_sm; size_t smem; };   // CTA width, resident CTAs per SM, dynamic shared memory

// The row front end's view of the input: [n_ch * n / 32] lines of 32 words (128 bytes), one box = one row
// (32 lines), 128-byte swizzle (fm_rows.cuh).  cuTensorMapEncodeTiled comes from the driver at run time, so the
// library has no link-time libcuda dependency.
static int fm_rows_map(const int16_t *d_in, long long lines, CUtensorMap *map)
{
	static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
	if (!encode) {
		cudaDriverEntryPointQueryResult q;
		if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", reinterpret_cast<void **>(&encode), cudaEnableDefault, &q) != cudaSuccess ||
		    q != cudaDriverEntryPointSuccess || !encode) {
			encode = nullptr;
			set_error("the CUDA driver has no cuTensorMapEncodeTiled (the row front end needs it)");
			return RXB200_EUNSUPPORTED;
		}
	}
	// the box's line coordinate is a signed 32-bit int; the map's base address must be 16-byte aligned
	if ((reinterpret_cast<uintptr_t>(d_in) & 15u) != 0 || lines < 32 || lines > 0x7fffffffLL) {
		set_error("row front end: input at %p with %lld lines of 128 bytes cannot be mapped (16-byte alignment, at most 2^31 - 1 lines)",
		          (const void *)d_in, lines);
		return RXB200_EUNSUPPORTED;
	}
	const cuuint64_t dims[2] = {32, (cuuint64_t)lines};
	const cuuint64_t strides[1] = {128};
	const cuuint32_t box[2] = {32, 32}, estr[2] = {1, 1};
	const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, const_cast<int16_t *>(d_in), dims, strides, box, estr,
	                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
	                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d) for %lld lines at %p", (int)r, lines, (const void *)d_in); return RXB200_EUNSUPPORTED; }
	return RXB200_OK;
}

// ---- the split kernel with the row front end (fm_rows.cuh).  Geometry in ROWS of ROW_LEN input samples:
// an item owns `rows_own` rows; its PCM buffer also holds the `rows_margin` rows before them (the back end's replay
// window), which the previous items of the channel hand over through global memory; the two PCM buffers and the
// warps' exchange areas share the CTA's dynamic shared memory.  Returns FM_ROWS_NO_ROOM when the margin leaves no room
// for an item's own rows (a de-emphasis replay longer than the PCM buffers hold): fm_launch takes the fused kernel then.
#define FM_ROWS_NO_ROOM 1

static int fm_plan_rows(const rxb200_fm *h, long long n, FmCall *k, FmGrid *g)
{
	const int P = h->p.downsample_passes;
	const long long rows_total = n / ROW_LEN;
	const long long row_pcm = ROW_LEN >> P;                 // PCM samples per row
	const long long W_dec = fm_replay(h, false);
	const long long margin_dec = fm_margin(h, W_dec);
	const long long rows_margin = (margin_dec + row_pcm - 1) / row_pcm;
	const int fe_warps = ROWS_FE_WARPS, be_lanes = ROWS_BE_LANES;
	const int threads = fe_warps * 32 + be_lanes;
	const int xs_words = rows_xs_words(P);
	// exchange areas, then the input rings from the next 1024-byte boundary (up to 1008 bytes of padding)
	const size_t xs_bytes = (size_t)fe_warps * xs_words * sizeof(uint32_t) + 1008 + (size_t)fe_warps * ROWS_STAGES * ROW_BYTES;
	cudaFuncAttributes fa;
	RXB_CUDA(cudaFuncGetAttributes(&fa, h->kern_rows));
	// shared memory of one CTA when ROWS_MINB of them share an SM
	long long dyn_max = (long long)h->smem_per_sm / ROWS_MINB - (long long)h->smem_reserved - (long long)fa.sharedSizeBytes;
	if (dyn_max > h->smem_optin - (long long)fa.sharedSizeBytes) { dyn_max = h->smem_optin - (long long)fa.sharedSizeBytes; }
	auto cap_for = [&](long long rows_item) -> long long {
		long long e = rows_item * row_pcm + 8;              // one entry of slack is read past the last sample (back_outputs)
		e += PCM_PAD_ROWS * (e >> 7) + 16;
		return (e + 7) & ~7LL;                               // the second buffer and the exchange areas stay 16-byte aligned
	};
	long long rows_item = ((dyn_max - (long long)xs_bytes) / 2 / (long long)sizeof(int16_t)) / (row_pcm + (row_pcm * PCM_PAD_ROWS) / 128 + 1);
	while (rows_item > rows_margin + 1 && 2 * cap_for(rows_item) * (long long)sizeof(int16_t) + (long long)xs_bytes > dyn_max) { rows_item--; }
	long long rows_own = rows_item - rows_margin;
	if (rows_own < 1) { return FM_ROWS_NO_ROOM; }
	if (h->tune_seg > 0) {
		long long t = h->tune_seg / ROW_LEN;
		if (t < 1) { t = 1; }
		if (t < rows_own) { rows_own = t; }
	} else {
		// Items go out in waves of the resident CTAs.  A warp spends on an item its even share of the rows plus the 1/8
		// row of its start state (row_start_state), so the estimate for a length is waves x (ceil(rows / fe_warps) + 1/8):
		// a slightly shorter item that splits evenly or fills the last wave beats the longest one that fits.  Lengths
		// down to 60 % of that are tried; the longest of equal estimates wins.
		const long long slots = (long long)h->n_sm * ROWS_MINB;
		const long long longest = rows_own;
		double best = 0.0;
		for (long long t = longest; t >= 1 && t * 10 >= longest * 6; t--) {
			const long long items = (rows_total + t - 1) / t * h->n_channels;
			const double est = (double)((items + slots - 1) / slots) * ((double)((t + fe_warps - 1) / fe_warps) + 0.125);
			if (t == longest || est < best) { best = est; rows_own = t; }
		}
	}
	if (rows_own > rows_total) { rows_own = rows_total; }
	const long long pcm_cap = cap_for(rows_own + rows_margin);
	*g = {threads, 1, 2 * (size_t)pcm_cap * sizeof(int16_t) + xs_bytes};
	RXB_CUDA(fm_occupancy(h->kern_rows, threads, g->smem, &g->per_sm));
	if (g->per_sm < 1) { set_error("split kernel does not fit an SM (%zu bytes of shared memory, %d threads)", g->smem, threads); return RXB200_EUNSUPPORTED; }
	k->Sf = ROW_LEN; k->n_extra = (int)rows_margin; k->n_own = (int)rows_own; k->n_cta = (int)((rows_total + rows_own - 1) / rows_own);
	k->W_dec = (int)W_dec; k->pcm_cap = (int)pcm_cap; k->be_lanes = be_lanes; k->fe_warps = fe_warps; k->fe_threads = fe_warps * 32;
	k->xs_words = xs_words;
	return RXB200_OK;
}

static int fm_plan_segments(const rxb200_fm *h, fm_kernel_fn kern, int T, long long n, bool stream, FmCall *k, FmGrid *g)
{
	const FmDev &dv = h->dev;
	const int P = h->p.downsample_passes;
	const long long Dtot = dv.D;
	const long long G = (1LL << P) > 8 ? (1LL << P) : 8;
	// front-end replay: decimated samples until cascade (6) + droop FIR (9) + discriminator (1) are exact
	const long long dec_exact = (P ? (dv.fir_on ? 16 : 8) : 3) + (dv.post_ds > 1 ? dv.post_ds : 0);
	const long long halo = round_up_ll(dec_exact * Dtot, G);
	const long long Dpcm = Dtot * dv.post_ds;   // input samples per PCM sample
	// the stream path's front kernel and the shapes without a serial stage store the output from the front end
	const int direct_out = (stream || dv.mode == RXB200_MODE_RAW || (!dv.deemph && !dv.resample && !dv.adc_on)) ? 1 : 0;
	const long long W_dec = direct_out ? 0 : fm_replay(h, false);
	const long long margin_dec = direct_out ? 0 : fm_margin(h, W_dec);
	// segment per thread: ~128 decimated samples, at least 4 halos, capped so the PCM buffer stays small
	long long Sf = h->tune_seg;
	if (Sf <= 0) {
		Sf = 128 * Dpcm;
		if (Sf > 2048) { Sf = 2048; }
		if (Sf < 4 * halo) { Sf = 4 * halo; }
	}
	// Boxcar shapes: a segment that is a whole number of boxcar periods (and of 8-sample blocks) starts every thread
	// of a warp at the same decimation phase, so all lanes emit their decimated sample in the same iteration.  With
	// other lengths the lanes emit in different iterations and the discriminator / LUT / store code runs once per
	// phase instead of once per period (fm5a, D = 100: more than twice the kernel time off multiples of 200).
	// Gs = lcm(D, 8) when that still leaves a sensible segment.
	long long Gs = G;
	if (P == 0) {
		long long a = Dpcm, b = 8;
		while (b) { long long t = a % b; a = b; b = t; }
		const long long l = Dpcm / a * 8;
		if (l <= 1024) { Gs = l; }
	}
	if (h->tune_seg <= 0 && Sf >= 2 * Gs) { Sf = (Sf / Gs) * Gs; }
	Sf = round_up_ll(Sf, G);
	long long n_extra = 0, n_own = 0, stretch = 0, n_cta = 0, ppt = 0, pcm_cap = 0;
	size_t smem = 0;
	// the PCM buffer shares the opt-in limit with the kernel's static shared memory
	cudaFuncAttributes fa;
	RXB_CUDA(cudaFuncGetAttributes(&fa, kern));
	const long long smem_max = (long long)h->smem_optin - (long long)fa.sharedSizeBytes;
	auto geometry = [&](long long sf) -> bool {
		n_extra = direct_out ? 0 : (margin_dec * Dpcm + halo + sf - 1) / sf;
		ppt = sf / Dpcm + 2;
		pcm_cap = direct_out ? 8 : (long long)T * ppt + 64;
		pcm_cap += PCM_PAD_SEG * (pcm_cap >> 7) + 8;
		smem = (size_t)pcm_cap * sizeof(int16_t);
		if ((long long)smem > smem_max || n_extra > T / 2) { return false; }
		n_own = T - n_extra;
		stretch = n_own * sf;
		n_cta = (n + stretch - 1) / stretch;
		return true;
	};
	if (!geometry(Sf)) {
		// long warm-up wants longer segments, a big PCM buffer shorter ones: scan for something that fits
		bool ok = false;
		for (long long sf = round_up_ll(Sf * 8, G); sf >= G && !ok; sf = round_up_ll(sf / 2, G)) {
			if (geometry(sf)) { Sf = sf; ok = true; }
			if (sf == G) { break; }
		}
		if (!ok) {
			set_error("no segment length fits: warm-up %lld samples, D=%lld, shared memory %d", margin_dec * Dtot, Dtot, h->smem_optin);
			return RXB200_EUNSUPPORTED;
		}
	}
	int per_sm = 1;
	RXB_CUDA(fm_occupancy(kern, T, smem, &per_sm));
	if (per_sm < 1) { per_sm = 1; }
	if (h->tune_seg <= 0) {
		// tail balancing: work items are handed out to n_sm*per_sm resident CTAs; prefer a slightly shorter
		// segment when it turns a ragged last wave into full waves (cost = replay overhead x wave round-up)
		const double slots = (double)h->n_sm * per_sm;
		long long best = Sf;
		double best_cost = 1e30;
		for (long long sf = Sf; sf >= Gs && sf * 10 >= Sf * 6; sf -= Gs) {
			if (!geometry(sf)) { continue; }
			double waves = (double)(n_cta * h->n_channels) / slots;
			double cost = (waves <= 1.0 ? 1.0 : ceil(waves) / waves) * (1.0 + (double)halo / (double)sf) *
			              ((double)T / (double)n_own);
			if (cost < best_cost - 1e-9) { best_cost = cost; best = sf; }
		}
		Sf = best;
		geometry(Sf);
		// little work (a rank's share of the channels): with less than one wave of items the launch lasts one item,
		// so shorter segments -- more, shorter items -- finish sooner although each replays its halo:
		// time ~ rounds x (segment + halo)
		if ((double)(n_cta * h->n_channels) < slots) {
			long long pick = Sf;
			double pick_t = (double)(Sf + halo) * ((double)T / (double)n_own);
			for (long long sf = Sf - Gs; sf >= Gs && sf >= 2 * halo; sf -= Gs) {
				if (!geometry(sf)) { continue; }
				const double rounds = ceil((double)(n_cta * h->n_channels) / slots);
				const double t = rounds * (double)(sf + halo) * ((double)T / (double)n_own);
				if (t < pick_t - 1e-9) { pick_t = t; pick = sf; }
			}
			Sf = pick;
			geometry(Sf);
		}
	}
	// the grid is sized by the occupancy at the final segment length
	*g = {T, 1, smem};
	RXB_CUDA(fm_occupancy(kern, T, smem, &g->per_sm));
	if (g->per_sm < 1) { g->per_sm = 1; }
	// back-end width: enough lanes that a piece is about half a replay long (more lanes shorten the
	// phase in which the other warps idle, but every lane pays the full replay)
	const long long item_pcm = n_own * Sf / Dpcm;
	const long long want = W_dec > 0 ? (2 * item_pcm / W_dec + 31) / 32 * 32 : 128;
	int bl = (int)want;
	if (bl < 32) { bl = 32; }
	if (bl > T) { bl = T; }
	k->Sf = (int)Sf; k->halo = (int)halo; k->n_extra = (int)n_extra; k->n_own = (int)n_own; k->n_cta = (int)n_cta;
	k->W_dec = (int)W_dec; k->pcm_cap = (int)pcm_cap; k->direct_out = direct_out; k->be_lanes = bl;
	return RXB200_OK;
}

// stream path, back kernel: a CTA covers `span` input samples of a channel, a lane one piece of the PCM scratch
struct FmBackPlan { fm_kernel_fn kern; long long W_dec, span, n_cta, pstride; FmGrid g; };

static int fm_plan_back(const rxb200_fm *h, long long n, FmBackPlan *b)
{
	const long long Dtot = h->dev.D, Dpcm = Dtot * h->dev.post_ds;
	const long long m_total = (n + Dtot - 1) / Dtot + 1;
	const int back_t = h->stream_t, back_ws = h->stream_win;
	b->kern = pick_back_kernel(back_ws, back_t);
	b->W_dec = fm_replay(h, true);
	b->g = {back_t, 1, (size_t)(back_t / 32) * 2 * 32 * (back_ws / 2 + 2) * sizeof(uint32_t) + 64};   // + slack for win_outputs' read-ahead
	RXB_CUDA(fm_occupancy(b->kern, back_t, b->g.smem, &b->g.per_sm));
	if (b->g.per_sm < 1) { b->g.per_sm = 1; }
	const long long lanes_target = (long long)h->n_sm * b->g.per_sm * back_t;      // one piece per resident lane
	long long piece = h->stream_piece > 0 ? h->stream_piece : (m_total * h->n_channels + lanes_target - 1) / lanes_target;
	if (h->stream_piece <= 0 && piece < b->W_dec / 2) { piece = b->W_dec / 2; }
	if (piece < 64) { piece = 64; }
	if (piece * back_t * Dpcm > 0x40000000LL) { piece = 0x40000000LL / (back_t * Dpcm); }
	b->span = piece * back_t * Dpcm;
	b->n_cta = (n + b->span - 1) / b->span;
	b->pstride = (m_total + back_ws + 64 + 7) & ~7LL;      // a window may reach past the last sample
	return RXB200_OK;
}

// whether a call runs the per-chunk reduction stages (fm_prepasses) before its main pass
static bool fm_chunk_stages(const FmDev &dv) { return dv.rdc_on || dv.squelch || dv.adc_on || dv.levels; }

// the pre-passes' chunk table -- [0]: complex per chunk, [1]: decimated per chunk, [2]: PCM per chunk, [3]: lp_len --
// and the refusal of a call in which a chunk produces no decimated sample
static int fm_chunk_table(rxb200_fm *h, size_t n_int16, size_t chunk_int16, std::vector<int> &lens)
{
	const size_t n_chunks = (n_int16 + chunk_int16 - 1) / chunk_int16;
	lens.assign(n_chunks * 4, 0);
	fm_count_outputs(h, n_int16, chunk_int16, nullptr, lens.data(), false);   // -o was checked before the launch
	for (size_t ci = 0; ci < n_chunks; ci++) {
		if (lens[n_chunks + ci] < 1) { set_error("a chunk produces no decimated sample"); return RXB200_EUNSUPPORTED; }
	}
	return RXB200_OK;
}

// per-chunk scalars: sizes (closed form), accumulators, then one recurrence per stage in the reference's order: raw DC
// block -> squelch (sees the DC-blocked data, its sums from pass(1)) -> audio DC block (sums from pass(2))
template <typename Pass>
static int fm_prepasses(rxb200_fm *h, FmCall &k, size_t n_int16, size_t chunk_int16, Pass pass, int *launches)
{
	const FmDev &dv = h->dev;
	const int n_chunks = k.n_chunks;
	const size_t cells = (size_t)n_chunks * h->n_channels;
	RXB_CUDA(fm_reserve(h->d_sums, h->sums_cap, cells * 2));
	RXB_CUDA(fm_reserve(h->d_rdc, h->rdc_cap, cells * 2));
	RXB_CUDA(fm_reserve(h->d_sqz, h->sqz_cap, cells));
	RXB_CUDA(fm_reserve(h->d_adc, h->adc_cap, cells));
	RXB_CUDA(fm_reserve(h->d_levels, h->levels_cap, cells));
	RXB_CUDA(fm_reserve(h->d_lens, h->lens_cap, (size_t)n_chunks * 4));
	RXB_CUDA(cudaStreamSynchronize(h->stream));   // the previous call may still be reading the host vector
	if (const int rc = fm_chunk_table(h, n_int16, chunk_int16, h->h_lens); rc != RXB200_OK) { return rc; }
	RXB_CUDA(cudaMemcpyAsync(h->d_lens, h->h_lens.data(), h->h_lens.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
	const unsigned cb = (unsigned)((h->n_channels + 63) / 64);
	if (dv.rdc_on) {
		RXB_CUDA(cudaMemsetAsync(h->d_sums, 0, cells * 2 * sizeof(long long), h->stream));
		dim3 grid(8, (unsigned)n_chunks, (unsigned)h->n_channels);
		fm_rdc_sum_kernel<<<grid, 256, 0, h->stream>>>(k.in, k.n, k.chunk, n_chunks, h->d_sums);
		RXB_CUDA(cudaGetLastError());
		fm_rdc_recur_kernel<<<cb, 64, 0, h->stream>>>(h->d_sums, h->d_lens, n_chunks, h->n_channels, dv.rdc_k, k.carry_in, k.carry_out,
		                                               h->state_words, h->d_rdc);
		RXB_CUDA(cudaGetLastError());
		*launches += 2;
		k.rdc = h->d_rdc;
	}
	if (dv.squelch || dv.levels) {
		RXB_CUDA(cudaMemsetAsync(h->d_sums, 0, cells * 2 * sizeof(long long), h->stream));
		k.sums = h->d_sums;
		const int rc = pass(1);
		if (rc != RXB200_OK) { return rc; }
		fm_squelch_kernel<<<cb, 64, 0, h->stream>>>(h->d_sums, h->d_lens + 3 * (size_t)n_chunks, n_chunks, h->n_channels, dv.squelch,
		                                             k.carry_in, k.carry_out, h->state_words, h->d_sqz, dv.levels ? h->d_levels : nullptr);
		RXB_CUDA(cudaGetLastError());
		(*launches)++;
		k.sqz = dv.squelch ? h->d_sqz : nullptr;
		h->level_chunks = n_chunks;
	}
	if (dv.adc_on) {
		RXB_CUDA(cudaMemsetAsync(h->d_sums, 0, cells * 2 * sizeof(long long), h->stream));
		k.sums = h->d_sums;
		const int rc = pass(2);
		if (rc != RXB200_OK) { return rc; }
		fm_adc_recur_kernel<<<cb, 64, 0, h->stream>>>(h->d_sums, h->d_lens + 2 * (size_t)n_chunks, n_chunks, h->n_channels, dv.adc_k,
		                                               k.carry_in, k.carry_out, h->state_words, h->d_adc);
		RXB_CUDA(cudaGetLastError());
		(*launches)++;
		k.adc = h->d_adc;
	}
	k.sums = nullptr;
	return RXB200_OK;
}

// Plans and launches one call -- the split kernel where the shape allows it, else the fused kernel, or on the stream
// path the front and back kernels -- then advances the host mirrors of the closed-form counters.  any: the call runs on
// the any-length kernel (kern_any) instead.
static int fm_launch(rxb200_fm *h, const int16_t *d_in, size_t n_int16, size_t chunk_int16, int16_t *d_out, size_t out_stride,
                     bool any)
{
	const FmDev &dv = h->dev;
	const long long n = (long long)(n_int16 / 2);
	bool rows = !any && h->kern_rows && (chunk_int16 / 2) % ROW_LEN == 0 && n % ROW_LEN == 0 && n >= 16LL * ROW_LEN;
	// Stream path: the front end of the whole call stores its PCM to global memory (SPEC 4 through the direct-output
	// path), fm_back_kernel then runs the serial stages with pieces as long as the call allows.  In the fused kernel a
	// piece is a lane's share of one shared-memory buffer -- at the capture rate (fm2a) 870 samples behind a 2960-step
	// replay, and the item's front end recomputes the replay region too; here the replay is paid once per piece of
	// a few thousand samples and the front end computes nothing twice.  Worth it from a few dozen replays of PCM per call.
	const long long Dpcm = (long long)dv.D * dv.post_ds;
	const size_t stream_min = h->stream_min != (size_t)-1 ? h->stream_min : (size_t)(32 * fm_replay(h, false) * Dpcm / h->n_channels);
	// an any-length call runs on its own kernel, front and back end fused, whatever the shape would take otherwise
	const bool stream = !any && h->kern_front != nullptr && dv.deemph && (size_t)n >= stream_min;
	const fm_kernel_fn kern = any ? h->kern_any : (stream ? h->kern_front : h->kern);
	FmCall k = {};
	FmGrid g;
	CUtensorMap in_map;
	int rc = rows ? fm_plan_rows(h, n, &k, &g) : RXB200_OK;
	if (rc == FM_ROWS_NO_ROOM) { rows = false; k = {}; rc = RXB200_OK; }   // the same call on the fused kernel
	if (rc == RXB200_OK) { rc = rows ? fm_rows_map(d_in, (long long)h->n_channels * (n / 32), &in_map) : fm_plan_segments(h, kern, any ? FM_ANY_THREADS : h->threads, n, stream, &k, &g); }
	if (rc != RXB200_OK) { return rc; }
	const size_t total_work = (size_t)k.n_cta * h->n_channels;
	FmBackPlan b = {};
	if (stream) {
		rc = fm_plan_back(h, n, &b);
		if (rc != RXB200_OK) { return rc; }
		RXB_CUDA(fm_reserve(h->d_pcm, h->d_pcm_cap, (size_t)b.pstride * h->n_channels));
	}
	const size_t total_back = (size_t)b.n_cta * h->n_channels;
	const size_t need_sync = 4 + 4 * (total_work > total_back ? total_work : total_back);
	RXB_CUDA(fm_reserve(h->d_sync, h->sync_cap, need_sync));
	if (rows) {
		RXB_CUDA(fm_reserve(h->d_margin, h->margin_cap, total_work * (size_t)k.n_extra * (size_t)(ROW_LEN >> dv.P)));
		k.margin = h->d_margin;
	}
	// the fields every kernel of the call shares; the stream path's front kernel writes the PCM scratch
	k.in = d_in; k.out = stream ? h->d_pcm : d_out; k.out_stride = stream ? b.pstride : (long long)out_stride;
	k.n = n; k.chunk = (int)(chunk_int16 / 2); k.n_chunks = (int)((n + k.chunk - 1) / k.chunk); k.n_ch = h->n_channels;
	k.state_words = h->state_words; k.carry_in = h->d_carry[h->cur]; k.carry_out = h->d_carry[h->cur ^ 1];
	k.ticket = h->d_sync; k.fix_count = h->d_sync + 1; k.pub = h->d_sync + 4; k.one = 1;
	size_t blocks = (size_t)h->n_sm * g.per_sm;
	if (blocks > total_work) { blocks = total_work; }
	int launches = 0;
	// one pass over the call; ev0/ev1 bracket the main pass (reduce_mode 0, the time rxb200_fm_kernel_ms reports)
	auto pass = [&](int reduce_mode) -> int {
		k.reduce_mode = reduce_mode;
		RXB_CUDA(cudaMemsetAsync(h->d_sync, 0, need_sync * sizeof(int), h->stream));
		if (reduce_mode == 0) { RXB_CUDA(cudaEventRecord(h->ev0, h->stream)); }
		if (rows) { h->kern_rows<<<(unsigned)blocks, g.threads, g.smem, h->stream>>>(dv, k, in_map); }
		else { kern<<<(unsigned)blocks, g.threads, g.smem, h->stream>>>(dv, k); }
		RXB_CUDA(cudaGetLastError());
		if (reduce_mode == 0) { RXB_CUDA(cudaEventRecord(h->ev1, h->stream)); }
		launches++;
		return RXB200_OK;
	};
	if (fm_chunk_stages(dv)) {
		rc = fm_prepasses(h, k, n_int16, chunk_int16, pass, &launches);
		if (rc != RXB200_OK) { return rc; }
	}
	rc = pass(0);
	if (rc != RXB200_OK) { return rc; }
	if (stream) {
		FmCall kb = k;
		kb.out = d_out; kb.out_stride = (long long)out_stride; kb.direct_out = 0;
		kb.pcm_g = h->d_pcm; kb.pcm_g_stride = b.pstride;
		kb.n_extra = 0; kb.n_own = 1; kb.Sf = (int)b.span; kb.n_cta = (int)b.n_cta; kb.W_dec = (int)b.W_dec; kb.be_lanes = b.g.threads;
		kb.ticket = h->d_sync + 2;
		size_t blocks_b = (size_t)h->n_sm * b.g.per_sm;
		if (blocks_b > total_back) { blocks_b = total_back; }
		b.kern<<<(unsigned)blocks_b, b.g.threads, b.g.smem, h->stream>>>(dv, kb);
		RXB_CUDA(cudaGetLastError());
		RXB_CUDA(cudaEventRecord(h->ev1, h->stream));
		launches++;
	}
	h->cur ^= 1;
	h->stats.launches = launches; h->stats.segments = (int)(total_work * (rows ? k.fe_warps : g.threads));
	h->stats.segment_len = rows ? k.n_own * ROW_LEN : k.Sf; h->stats.warmup_len = (int)((stream ? b.W_dec : k.W_dec) * (long long)dv.D);
	h->stats.fixup_segments = -1; h->stats.kernel_kind = rows ? 1 : (stream ? 3 : 0);
	fm_count_outputs(h, n_int16, chunk_int16, nullptr, nullptr, true);
	return RXB200_OK;
}

// what every process call checks before it launches, in the order its refusals are reported, and the call's output
// count (*total PCM samples per channel) and route (*any, fm_route).  device: `in` is a device pointer, read at the
// alignment of the kernel the call runs on (the any-length kernel reads one complex sample at a time); a host input is
// staged into the handle's buffer, which is aligned.  read: a call of rxb200_fm_process_read (one chunk, its own shape rule)
static int fm_prologue(rxb200_fm *h, const void *in, const void *out, size_t n_int16, size_t chunk_int16, size_t pcm_stride,
                       int *chunk_result_len, size_t *total, size_t *n_pcm, bool read, bool device, bool *any)
{
	if (!h || !in || !out) { set_error("null argument"); return RXB200_EINVAL; }
	const uintptr_t addr = device ? (uintptr_t)in : 0u;
	const int rc = fm_route(h, n_int16, chunk_int16, read, (addr & 31u) == 0, any);
	const uintptr_t align = *any ? 4u : 32u;
	if ((addr & (align - 1u)) != 0) { set_error("d_cs16 must be %d-byte aligned", (int)align); return RXB200_EINVAL; }
	if (rc != RXB200_OK) { return rc; }
	RXB_CUDA(cudaSetDevice(h->device));
	if (n_int16 == 0) { h->level_chunks = 0; if (n_pcm) { *n_pcm = 0; } }
	*total = fm_count_outputs(h, n_int16, chunk_int16, chunk_result_len, nullptr, false);
	if (*total == (size_t)-1) { set_error("-o %d needs every chunk to decimate to a multiple of it", h->dev.post_ds); return RXB200_EUNSUPPORTED; }
	if (*total > pcm_stride) { set_error("pcm_stride %zu < %zu outputs", pcm_stride, *total); return RXB200_ECAPACITY; }
	if (*any && !h->kern_any) { set_error("no any-length kernel for downsample_passes %d in this build", h->dev.P); return RXB200_EUNSUPPORTED; }
	return RXB200_OK;
}

int rxb::fm_check_host_call(rxb200_fm *h, const int16_t *cs16, size_t n_int16, size_t chunk_int16, int16_t *pcm,
                            size_t pcm_stride, int *chunk_result_len, size_t *n_pcm, bool read, size_t *total)
{
	bool any = false;
	const int rc = fm_prologue(h, cs16, pcm, n_int16, chunk_int16, pcm_stride, chunk_result_len, total, n_pcm, read, false, &any);
	if (rc != RXB200_OK || n_int16 == 0 || !fm_chunk_stages(h->dev)) { return rc; }
	std::vector<int> lens;
	return fm_chunk_table(h, n_int16, chunk_int16, lens);
}

static int fm_process_device(rxb200_fm *h, const int16_t *d_cs16, size_t n_int16, size_t chunk_int16, int16_t *d_pcm,
                             size_t pcm_stride, size_t *n_pcm, int sync, bool read)
{
	size_t total = 0;
	bool any = false;
	int rc = fm_prologue(h, d_cs16, d_pcm, n_int16, chunk_int16, pcm_stride, nullptr, &total, n_pcm, read, true, &any);
	if (rc != RXB200_OK || n_int16 == 0) { return rc; }
	rc = fm_launch(h, d_cs16, n_int16, chunk_int16, d_pcm, pcm_stride, any);
	if (rc != RXB200_OK) { return rc; }
	if (n_pcm) { *n_pcm = total; }
	if (sync) {
		RXB_CUDA(cudaStreamSynchronize(h->stream));
		RXB_CUDA(cudaMemcpy(&h->stats.fixup_segments, h->d_sync + 1, sizeof(int), cudaMemcpyDeviceToHost));
	}
	return RXB200_OK;
}

static int fm_process_host(rxb200_fm *h, const int16_t *cs16, size_t n_int16, size_t chunk_int16, int16_t *pcm,
                           size_t pcm_stride, size_t *n_pcm, int *chunk_result_len, bool read)
{
	size_t total = 0;
	bool any = false;
	int rc = fm_prologue(h, cs16, pcm, n_int16, chunk_int16, pcm_stride, chunk_result_len, &total, n_pcm, read, false, &any);
	if (rc != RXB200_OK || n_int16 == 0) { return rc; }
	const size_t in_elems = n_int16 * (size_t)h->n_channels;
	const size_t out_elems = (total + 8) * (size_t)h->n_channels;
	RXB_CUDA(fm_reserve(h->d_in, h->d_in_cap, in_elems));
	RXB_CUDA(fm_reserve(h->d_out, h->d_out_cap, out_elems));
	RXB_CUDA(cudaMemcpyAsync(h->d_in, cs16, in_elems * sizeof(int16_t), cudaMemcpyHostToDevice, h->stream));
	rc = fm_launch(h, h->d_in, n_int16, chunk_int16, h->d_out, total + 8, any);
	if (rc != RXB200_OK) { return rc; }
	if (pcm_stride == total + 8 || h->n_channels == 1) {
		RXB_CUDA(cudaMemcpyAsync(pcm, h->d_out, (h->n_channels == 1 ? total : out_elems) * sizeof(int16_t),
		                         cudaMemcpyDeviceToHost, h->stream));
	} else {
		RXB_CUDA(cudaMemcpy2DAsync(pcm, pcm_stride * sizeof(int16_t), h->d_out, (total + 8) * sizeof(int16_t),
		                           total * sizeof(int16_t), (size_t)h->n_channels, cudaMemcpyDeviceToHost, h->stream));
	}
	RXB_CUDA(cudaMemcpyAsync(&h->stats.fixup_segments, h->d_sync + 1, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
	RXB_CUDA(cudaStreamSynchronize(h->stream));
	if (n_pcm) { *n_pcm = total; }
	return RXB200_OK;
}

extern "C" int rxb200_fm_process_device(rxb200_fm *h, const int16_t *d_cs16, size_t n_int16, size_t chunk_int16,
                                        int16_t *d_pcm, size_t pcm_stride, size_t *n_pcm, int sync)
{
	return fm_process_device(h, d_cs16, n_int16, chunk_int16, d_pcm, pcm_stride, n_pcm, sync, false);
}

extern "C" int rxb200_fm_process(rxb200_fm *h, const int16_t *cs16, size_t n_int16, size_t chunk_int16,
                                 int16_t *pcm, size_t pcm_stride, size_t *n_pcm, int *chunk_result_len)
{
	return fm_process_host(h, cs16, n_int16, chunk_int16, pcm, pcm_stride, n_pcm, chunk_result_len, false);
}

extern "C" int rxb200_fm_process_read(rxb200_fm *h, const int16_t *cs16, size_t n_int16, int16_t *pcm, size_t pcm_stride,
                                      size_t *n_pcm)
{
	return fm_process_host(h, cs16, n_int16, n_int16, pcm, pcm_stride, n_pcm, nullptr, true);
}

extern "C" int rxb200_fm_process_read_device(rxb200_fm *h, const int16_t *d_cs16, size_t n_int16, int16_t *d_pcm,
                                             size_t pcm_stride, size_t *n_pcm, int sync)
{
	return fm_process_device(h, d_cs16, n_int16, n_int16, d_pcm, pcm_stride, n_pcm, sync, true);
}

extern "C" int rxb200_fm_squelch_hits(rxb200_fm *h, int *hits)
{
	if (!h || !hits) { return RXB200_EINVAL; }
	RXB_CUDA(cudaSetDevice(h->device));
	std::vector<uint32_t> st((size_t)h->n_channels * h->state_words);
	RXB_CUDA(cudaMemcpyAsync(st.data(), h->d_carry[h->cur], st.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
	RXB_CUDA(cudaStreamSynchronize(h->stream));
	for (int c = 0; c < h->n_channels; c++) { hits[c] = (int)st[(size_t)c * h->state_words + ST_SQ_HITS]; }
	return RXB200_OK;
}

extern "C" int rxb200_fm_levels(rxb200_fm *h, int *levels, size_t cap, size_t *n_chunks)
{
	if (!h || !levels || !n_chunks) { set_error("null argument"); return RXB200_EINVAL; }
	if (!h->p.report_levels) { set_error("handle was created without report_levels"); return RXB200_EINVAL; }
	const size_t cells = (size_t)h->level_chunks * h->n_channels;
	*n_chunks = (size_t)h->level_chunks;
	if (cap < cells) { set_error("levels capacity %zu < %zu", cap, cells); return RXB200_ECAPACITY; }
	if (!cells) { return RXB200_OK; }
	RXB_CUDA(cudaSetDevice(h->device));
	RXB_CUDA(cudaMemcpyAsync(levels, h->d_levels, cells * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
	RXB_CUDA(cudaStreamSynchronize(h->stream));
	return RXB200_OK;
}

extern "C" void *rxb200_fm_stream(rxb200_fm *h) { return h ? (void *)h->stream : nullptr; }

extern "C" int rxb200_fm_last_stats(rxb200_fm *h, rxb200_fm_stats *out)
{
	if (!h || !out) { return RXB200_EINVAL; }
	if (h->stats.fixup_segments < 0 && h->d_sync) {
		RXB_CUDA(cudaSetDevice(h->device));
		RXB_CUDA(cudaStreamSynchronize(h->stream));
		RXB_CUDA(cudaMemcpy(&h->stats.fixup_segments, h->d_sync + 1, sizeof(int), cudaMemcpyDeviceToHost));
	}
	*out = h->stats;
	return RXB200_OK;
}

extern "C" int rxb200_fm_tune(rxb200_fm *h, int segment_len, int deemph_warmup)
{
	if (!h || segment_len < 0 || deemph_warmup < 0) { return RXB200_EINVAL; }
	h->tune_seg = segment_len; h->tune_warm = deemph_warmup;
	return RXB200_OK;
}

extern "C" int rxb200_fm_disc_device(int form, const int32_t *d_quads, size_t n, int32_t *d_out, void *stream)
{
	if (form < RXB200_DISC_STD || form > RXB200_DISC_AM) { set_error("unknown discriminator form %d", form); return RXB200_EINVAL; }
	if (!d_quads || !d_out) { set_error("bad disc request (null pointer)"); return RXB200_EINVAL; }
	if ((uintptr_t)d_quads & 15u) { set_error("quads must be 16-byte aligned"); return RXB200_EINVAL; }
	if (n == 0) { return RXB200_OK; }
	const cudaStream_t st = (cudaStream_t)stream;
	int *d_lut = nullptr;
	if (form == RXB200_DISC_LUT) {
		const std::vector<int> lut = atan_lut_host();
		RXB_CUDA(cudaMallocAsync((void **)&d_lut, lut.size() * sizeof(int), st));
		// from pageable memory: the copy has read its source when it returns
		if (cudaMemcpyAsync(d_lut, lut.data(), lut.size() * sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess) {
			set_error("lut upload failed: %s", cudaGetErrorString(cudaGetLastError()));
			cudaFreeAsync(d_lut, st);
			return RXB200_ECUDA;
		}
	}
	const long long want = ((long long)n + 255) / 256, blocks = want < 8192 ? want : 8192;
	fm_disc_kernel<<<(unsigned)blocks, 256, 0, st>>>(form, reinterpret_cast<const int4 *>(d_quads), (long long)n, d_lut, d_out);
	const cudaError_t e = cudaGetLastError();
	if (d_lut) { cudaFreeAsync(d_lut, st); }
	if (e != cudaSuccess) { set_error("fm_disc_kernel launch failed: %s", cudaGetErrorString(e)); return RXB200_ECUDA; }
	return RXB200_OK;
}

#ifdef RXB_PROF
// scratch builds: copy the per-warp phase sums out (clear = 1: and zero them), [PROF_CTAS][32][PROF_SLOTS] words
extern "C" int rxb200_fm_prof_read(unsigned long long *dst, size_t n, int clear)
{
	const size_t all = (size_t)PROF_CTAS * 32 * PROF_SLOTS;
	if (dst && n) { RXB_CUDA(cudaMemcpyFromSymbol(dst, rxb_prof, (n < all ? n : all) * sizeof(unsigned long long))); }
	if (clear) {
		void *p = nullptr;
		RXB_CUDA(cudaGetSymbolAddress(&p, rxb_prof));
		RXB_CUDA(cudaMemset(p, 0, all * sizeof(unsigned long long)));
	}
	return RXB200_OK;
}
#endif
