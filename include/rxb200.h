/* rxb200.h — C-ABI of librxb200.so, the H100 (sm_90a) replacement for the rx_tools DSP hot path.
 *
 * The reference (rxseger/rx_tools @ 811b21c) has no plugin/FFI interface; the boundary is plain C
 * functions over file-scope globals (SURVEY.md §8b).  Each entry point below names the reference
 * function(s) it replaces.  All entry points are extern "C", take plain pointers and sizes, return
 * 0 or a negative RXB200_E* code, never call exit(), and keep no global state: one handle is used
 * by one thread at a time, different handles may be used concurrently.  There is NO CPU fallback:
 * without a CUDA device every create call fails with RXB200_ENODEV.
 *
 * INTEGRATION.md shows the two call sites a maintainer re-points in rtl_fm.c / rtl_power.c.
 */
#ifndef RXB200_H
#define RXB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RXB200_ABI_VERSION 3

/* error codes */
#define RXB200_OK            0
#define RXB200_EINVAL       (-1)   /* bad argument / parameter combination            */
#define RXB200_ENODEV       (-2)   /* no CUDA device / device index out of range      */
#define RXB200_ECUDA        (-3)   /* a CUDA runtime call failed (see rxb200_last_error) */
#define RXB200_ENOMEM       (-4)   /* host or device allocation failed                */
#define RXB200_EUNSUPPORTED (-5)   /* legal for the reference but not implemented here (documented in DESIGN.md) */
#define RXB200_ECAPACITY    (-6)   /* caller's output buffer too small                */

/* Human-readable text for the last failure on the calling thread. */
const char *rxb200_last_error(void);
int rxb200_abi_version(void);
/* Number of visible CUDA devices (0 when none: every create call will then fail). */
int rxb200_device_count(void);

/* ======================================================================== rx_fm
 * Replaces, per chunk, the DSP body of rtlsdr_callback() (src/rtl_fm.c:844-857: CS16 -> 8-bit-range
 * scale, dc_block_raw_filter, rotate16_90) followed by full_demod() (src/rtl_fm.c:759-824:
 * low_pass | fifth_order x P + generic_fir, rms squelch, fm/am/usb/lsb/raw demod, low_pass_simple,
 * deemph_filter, dc_block_audio_filter, low_pass_real) with every carry of struct demod_state
 * (src/rtl_fm.c:124-159) held device-side in the handle.
 */

/* demod modes: demod.mode_demod, src/rtl_fm.c:1320-1342 */
#define RXB200_MODE_FM  0   /* fm_demod   :584 */
#define RXB200_MODE_AM  1   /* am_demod   :617 */
#define RXB200_MODE_USB 2   /* usb_demod  :634 */
#define RXB200_MODE_LSB 3   /* lsb_demod  :646 */
#define RXB200_MODE_RAW 4   /* raw_demod  :658 */

/* discriminators: demod.custom_atan, src/rtl_fm.c:592-609 */
#define RXB200_ATAN_STD  0  /* polar_discriminant :476 (fp64 atan2)  */
#define RXB200_ATAN_FAST 1  /* polar_disc_fast    :508 (integer)     */
#define RXB200_ATAN_LUT  2  /* polar_disc_lut     :528 (integer LUT) */
#define RXB200_ATAN_ALE  3  /* esbensen           :566 (integer)     */
/* One deviation from the reference in -A lut: where (cj << 8) wraps to INT_MIN with |cr| = 1 (cj = 2^23 mod 2^24,
 * reachable once decimated samples pass 2048), polar_disc_lut indexes its table at INT_MIN (cr = 1) or divides INT_MIN
 * by -1 (cr = -1) and the reference process crashes; the library returns cj > 0 ? 8192 : -8192 there, the value its
 * linear-range branch gives every other |x| it cannot look up (DESIGN.md section 6). */

/* The configuration fields of struct demod_state / dongle_state the DSP reads, with the reference's
 * names (src/rtl_fm.c:124-159).  Fill them as main()/optimal_settings() would, or let
 * rxb200_fm_derive() do it from the CLI-level values. */
typedef struct rxb200_fm_params {
	int mode;               /* RXB200_MODE_*                                              */
	int downsample;         /* boxcar length, 1..256 (used when downsample_passes == 0)   */
	int downsample_passes;  /* number of fifth_order passes P, 0..10                      */
	int comp_fir_size;      /* 9 enables generic_fir droop compensation (with P >= 1)     */
	int custom_atan;        /* RXB200_ATAN_*                                              */
	int output_scale;       /* am/usb/lsb gain                                            */
	int post_downsample;    /* -o; 1 = off                                                */
	int deemph;             /* 0/1                                                        */
	int deemph_a;           /* round(1/(1-exp(-1/(rate_out*tc))))                         */
	int rate_out;           /* low_pass_real "fast" rate                                  */
	int rate_out2;          /* low_pass_real "slow" rate, <= 0 disables                   */
	int squelch_level;      /* 0 = off                                                    */
	int dc_block_audio;     /* -E adc                                                     */
	int adc_block_const;    /* 9                                                          */
	int dc_block_raw;       /* -E rdc                                                     */
	int rdc_block_const;    /* -q, default 9                                              */
	int offset_tuning;      /* 1: skip rotate16_90 (dongle.offset_tuning)                 */
	int report_levels;      /* -L: keep every chunk's rms() for rxb200_fm_levels          */
} rxb200_fm_params;

/* CLI-level inputs of rx_fm and what main() + optimal_settings() derive from them
 * (src/rtl_fm.c:1224-1371, :960-997, :1410-1415).  Pure host arithmetic. */
typedef struct rxb200_fm_cli {
	int mode;               /* -M : RXB200_MODE_*                         */
	int wbfm;               /* -M wbfm preset (src/rtl_fm.c:1331-1341)    */
	int rate_s;             /* -s, 0 = keep default/preset                */
	int rate_r;             /* -r, 0 = none                               */
	int use_F;              /* -F given                                   */
	int comp_fir_size;      /* -F argument                                */
	int custom_atan;        /* -A, -1 = keep default/preset               */
	int post_downsample;    /* -o, default 1                              */
	int deemph;             /* -E deemp: 1, -1 = keep default/preset      */
	int time_constant_us;   /* -c: 75 (us), 50 (eu) or N                  */
	int offset_tuning;      /* -E offset / -w                             */
	int squelch_level;      /* -l                                         */
	int dc_block_audio;     /* -E adc                                     */
	int dc_block_raw;       /* -E rdc                                     */
	int rdc_block_const;    /* -q, 0 = default 9                          */
} rxb200_fm_cli;

typedef struct rxb200_fm_derived {
	rxb200_fm_params params;
	int capture_rate;        /* dongle.rate  = downsample * rate_in          */
	int capture_freq_offset; /* dongle.freq - freq (capture_rate/4 unless offset tuning) */
	int output_rate;         /* output.rate                                  */
} rxb200_fm_derived;

int rxb200_fm_derive(const rxb200_fm_cli *cli, rxb200_fm_derived *out);

typedef struct rxb200_fm rxb200_fm;

/* One handle = n_channels independent streams with identical parameters (struct demod_state x
 * n_channels; the reference has "multiple of these, eventually", src/rtl_fm.c:189).  device is
 * the CUDA ordinal. */
int rxb200_fm_create(const rxb200_fm_params *params, int device, int n_channels, rxb200_fm **out);
void rxb200_fm_destroy(rxb200_fm *h);
/* Back to the state right after create (demod_init, src/rtl_fm.c:1084). */
int rxb200_fm_reset(rxb200_fm *h);

/* Upper bound of int16 PCM produced per channel for n_int16 input values per channel. */
size_t rxb200_fm_max_output(const rxb200_fm *h, size_t n_int16, size_t chunk_int16);

/* "As if rtlsdr_callback()+full_demod() were called once per chunk_int16 slice, in order."
 *   cs16      : HOST pointer, n_channels streams of n_int16 interleaved I,Q int16 each,
 *               channel c at cs16 + c*n_int16.  n_int16 and chunk_int16 are int16 counts like the
 *               reference's len / lp_len (src/rtl_fm.c:828, :860).
 *   pcm       : HOST pointer, channel c's concatenated demod.result at pcm + c*pcm_stride.
 *   n_pcm     : receives the int16 count produced per channel (identical for all channels).
 *   chunk_result_len : optional, receives demod.result_len of every chunk (n_chunks ints).
 * Constraints (RXB200_EUNSUPPORTED otherwise): 2 <= chunk_int16 <= 262144.  Without fifth_order
 * passes (downsample_passes == 0) chunk_int16 and n_int16 may be any even count, the last chunk
 * any even length (whole complex samples, as readStream returns them).  With passes every chunk
 * (the last one included) is a multiple of 16 int16 and of 2*2^P int16.  Every chunk must produce
 * a decimated sample when a per-chunk reduction stage is on, and decimate to a multiple of
 * post_downsample.  Otherwise a chunk shorter than the boxcar may complete none: fm_demod's carried
 * sample then becomes (0, 0), as the reference pinned in tests reads it (DESIGN.md section 4.1), so
 * the next FM output is 0.  rxb200_fm_process_device wants d_cs16 32-byte aligned, or 4-byte aligned for
 * a call without passes whose chunk or length is not a multiple of 16 int16. */
int rxb200_fm_process(rxb200_fm *h, const int16_t *cs16, size_t n_int16, size_t chunk_int16,
                      int16_t *pcm, size_t pcm_stride, size_t *n_pcm, int *chunk_result_len);

/* Same with DEVICE pointers (inputs already resident in HBM); asynchronous on the handle's stream
 * unless sync != 0.  n_pcm is computed on the host (closed form) and valid at return.  A call on
 * the split kernel (kernel_kind 1) that directly follows the handle's previous split call on its
 * stream may start reading d_cs16 while that call is still running: a kernel the caller puts on
 * the handle's stream between two calls must not write the second call's input (copies,
 * and anything ordered before the first call, may). */
int rxb200_fm_process_device(rxb200_fm *h, const int16_t *d_cs16, size_t n_int16, size_t chunk_int16,
                             int16_t *d_pcm, size_t pcm_stride, size_t *n_pcm, int sync);

/* "One rtlsdr_callback()+full_demod() per channel on a read of n_int16" -- the reference's call
 * site for each readStream read (src/rtl_fm.c:828-863, :923), so a stream demodulated read by read
 * gives the reference's bytes whatever lengths the device returns.  Channel c's read is at
 * cs16 + c*n_int16; pcm, pcm_stride and n_pcm as in rxb200_fm_process.
 * Constraints (RXB200_EUNSUPPORTED otherwise): n_int16 even, 2 <= n_int16 <= 262144, and with
 * fifth_order passes n_int16 >= 2*2^P (below that the reference reads before its buffer).  The
 * read must produce a decimated sample when a per-chunk reduction stage is on, and decimate to a
 * multiple of post_downsample; otherwise a read shorter than the boxcar is accepted and carries
 * (0, 0) on as in rxb200_fm_process.  A read rxb200_fm_process(h, cs16, n_int16, n_int16, ...) takes
 * runs exactly as that call; a read with passes off their granule runs on the any-length kernel
 * (kernel_kind 0), where every pass ends where the reference's does: raw mode then returns
 * n_int16 >> P values, an odd count when L_P = n_int16 >> P is odd.  A refused call leaves the
 * handle's state untouched.  levels, squelch_hits, last_stats and kernel_ms report the read as
 * one chunk.  Calls of every process entry point may follow one another on one handle. */
int rxb200_fm_process_read(rxb200_fm *h, const int16_t *cs16, size_t n_int16, int16_t *pcm,
                           size_t pcm_stride, size_t *n_pcm);

/* Same with DEVICE pointers, like rxb200_fm_process_device; d_cs16 needs only 4-byte alignment
 * (a read below 32-byte alignment runs on the any-length kernel of its pass count). */
int rxb200_fm_process_read_device(rxb200_fm *h, const int16_t *d_cs16, size_t n_int16, int16_t *d_pcm,
                                  size_t pcm_stride, size_t *n_pcm, int sync);

/* squelch_hits after the last processed chunk, per channel (demod.squelch_hits,
 * src/rtl_fm.c:781-790) so the host thread can keep the hop logic of :928-933. */
int rxb200_fm_squelch_hits(rxb200_fm *h, int *hits /* n_channels */);

/* With params.report_levels: the rms() of every chunk of the LAST process call, laid out
 * [n_channels][n_chunks] -- the value `sr` that feeds the -L statistics (src/rtl_fm.c:792-806:
 * the squelch's rms when squelch is on, else rms(lowpassed) after the decimation filters).
 * n_chunks receives the chunk count of that call; RXB200_ECAPACITY if cap is too small. */
int rxb200_fm_levels(rxb200_fm *h, int *levels, size_t cap, size_t *n_chunks);

/* The handle's CUDA stream (cudaStream_t) for callers that time or order work themselves. */
void *rxb200_fm_stream(rxb200_fm *h);
/* Statistics of the last process call: kernel launches, de-emphasis segments that needed the
 * serial fix-up, segment length (complex samples) and warm-up length used. */
typedef struct rxb200_fm_stats {
	int launches;
	int segments;
	int fixup_segments;
	int segment_len;
	int warmup_len;
	int kernel_kind;        /* 0: fm_fused_kernel (one segment per thread), 1: fm_split_kernel with warp rows (front and back
	                           end on different items; the wbfm shape with 1..3 fifth_order passes, whole-row calls),
	                           2: no longer produced (was fm_split_kernel with per-thread segments),
	                           3: stream path, two launches -- fm_fused_kernel's front end alone (PCM to global memory), then
	                              fm_back_kernel (the wbfm shape without decimating passes, long calls) */
} rxb200_fm_stats;
int rxb200_fm_last_stats(rxb200_fm *h, rxb200_fm_stats *out);
/* Tuning knobs (0 keeps the automatic choice): segment length in complex samples, de-emphasis
 * warm-up in decimated samples.  The warm-up (default 16*deemph_a + 64) plus the resampler group
 * must fit one CTA's PCM buffer: a call whose warm-up the split kernel cannot hold runs on the fused
 * kernel (kernel_kind 0); beyond 32750 decimated samples with fifth_order passes (fewer for long
 * boxcars, DESIGN.md section 6) the call returns RXB200_EUNSUPPORTED. */
int rxb200_fm_tune(rxb200_fm *h, int segment_len, int deemph_warmup);
/* Device time of the last process call's main kernels, in milliseconds: on the row path the split
 * kernel from its first CTA's start to its last CTA's end by the GPU's global timer (no event sits
 * between two calls there, since one would keep the next call from starting early), else CUDA
 * events on the handle's stream around the fused kernel's main pass (not its per-chunk reduction
 * pre-passes) or the front and back kernels on the stream path.  Synchronises the stream. */
int rxb200_fm_kernel_ms(rxb200_fm *h, float *ms);

/* The discriminators alone, for tests: one thread per element of n quads (ar, aj, br, bj) of int32 -- the sample
 * x[n] = (ar, aj) and the one before it -- in DEVICE memory (16-byte aligned), on `stream` (a cudaStream_t, may be NULL).
 * The kernel forms the conjugate product cr = ar br + aj bj, cj = aj br - ar bj with int32 wrap, as the chains do (so the
 * quad (cr, cj, 1, 0) hands any operand pair through), and writes d_out[i] (int32) of the device function `form` names:
 *   RXB200_DISC_STD      disc_std_f32: every -A std sample
 *   RXB200_DISC_FAST     fast_atan2_i: -A fast on the fused and any-length kernels
 *   RXB200_DISC_LUT      disc_lut on the host-built table: -A lut
 *   RXB200_DISC_ALE      disc_ale: -A ale
 *   RXB200_DISC_ATAN2    disc_std (libm atan2): the first FM sample of every chunk in every mode
 *   RXB200_DISC_STD_FP64 disc_std_lean: the fp64 form alone, also on operands disc_std_f32 decides in FP32
 *   RXB200_DISC_ROWS     the int16 the row front end stores for one sample (FP32 fast_atan2, the integer form past
 *                        ||cr| - |cj|| >= 2^19); exact for |cr| + |cj| < 2^24, which its operands always meet
 *   RXB200_DISC_STREAM   the int16 the undecimated stream front end stores (FP32 product and fast_atan2); exact for
 *                        8-bit-range samples
 *   RXB200_DISC_AM       (int16)(int)sqrt(ar^2 + aj^2) with int32 wrap: the AM envelope
 * Asynchronous (the LUT form's table is freed behind the launch).  RXB200_EINVAL for an unknown form or bad pointer. */
#define RXB200_DISC_STD      RXB200_ATAN_STD
#define RXB200_DISC_FAST     RXB200_ATAN_FAST
#define RXB200_DISC_LUT      RXB200_ATAN_LUT
#define RXB200_DISC_ALE      RXB200_ATAN_ALE
#define RXB200_DISC_ATAN2    4
#define RXB200_DISC_STD_FP64 5
#define RXB200_DISC_ROWS     6
#define RXB200_DISC_STREAM   7
#define RXB200_DISC_AM       8
int rxb200_fm_disc_device(int form, const int32_t *d_quads, size_t n, int32_t *d_out, void *stream);

/* ======================================================================== rx_power
 * Replaces scanner()'s per-hop body (src/rtl_power.c:709-771): copy, boxcar | downsample_iq x P +
 * generic_fir, remove_dc x2, and per N-point block window multiply, fix_fft() (:264-320) and
 * real_conj accumulate (sum or peak hold); rms_power() (:403-429) when bin_e == 0.
 * Accumulators (tunes[i].avg / .samples, :95-96) live device-side in the handle.
 */
typedef struct rxb200_power_params {
	int n_hops;             /* tune_count                                       */
	int bin_e;              /* tunes[0].bin_e; FFT length N = 1 << bin_e        */
	int buf_len;            /* tunes[0].buf_len, int16 per hop buffer           */
	int downsample;         /* tunes[0].downsample                              */
	int downsample_passes;  /* tunes[0].downsample_passes                       */
	int comp_fir_size;      /* global comp_fir_size (-F arg)                    */
	int boxcar;             /* global boxcar (0 with -F)                        */
	int peak_hold;          /* global peak_hold (-P)                            */
} rxb200_power_params;

/* frequency_range() (src/rtl_power.c:431-543): the hop/bin planner.  Pure host arithmetic. */
typedef struct rxb200_power_plan {
	rxb200_power_params params;
	int rate;               /* tunes[i].rate (bw_used)                          */
	double crop;            /* tunes[i].crop                                    */
	int64_t first_freq;     /* tunes[0].freq                                    */
	int64_t freq_step;      /* tunes[i+1].freq - tunes[i].freq (bw_seen)        */
	double bin_size_hz;
} rxb200_power_plan;
int rxb200_power_plan_range(int64_t lower, int64_t upper, int64_t max_bin_hz, double crop,
                            int boxcar, int comp_fir_size, int peak_hold, rxb200_power_plan *out);

/* Window shapes of rx_power -w (src/rtl_power.c:322-401, :881-898) plus plain Hann.  Writes
 * (int)(256*w(i,length)) like main() does (:1034-1037). */
#define RXB200_WIN_RECTANGLE 0
#define RXB200_WIN_HAMMING 1
#define RXB200_WIN_BLACKMAN 2
#define RXB200_WIN_BLACKMAN_HARRIS 3
#define RXB200_WIN_HANN_POISSON 4
#define RXB200_WIN_YOUSSEF 5
#define RXB200_WIN_KAISER 6
#define RXB200_WIN_BARTLETT 7
#define RXB200_WIN_HANN 8
int rxb200_window_table(int window, int length, int *coefs);
/* sine_table() (src/rtl_power.c:240-254): 3N/4 entries of round(32767*sin(2*pi*i/N)). */
int rxb200_sine_table(int log2_n, int16_t *sine);

typedef struct rxb200_power rxb200_power;

/* window_coefs: N ints (the global window_coefs table; only w mod 2^16 changes the result); sinewave:
 * 3N/4 int16 (the global Sinewave, any values, -32768 included) or NULL to build it with rxb200_sine_table. */
int rxb200_power_create(const rxb200_power_params *params, const int *window_coefs,
                        const int16_t *sinewave, int device, rxb200_power **out);
void rxb200_power_destroy(rxb200_power *h);

/* n_pass sweeps over hops [hop_begin, hop_end): hop_bufs is int16[n_pass][hop_end-hop_begin][buf_len],
 * each row "what readStream left in ts->buf16[0..buf_len)" (SURVEY.md F10).  Accumulates into the
 * handle's avg/samples exactly like n_pass calls of scanner() would for those hops. */
int rxb200_power_accumulate(rxb200_power *h, const int16_t *hop_bufs, int n_pass, int hop_begin, int hop_end);
int rxb200_power_accumulate_device(rxb200_power *h, const int16_t *d_hop_bufs, int n_pass,
                                   int hop_begin, int hop_end, int sync);
/* Copy out tunes[i].avg (int64[n_hops][N]) and tunes[i].samples (int[n_hops]); either may be NULL. */
int rxb200_power_read(rxb200_power *h, int64_t *avg, int *samples);
/* Device pointer to the int64[n_hops][N] accumulator rows (for an NCCL all-gather by the caller). */
int64_t *rxb200_power_device_avg(rxb200_power *h);
/* csv_dbm()'s side effect: zero avg and samples (src/rtl_power.c:813-816). */
int rxb200_power_reset(rxb200_power *h);
void *rxb200_power_stream(rxb200_power *h);
int rxb200_power_last_launches(rxb200_power *h);
/* Device time of the batched kernel alone in the last accumulate call (ms); synchronises. */
int rxb200_power_kernel_ms(rxb200_power *h, float *ms);
/* What the last accumulate call with n_pass > 0 ran (kernel RXB200_POWER_PATH_NONE before the first). */
#define RXB200_POWER_PATH_NONE 0
#define RXB200_POWER_PATH_RMS 1          /* power_rms_kernel (bin_e == 0)                                     */
#define RXB200_POWER_PATH_FFT8 2         /* power_fft8_kernel<bin_e, threads>                                 */
#define RXB200_POWER_PATH_GENERIC 3      /* power_fft_kernel<nb>                                              */
#define RXB200_POWER_PATH_BIG_LOAD 4     /* hop buffer beyond shared memory: copy / boxcar, then the FFT steps  */
#define RXB200_POWER_PATH_BIG_DECIM 5    /* hop buffer beyond shared memory: -F passes, then the FFT steps      */
typedef struct rxb200_power_path {
	int kernel;             /* RXB200_POWER_PATH_*                                                          */
	int bin_e;
	int threads;            /* CTA width of the main kernel                                                 */
	int nb;                 /* GENERIC: bins each thread accumulates in registers, 0 = straight to global; else -1 */
	int tables_in_smem;     /* GENERIC: sine and window tables staged in shared memory; FFT8: 1; else 0      */
	int slices;             /* CTAs per hop, each taking every slices-th pass; 0 on the big paths           */
	int launches;           /* kernel launches of the call (rxb200_power_last_launches)                     */
} rxb200_power_path;
int rxb200_power_last_path(rxb200_power *h, rxb200_power_path *out);

/* csv_dbm()'s numeric half ON THE DEVICE (src/rtl_power.c:783-811): DC-bin patch, half swap, crop and
 * power -> dB in the reference's fp64 operation order, so that only the final dB values leave the GPU.
 * db receives [n_hops][row_len] doubles, row_len = kept bins + 1 (the reference prints the last bin
 * twice, :807-811); rows are row_stride doubles apart.  The accumulators are NOT modified (call
 * rxb200_power_reset for csv_dbm's zeroing, :813-816).  RXB200_ECAPACITY if row_stride < row_len. */
int rxb200_power_row_len(int bin_e, double crop);
int rxb200_power_read_db(rxb200_power *h, int rate, double crop, double *db, size_t row_stride, int *samples);
/* The text half: same line as rxb200_power_format_row from one row of rxb200_power_read_db. */
int rxb200_power_format_db_row(const double *db_row, int bin_e, int64_t freq, int rate, int downsample,
                               double crop, int samples, char *dst, size_t cap);

/* csv_dbm() (src/rtl_power.c:774-817) for one hop row on the host: formats
 * "Hz low, Hz high, Hz step, samples, dB, dB, ...\n" into dst (the caller prints the date/time
 * prefix, :1048).  avg_row (N int64) is modified like the reference does (DC nuke + fft-shift).
 * Returns the number of bytes written, or RXB200_ECAPACITY. */
int rxb200_power_format_row(int64_t *avg_row, int bin_e, int64_t freq, int rate, int downsample,
                            double crop, int samples, char *dst, size_t dst_cap);

/* ======================================================================== rx_power on several GPUs (SURVEY.md §8e)
 * Tuner hops are independent (one scanner() iteration each, src/rtl_power.c:679-771), so they shard over GPUs:
 * rank r of n owns the contiguous hops [r*per, (r+1)*per), per = ceil(n_hops/n) (rxb200_power_shard).  The only
 * exchange is the collation before the report loop (src/rtl_power.c:1047-1050 walks tunes[] in hop order): ONE NCCL
 * all-gather of the int64 accumulator rows (+ the samples vector), done IN PLACE on the handle's accumulator array,
 * after which every rank holds every row and rxb200_power_read / _read_db work as on a single GPU.
 * NCCL is bound at run time (libnccl.so.2); RXB200_EUNSUPPORTED when it cannot be loaded. */
typedef struct rxb200_comm rxb200_comm;
#define RXB200_UNIQUE_ID_BYTES 128
#define RXB200_MAX_RANKS 16
/* one process per GPU: rank 0 makes the id, the launcher's own transport carries the 128 bytes to the others */
int rxb200_comm_unique_id(void *id128);
int rxb200_comm_create(int n_ranks, int rank, const void *id128, int device, rxb200_comm **out);
/* one process, n_dev GPUs (devices == NULL: 0..n_dev-1): out receives n_dev communicators */
int rxb200_comm_create_all(int n_dev, const int *devices, rxb200_comm **out);
void rxb200_comm_destroy(rxb200_comm *c);
int rxb200_comm_size(const rxb200_comm *c);
int rxb200_comm_rank(const rxb200_comm *c);
int rxb200_power_shard(int n_hops, int n_ranks, int rank, int *hop_begin, int *hop_end);
/* The collation, enqueued on the handle's stream behind its kernels; collective: every rank of the communicator calls
 * it with a handle of identical parameters that accumulated (only) its own hop range since the last reset. */
int rxb200_power_gather(rxb200_power *h, rxb200_comm *c, int sync);

/* All ranks inside ONE process (what the drop-in rx_power shell uses): n_dev handles, one per GPU. */
typedef struct rxb200_power_group rxb200_power_group;
int rxb200_power_group_create(const rxb200_power_params *params, const int *window_coefs, const int16_t *sinewave,
                              int n_dev, const int *devices, rxb200_power_group **out);
void rxb200_power_group_destroy(rxb200_power_group *g);
int rxb200_power_group_size(const rxb200_power_group *g);
rxb200_power *rxb200_power_group_member(rxb200_power_group *g, int i);
/* like rxb200_power_accumulate (HOST hop buffers); each member takes the hops of the range it owns */
int rxb200_power_group_accumulate(rxb200_power_group *g, const int16_t *hop_bufs, int n_pass, int hop_begin, int hop_end);
/* the all-gather; afterwards member 0 (every member) reads/reports all hops */
int rxb200_power_group_gather(rxb200_power_group *g);
int rxb200_power_group_reset(rxb200_power_group *g);

/* ======================================================================== rx_fm on several GPUs (SURVEY.md §8e)
 * Channels are independent demod_state streams, so they split over GPUs with no exchange at all: one process, n_dev
 * rxb200_fm handles, member i owning the contiguous channels [b, e) that rxb200_power_shard(n_channels, n_dev, i, &b, &e)
 * gives (5 channels over 4 members: 2 + 2 + 1 + 0).  A member whose range is empty has no handle.  devices == NULL
 * means 0..n_dev-1; an ordinal may repeat (several members on one GPU).
 * The group behaves byte for byte like ONE rxb200_fm handle with n_channels channels: the same pcm, n_pcm,
 * chunk_result_len, squelch hits, levels ([n_channels][n_chunks]) and refusal codes, over any sequence of process,
 * process_read and reset calls.  cs16 and pcm are HOST pointers laid out as for rxb200_fm_process (channel c at
 * cs16 + c*n_int16 and pcm + c*pcm_stride).  A call refused for its shape or capacity is refused before any member
 * starts and leaves every member's state untouched.  Each member copies its block of channels to its GPU, runs
 * rxb200_fm_process_device / _read_device and copies its PCM rows back, all on its own stream; the call returns when
 * every member is done, also after a CUDA failure, and leaves the caller's current device as it found it.  The copies
 * of different GPUs overlap only with pinned (page-locked) host buffers: with pageable ones they run one after the
 * other and only the kernels overlap them (the bytes are the same either way). */
typedef struct rxb200_fm_group rxb200_fm_group;
int rxb200_fm_group_create(const rxb200_fm_params *params, int n_channels, int n_dev, const int *devices,
                           rxb200_fm_group **out);
void rxb200_fm_group_destroy(rxb200_fm_group *g);
int rxb200_fm_group_size(const rxb200_fm_group *g);
/* member i's handle (its channels are channel 0.. of that handle), NULL for a member that owns no channel */
rxb200_fm *rxb200_fm_group_member(rxb200_fm_group *g, int i);
int rxb200_fm_group_process(rxb200_fm_group *g, const int16_t *cs16, size_t n_int16, size_t chunk_int16,
                            int16_t *pcm, size_t pcm_stride, size_t *n_pcm, int *chunk_result_len);
int rxb200_fm_group_process_read(rxb200_fm_group *g, const int16_t *cs16, size_t n_int16,
                                 int16_t *pcm, size_t pcm_stride, size_t *n_pcm);
int rxb200_fm_group_squelch_hits(rxb200_fm_group *g, int *hits /* n_channels */);
int rxb200_fm_group_levels(rxb200_fm_group *g, int *levels, size_t cap, size_t *n_chunks);
int rxb200_fm_group_reset(rxb200_fm_group *g);

/* ======================================================================== rx_fm channels of one capture
 * Several channels of ONE wideband CS16 capture: channel k is the reference's rtlsdr_callback() + full_demod() run on
 * mix_k(x), what a tuner set f_k (Hz) away from the capture's centre would have delivered (DESIGN.md section 4.4).  The
 * integer mixer, for a capture rate R (Hz, > 0) and an offset f with |f| < R/2:
 *   period L = R / gcd(R, |f|) complex samples (1 for f = 0), at most 2^20 (RXB200_EUNSUPPORTED beyond);
 *   table entry m = (c, s) = ((int)round(32768 cos t), (int)round(32768 sin t)), t = -2 pi r / R in fp64, where
 *     r = (m f) mod R taken in 64-bit integers as the representative in (-R/2, R/2] (the same angle modulo 2 pi; it
 *     makes the tables of f and -f exact conjugates);
 *   complex sample n of the stream (counted from create or reset, across calls) uses entry p = (phase + n) mod L:
 *     I' = (int16)((I c - Q s + 2^14) >> 15),  Q' = (int16)((I s + Q c + 2^14) >> 15)   (arithmetic shift, int16 wrap).
 * Unity 2^15 makes f = 0 the identity and f = +-R/4 an exact rotation.  Then the chain runs as configured: pick
 * offset_tuning = 1 (the mixer already put the channel at DC, so rotate16_90 should not run) and downsample =
 * R / rate_in, so the boxcar is the channel filter. */

/* The mixer table of (R, f): table receives 2*L int32 (c, s pairs), *period receives L.  RXB200_EINVAL for R <= 0 or
 * |f| >= R/2, RXB200_EUNSUPPORTED for L > 2^20, RXB200_ECAPACITY (with *period set) when cap < 2*L int32. */
int rxb200_fm_mix_table(int capture_rate, int offset_hz, int32_t *table, size_t cap, size_t *period);
/* The mixer alone on DEVICE pointers, on `stream` (a cudaStream_t, may be NULL): n_complex samples of d_src, starting
 * at table entry phase mod L (phase >= 0), to d_dst.  Both pointers 4-byte aligned; 16-byte aligned ones take vector
 * loads and stores.  Asynchronous. */
int rxb200_mix_device(int capture_rate, int offset_hz, long long phase, const int16_t *d_src, size_t n_complex,
                      int16_t *d_dst, void *stream);

/* A handle of n_channels channels of one capture: one rxb200_fm handle with n_channels channels (the member) plus the
 * mixer of each channel, whose phases start at 0.  Every call takes ONE input stream: the capture's n_int16 int16.
 * fm_mix_kernel reads it once and writes the n_channels mixed streams to a scratch buffer of the handle ([n_channels]
 * [n_int16], rows n_int16 apart from a 256-byte aligned base); the member's rxb200_fm_process_device / _read_device
 * then runs on that buffer, so every kernel route, carry, statistic and result of the member is that of a plain handle
 * fed the mixed streams.  pcm, pcm_stride, n_pcm and chunk_result_len are those of rxb200_fm_process*, channel k's PCM
 * at pcm + k*pcm_stride.  Refusals are those of the matching rxb200_fm_process* call, checked before anything is
 * launched, except that a device capture needs only 4-byte alignment; a refused call changes neither the phases nor
 * the member's state.  A successful call advances every phase by its n_int16 / 2 complex samples. */
typedef struct rxb200_fm_mix rxb200_fm_mix;
int rxb200_fm_mix_create(const rxb200_fm_params *params, int capture_rate, const int *offsets_hz, int n_channels,
                         int device, rxb200_fm_mix **out);
void rxb200_fm_mix_destroy(rxb200_fm_mix *m);
/* phases back to 0 and the member back to the state right after create */
int rxb200_fm_mix_reset(rxb200_fm_mix *m);
/* the inner handle, for rxb200_fm_last_stats / _kernel_ms / _tune / _stream (and the mixer runs on its stream) */
rxb200_fm *rxb200_fm_mix_member(rxb200_fm_mix *m);
int rxb200_fm_mix_process(rxb200_fm_mix *m, const int16_t *cs16, size_t n_int16, size_t chunk_int16, int16_t *pcm,
                          size_t pcm_stride, size_t *n_pcm, int *chunk_result_len);
int rxb200_fm_mix_process_device(rxb200_fm_mix *m, const int16_t *d_cs16, size_t n_int16, size_t chunk_int16,
                                 int16_t *d_pcm, size_t pcm_stride, size_t *n_pcm, int sync);
int rxb200_fm_mix_process_read(rxb200_fm_mix *m, const int16_t *cs16, size_t n_int16, int16_t *pcm, size_t pcm_stride,
                               size_t *n_pcm);
int rxb200_fm_mix_process_read_device(rxb200_fm_mix *m, const int16_t *d_cs16, size_t n_int16, int16_t *d_pcm,
                                      size_t pcm_stride, size_t *n_pcm, int sync);
int rxb200_fm_mix_squelch_hits(rxb200_fm_mix *m, int *hits /* n_channels */);
int rxb200_fm_mix_levels(rxb200_fm_mix *m, int *levels, size_t cap, size_t *n_chunks);
/* Device time (CUDA events on the member's stream) of the last successful call's fm_mix_kernel (fm_ddc_kernel for a
 * decimating handle), in milliseconds; synchronises the stream. */
int rxb200_fm_mix_kernel_ms(rxb200_fm_mix *m, float *ms);

/* ---- decimating mixing handles: mixer, channel filter and decimation before the chain (a digital down-converter)
 * A decimating handle has a capture rate R and K offsets as above, plus one rxb200_ddc shared by every channel: a
 * decimation factor M (1..4096), T int32 taps h[0..T) (1 <= T <= 8192, copied at create) and a rounding shift S
 * (0..62).  For channel k let z[n] = mix_k(x)[n], n counting capture samples from create or reset across calls, and
 * z[n] = 0 for n < 0.  Output m >= 0 is emitted at capture sample e_m = m*M + M - 1; for I and Q separately
 *     A = sum_{j<T} h[j] * z[e_m - j]   (exact, 64-bit);   y = S ? (A + 2^(S-1)) >> S : A   (arithmetic);
 *     out = y saturated to [-32768, 32767].
 * Channel k is the reference's rtlsdr_callback() + full_demod() on that decimated CS16 stream, through the member's
 * chain with any parameters; typically offset_tuning = 1 and downsample = R / (M * rate_in).
 * A call covering capture samples [n0, n0 + c) hands the chain the floor((n0+c)/M) - floor(n0/M) outputs whose e_m
 * falls in it (rxb200_fm_mix_decimated_len).  Read calls (_process_read*): those outputs are one read of the member; a
 * read with no output runs no chain call, returns n_pcm = 0 and zero level chunks, and still advances the phases and
 * the filter history; a decimated read the member refuses (for example fewer than 2^P complex samples with passes)
 * refuses the whole call.  Chunk calls (_process*): chunk_int16 must be a multiple of 2M (else RXB200_EUNSUPPORTED);
 * capture chunk c is then decimated chunk c of chunk_int16 / M int16 at any phase, the last partial capture chunk the
 * decimated remainder, and chunk_result_len entries of capture chunks with no decimated sample are 0.  Every other
 * refusal is the member's on the decimated shape; a refused call changes nothing.  fm_ddc_kernel mixes and filters in
 * one pass (int32 accumulation when sum |h| * 32768 + 2^(S-1) < 2^31, else int64), so only the decimated streams,
 * [K][n_dec_int16], reach the scratch buffer.  Reset also zeroes the filter history.  M = 1, h = {1}, S = 0 gives
 * the bytes of the plain mixing handle. */
typedef struct rxb200_ddc {
	int decim;             /* M */
	int n_taps;            /* T */
	const int32_t *taps;   /* h[0..T) */
	int shift;             /* S */
} rxb200_ddc;
/* RXB200_EINVAL for a NULL ddc or taps, M, T or S out of range, or sum |h| * 32768 + 2^(S-1) >= 2^63; every refusal
 * of rxb200_fm_mix_create otherwise.  The handle takes every rxb200_fm_mix_* entry point. */
int rxb200_fm_mix_create_ddc(const rxb200_fm_params *params, int capture_rate, const int *offsets_hz, int n_channels,
                             const rxb200_ddc *ddc, int device, rxb200_fm_mix **out);
/* *n_dec_int16: the int16 per channel the next call of n_int16 capture int16 hands the chain, at the current phase
 * (n_int16 for a plain mixing handle), so that a caller with passes can check a read before making it. */
int rxb200_fm_mix_decimated_len(const rxb200_fm_mix *m, size_t n_int16, size_t *n_dec_int16);
/* A bound on the PCM per channel of a call of n_int16 capture int16 in chunks of chunk_int16, at any phase (any
 * mixing handle). */
size_t rxb200_fm_mix_max_output(const rxb200_fm_mix *m, size_t n_int16, size_t chunk_int16);
/* The DDC alone on DEVICE pointers, stateless, on `stream`: the samples before d_src are zero, the mixer starts at
 * table entry phase mod L (phase >= 0), and floor(n_complex / M) outputs go to d_dst, e_m counted from d_src.  Both
 * pointers 4-byte aligned.  Asynchronous. */
int rxb200_ddc_device(int capture_rate, int offset_hz, long long phase, const rxb200_ddc *ddc, const int16_t *d_src,
                      size_t n_complex, int16_t *d_dst, void *stream);

/* ---- rx_fm channels of one capture in the shell (DESIGN.md section 4.4, "Capture mode in the rx_fm shell")
 * The plan the rx_fm shell's capture mode (RXB200_CAPTURE_RATE) uses to take K tuned frequencies t_k (Hz) from one
 * capture through a decimating handle, for a chain whose capture rate is c (rxb200_fm_derived.capture_rate):
 *   tmin, tmax = the smallest and largest t_k; g = gcd of every t_k - tmin (g = 0 when every t_k is equal);
 *   fc = tmin when g = 0, else tmin + g floor((tmax - tmin) / (2 g)), so every offset is a multiple of the channel grid
 *     and the mixer's period L = R / gcd(R, |o|) stays small for ordinary rasters;
 *   o_k = t_k - fc, A = max |o_k|;  M = ceil((2 A + c) / c), so |o_k| < R / 2;  R = M c;  T = min(8191, 32 M + 1);
 *   the filter is rxb200_ddc_lowpass(M, T, 15) at shift S = 15, the one rx_power's capture mode uses.
 * Refusals, pure host arithmetic: RXB200_EINVAL for a NULL pointer, K < 1, c < 1, any t_k outside [0, 2^61), and R
 * above max_capture_rate or 2^31 - 1 or M > 256 (the message names R); for an offset whose mixer table
 * rxb200_fm_mix_table refuses, that call's code and message (RXB200_EUNSUPPORTED for a period above 2^20).  M is capped
 * at 256 because the shell holds each block of M * 131072 complex capture samples (M * 512 KiB) on the host, four in
 * flight. */
typedef struct rxb200_fm_capture_plan {
	int64_t centre_hz;   /* fc */
	int decim;           /* M */
	int capture_rate;    /* R = M c */
	int n_taps;          /* T */
} rxb200_fm_capture_plan;
/* offsets_hz receives the K offsets o_k. */
int rxb200_fm_plan_capture(const int64_t *tuned_hz /* n_channels */, int n_channels, int chain_rate,
                           long long max_capture_rate, rxb200_fm_capture_plan *out, int *offsets_hz /* n_channels */);

/* ---- raster mixing handles: the channels of a uniform raster through a polyphase channelizer (DESIGN.md section 4.4,
 * "Channels on a raster")
 * A raster handle has K bins (3 <= K <= 4096) over the capture and n_channels channels, channel c being bin k_c
 * (0 <= k_c < K; bins may repeat), centred at k_c R / K for a capture rate R (negative for k_c > K/2), plus one rxb200_ddc
 * (M, T taps h, S) shared by every channel.  Let x[n] be the capture, n counting complex samples from create or reset
 * across calls, x[n] = 0 for n < 0, and tw[r] = (c, s) entry r of rxb200_fm_mix_table(K, 1) (the period-K table:
 * round(2^15 cos, sin) of -2 pi r' / K, r' the representative of r in (-K/2, K/2], so bins k and K - k are conjugates).
 * Output m of channel c (bin k) is emitted at e_m = m*M + M - 1:
 *     A = sum_{j<T} h[j] * x[e_m - j] * tw[(k (e_m - j)) mod K]   (complex, exact: no rounding anywhere in the sum);
 *     y = S ? (A + 2^(S-1)) >> S : A   (arithmetic, I and Q separately);   out = y saturated to [-32768, 32767].
 * This is the decimating handle's rule at offset k R / K without the mixer's per-sample >> 15 rounding and int16 wrap, so
 * it is not byte for byte that handle.  Two anchors are exact: bin 0 at shift S + 15 is the decimating handle at offset 0
 * with shift S; and bin K/4 (4 | K) at shift S + 15 is the decimating handle at offset R/4 with shift S whenever no I or
 * Q sample is -32768 (the quarter-turn mixer wraps there).  Everything else is a decimating handle's: the decimated length, the chunk rule (multiples of 2M), a
 * read with no output, the refusals on the decimated shape, reset, and every rxb200_fm_mix_* entry point; there is no
 * capture rate, and rxb200_fm_mix_kernel_ms reports the two raster kernels of the last call summed.
 * raster_branch_kernel sums each output's taps by residue rho = (e_m - j) mod K into v_rho (fp64, exact below 2^37),
 * and raster_dft_kernel multiplies those rows by the handle's constant [2K][2C] twiddle matrix on FP64 tensor cores
 * (DMMA); every product and partial sum is an integer below 2^53, so the result is exact in any summation order.  The
 * branch sums of a long call go through a scratch buffer in groups of at most RXB200_RASTER_SCRATCH_BYTES of frames;
 * the bytes are the same as with one group. */
#define RXB200_RASTER_SCRATCH_BYTES (64u << 20)
/* Refusals, all before any device is touched: those of rxb200_fm_mix_create_ddc for params and ddc; RXB200_EINVAL for
 * K outside [3, 4096], NULL bins, n_channels < 1, any bin outside [0, K), or sum |h| >= 2^22 (which keeps every partial
 * sum, |A| <= sum |h| 2^31, below 2^53). */
int rxb200_fm_mix_create_raster(const rxb200_fm_params *params, int n_bins, const int *bins /* n_channels */,
                                int n_channels, const rxb200_ddc *ddc, int device, rxb200_fm_mix **out);
/* The raster down-converter alone on DEVICE pointers, stateless, on `stream`: d_src[i] is capture sample n0 + i (its
 * twiddle uses (k (n0 + i)) mod K, n0 + i taken as an exact integer), the samples before d_src are zero, and
 * floor(n_complex / M) outputs per channel go to d_dst, channel c's at d_dst + 2 c floor(n_complex / M), e_m counted
 * from d_src.  Both pointers 4-byte aligned.  The refusals of rxb200_fm_mix_create_raster for K, bins and ddc.
 * Asynchronous. */
int rxb200_raster_device(int n_bins, const int *bins, int n_channels, unsigned long long n0, const rxb200_ddc *ddc,
                         const int16_t *d_src, size_t n_complex, int16_t *d_dst, void *stream);

/* ---- two-stage mixing handles: channels at any offset through a shared polyphase stage, then a per-channel NCO stage
 * (DESIGN.md section 4.4, "Channels at any offset in two stages")
 * A two-stage handle has a capture rate R > 0 (Hz), one integer offset f_c per channel with |f_c| < R/2, K coarse bins
 * (3 <= K <= 4096), a coarse rxb200_ddc d1 = (M1, T1, h1, S1) with sum |h1| < 2^22 (the raster bound) and a fine
 * rxb200_ddc d2 = (M2, T2, h2, S2), with M = M1 M2 <= 4096.  Indices n count capture samples from create or reset across
 * calls; every stream is 0 before index 0.
 *   Bin and word of channel c: b_c = floor((f_c K + floor(R/2)) / R) mod K (the nearest bin centre b R / K, ties
 *     rounded up); N_c = (f_c K - b'_c R) M1 with b'_c the representative of b_c in (-K/2, K/2]; D = K R;
 *     w_c = floor((N_c 2^32 + floor(D/2)) / D) mod 2^32, exact (128-bit host integers): the rx_power NCO word of the
 *     residual offset f_c - b'_c R / K at the coarse rate R / M1 (rxb200_two_stage_word).
 *   Coarse stage: for each bin b that holds a channel, y_b[m] is output m of the raster rule above for bin b with d1:
 *     emitted at e1_m = m M1 + M1 - 1, twiddle tw[(b n) mod K] of rxb200_fm_mix_table(K, 1), no rounding inside the
 *     sum, then the S1 shift and int16 saturation.
 *   Fine stage: z_c[m] = y_{b_c}[m] through the rx_power NCO mixer (rxb200_nco_table) at phase m w_c mod 2^32, with
 *     mix_one's rounding and int16 wrap; output q is emitted at coarse index q M2 + M2 - 1:
 *     A = sum_{j<T2} h2[j] z_c[q M2 + M2 - 1 - j] (exact), then the S2 shift and int16 saturation.
 * Fine output q falls at capture sample q M + M - 1, so the decimated length (rxb200_fm_mix_decimated_len), the chunk
 * rule (multiples of 2M), a read with no output, the refusals on the decimated shape, reset and every rxb200_fm_mix_*
 * entry point behave exactly as for a decimating handle with decimation M; rxb200_fm_mix_kernel_ms reports both stages
 * of the last call summed.  It is neither the decimating handle, the raster handle nor a single-stage filter byte for
 * byte.  Two anchors are exact: M1 = 1, T1 = 1, h1 = {1}, S1 = 15 and a channel on bin 0 give rxb200_power_ddc_device
 * (R, f_c, n0, d2) (the twiddle of bin 0 is 2^15, so the coarse stage is the identity, and for even R the word is the
 * rx_power word); and M2 = 1, T2 = 1, h2 = {1}, S2 = 0 with f_c = b_c R / K exactly (so w_c = 0) give the raster
 * handle with bins b_c.
 * The coarse stage runs the raster kernels for the distinct bins only; the fine stage runs fine_ddc_kernel (ddc.cuh's
 * down-converter with the NCO mixer) with the channels in bin order, each grid row staging its bin's coarse stream once.
 * The handle carries the capture count, the coarse stage's last T1 - 1 raw samples and each bin's last T2 - 1 coarse
 * samples, and a call's next histories become live only when it succeeds.  A long call runs in groups of coarse frames
 * whose branch sums and coarse rows fit about RXB200_RASTER_SCRATCH_BYTES; the bytes are the same as with one group.
 * Refusals, all before any device is touched: those of rxb200_fm_mix_create_ddc for params and d2; those of
 * rxb200_fm_mix_create_raster for K and d1; RXB200_EINVAL for R <= 0, NULL offsets, n_channels < 1, any |f_c| >= R/2
 * and M1 M2 > 4096. */
int rxb200_fm_mix_create_two_stage(const rxb200_fm_params *params, int capture_rate, int n_bins,
                                   const int *offsets_hz /* n_channels */, int n_channels, const rxb200_ddc *coarse,
                                   const rxb200_ddc *fine, int device, rxb200_fm_mix **out);
/* b_c into bins[c] and w_c into words[c] for M1 = coarse_decim, pure host arithmetic.  RXB200_EINVAL for a NULL pointer,
 * n_channels < 1, R <= 0, K outside [3, 4096], M1 outside [1, 4096] or any |f_c| >= R/2. */
int rxb200_two_stage_word(int capture_rate, int n_bins, int coarse_decim, const int *offsets_hz /* n_channels */,
                          int n_channels, int *bins /* n_channels */, uint32_t *words /* n_channels */);
/* The two stages alone on DEVICE pointers, stateless, on `stream`: d_src[i] is capture sample n0 + i (its twiddle uses
 * (b (n0 + i)) mod K, n0 + i an exact integer), the samples before d_src are zero, coarse output m is emitted at d_src
 * index m M1 + M1 - 1 and mixed at phase (floor(n0 / M1) + m) w_c, and fine output q at coarse output q M2 + M2 - 1;
 * floor(n_complex / M) outputs per channel go to d_dst, channel c's at d_dst + 2 c floor(n_complex / M).  For M | n0
 * this is the rule for a capture that is zero before n0.  Both pointers 4-byte aligned.  The refusals of
 * rxb200_fm_mix_create_two_stage but the params'.  Asynchronous. */
int rxb200_two_stage_device(int capture_rate, int n_bins, const int *offsets_hz /* n_channels */, int n_channels,
                            unsigned long long n0, const rxb200_ddc *coarse, const rxb200_ddc *fine,
                            const int16_t *d_src, size_t n_complex, int16_t *d_dst, void *stream);
/* The plan the rx_fm shell's capture mode uses with RXB200_CAPTURE_STAGES=2 for K tuned frequencies t_k of a chain whose
 * capture rate is c: fc and the offsets o_k as rxb200_fm_plan_capture gives them; M from that plan's rule,
 * M' = 4 ceil(M / 4); R = M' c; M2 = 4, M1 = M' / 4 and K = 2 M1 (bins 2c apart, coarse rate 4c, residual at most c);
 * the coarse filter rxb200_ddc_lowpass(M1, min(8191, 24 M1 + 1), 15) at S1 = 30 (Q15 taps times the 2^15 twiddle) and
 * the fine filter rxb200_ddc_lowpass(4, 129, 15) at S2 = 15, so the final cutoff is c/2 as in the single-stage plan.
 * Refusals, pure host arithmetic: RXB200_EINVAL for a NULL pointer, K < 1, c < 1, any t_k outside [0, 2^61), M' < 8, and
 * R above max_capture_rate or 2^31 - 1 or M' > 256 (the message names R). */
typedef struct rxb200_fm_two_stage_plan {
	int64_t centre_hz;     /* fc */
	int capture_rate;      /* R = M' c */
	int n_bins;            /* K = 2 M1 */
	int coarse_decim;      /* M1 */
	int coarse_taps;       /* T1 */
	int coarse_shift;      /* S1 = 30 */
	int fine_decim;        /* M2 = 4 */
	int fine_taps;         /* T2 = 129 */
	int fine_shift;        /* S2 = 15 */
} rxb200_fm_two_stage_plan;
/* offsets_hz receives the K offsets o_k. */
int rxb200_fm_plan_capture_two_stage(const int64_t *tuned_hz /* n_channels */, int n_channels, int chain_rate,
                                     long long max_capture_rate, rxb200_fm_two_stage_plan *out,
                                     int *offsets_hz /* n_channels */);
/* The plan the rx_fm and rx_sdr shells' capture modes use with RXB200_CAPTURE_STAGES=raster, for K tuned frequencies t_k
 * on a common grid and a chain capture rate c (rx_sdr: its -s): the channels as bins of one raster handle.
 *   fc, M, R = M c and T = min(8191, 32 M + 1) are exactly those of rxb200_fm_plan_capture, and g is its grid (the gcd
 *     of every t_k - tmin, 0 when every t_k is equal), so every o_k = t_k - fc is a multiple of g;
 *   K0 = R / gcd(R, g) (K0 = 1 for g = 0); K = K0 when K0 >= 3, else 3 (then every o_k is 0);
 *   bin of channel k: b_k = (o_k K / R) mod K, exact since R / K divides every o_k; so a channel at fc is bin 0;
 *   the filter is rxb200_ddc_lowpass(M, T, 15) at shift S = 30 (Q15 taps times the 2^15 twiddle).
 * By the raster anchor (bin 0 at shift S + 15 is the decimating handle at offset 0 with shift S), the stream of a channel
 * at fc is byte for byte the one the default capture mode gives it; every other channel's differs from it.
 * Worked examples (the FM broadcast band is one -f per station):
 *   -f set                                 chain rate c          fc            M   R           T     K
 *   88.1-107.9 MHz, 200 kHz grid (100 ch)  250 kHz (rx_sdr -s)   97.9 MHz      81  20 250 000  2593  405
 *   162.400-162.550 MHz, 25 kHz (7 ch)     25 kHz (rx_sdr -s)    162.475 MHz   7   175 000     225   7
 *   162.400-162.550 MHz, 25 kHz (7 ch)     1 008 000 (-s 24k)    162.475 MHz   2   2 016 000   65    2016
 *   162.400, 162.400001, 162.550 MHz       25 kHz                refused: g = 1 Hz, M = 7, K = 175 000
 * Refusals, pure host arithmetic: those of rxb200_fm_plan_capture for the arguments, the cap, 2^31 - 1 and M > 256 (no
 * mixer-table refusal: there is no table mixer); RXB200_EINVAL for K > 4096 (the message names K and the grid, and
 * RXB200_CAPTURE_STAGES=2 for channels off a grid). */
typedef struct rxb200_fm_raster_plan {
	int64_t centre_hz;     /* fc */
	int capture_rate;      /* R = M c */
	int n_bins;            /* K */
	int decim;             /* M */
	int n_taps;            /* T */
	int shift;             /* S = 30 */
} rxb200_fm_raster_plan;
/* bins receives the K bins b_k. */
int rxb200_fm_plan_capture_raster(const int64_t *tuned_hz /* n_channels */, int n_channels, int chain_rate,
                                  long long max_capture_rate, rxb200_fm_raster_plan *out, int *bins /* n_channels */);

/* ======================================================================== rx_fm channels of one capture on several GPUs
 * The channels of ONE capture split over GPUs: one process, n_dev rxb200_fm_mix handles, member i owning the contiguous
 * channels [b, e) that rxb200_power_shard(n_channels, n_dev, i, &b, &e) gives, with offsets offsets_hz[b..e).  A member
 * whose range is empty has no handle.  devices == NULL means 0..n_dev-1; an ordinal may repeat (several members on one
 * GPU).  Every member gets its own copy of the capture (4 bytes per complex sample) and mixes and demodulates only its
 * channels, so a call's mixer writes and chain work, which grow with the channel count, split over the GPUs.
 * The group behaves byte for byte like ONE rxb200_fm_mix handle with n_channels channels: the same pcm, n_pcm,
 * chunk_result_len, squelch hits, levels ([n_channels][n_chunks]) and refusal codes, over any sequence of process,
 * process_read and reset calls.  cs16 and pcm are HOST pointers laid out as for rxb200_fm_mix_process (the one capture
 * at cs16, channel k's PCM at pcm + k*pcm_stride).  Create checks every channel's table (rxb200_fm_mix_table) before it
 * creates any member: a bad offset on any channel gets the code rxb200_fm_mix_create returns, before any device is
 * touched.  A call refused for its shape or capacity is refused before any member starts and moves no member's phases
 * and carries.  Each member copies the whole capture to its GPU, runs rxb200_fm_mix_process_device / _read_device and
 * copies its PCM rows back, all on its own stream; the call returns when every member that started is done, also after
 * a failure, and leaves the caller's current device as it found it.  A call that fails after members started
 * (RXB200_ECUDA, RXB200_ENOMEM) may leave the members at different phases and carries; rxb200_fm_mix_group_reset brings
 * every member back to the state right after create.  The capture copies of different GPUs overlap only with a pinned
 * (page-locked) capture: from pageable memory the N copies run one after the other and only the kernels overlap them
 * (the bytes are the same either way). */
typedef struct rxb200_fm_mix_group rxb200_fm_mix_group;
int rxb200_fm_mix_group_create(const rxb200_fm_params *params, int capture_rate, const int *offsets_hz, int n_channels,
                               int n_dev, const int *devices, rxb200_fm_mix_group **out);
/* The same with decimating members (rxb200_fm_mix_create_ddc), all sharing one rxb200_ddc: the group behaves like ONE
 * decimating handle with every channel, and every member checks a call's refusals on the decimated shape it will see.
 * The ddc is checked before the offsets. */
int rxb200_fm_mix_group_create_ddc(const rxb200_fm_params *params, int capture_rate, const int *offsets_hz,
                                   int n_channels, const rxb200_ddc *ddc, int n_dev, const int *devices,
                                   rxb200_fm_mix_group **out);
void rxb200_fm_mix_group_destroy(rxb200_fm_mix_group *g);
int rxb200_fm_mix_group_size(const rxb200_fm_mix_group *g);
/* member i's mixing handle (its channels are channel 0.. of that handle), NULL for a member that owns no channel */
rxb200_fm_mix *rxb200_fm_mix_group_member(rxb200_fm_mix_group *g, int i);
int rxb200_fm_mix_group_process(rxb200_fm_mix_group *g, const int16_t *cs16, size_t n_int16, size_t chunk_int16,
                                int16_t *pcm, size_t pcm_stride, size_t *n_pcm, int *chunk_result_len);
int rxb200_fm_mix_group_process_read(rxb200_fm_mix_group *g, const int16_t *cs16, size_t n_int16, int16_t *pcm,
                                     size_t pcm_stride, size_t *n_pcm);
int rxb200_fm_mix_group_squelch_hits(rxb200_fm_mix_group *g, int *hits /* n_channels */);
int rxb200_fm_mix_group_levels(rxb200_fm_mix_group *g, int *levels, size_t cap, size_t *n_chunks);
/* every member's phases back to 0 and its chain back to the state right after create */
int rxb200_fm_mix_group_reset(rxb200_fm_mix_group *g);

/* ======================================================================== rx_power hops of one capture
 * Every hop of a sweep from ONE wideband CS16 capture, instead of a retune and a read per hop (DESIGN.md section 4.5).
 * A power mixing handle has a capture rate R (Hz, > 0), one integer offset f_i per hop with |f_i| < R/2, one rxb200_ddc
 * (M, T taps h, shift S; the ranges of rxb200_fm_mix_create_ddc) and the rxb200_power_params, window and sine table of
 * rxb200_power_create.
 * NCO.  Frequency word w_i = floor((f_i 2^32 + floor(R/2)) / R) mod 2^32, exact in 64-bit integers (floor, also for
 * negative f).  Capture sample n, counted from create or reset across calls, has phase theta = n w_i mod 2^32 and table
 * index j = ((theta + 2^15) mod 2^32) >> 16.  One shared table of 2^16 entries (rxb200_nco_table) holds
 * (c_j, s_j) = ((int)round(32768 cos t), (int)round(32768 sin t)), t = -2 pi j' / 65536 in fp64, j' the representative
 * of j in (-32768, 32768], so the entries of j and 65536 - j are exact conjugates.  Mixing is the rx_fm mixer's rule:
 *     I' = (int16)((I c - Q s + 2^14) >> 15),  Q' = (int16)((I s + Q c + 2^14) >> 15)   (arithmetic shift, int16 wrap).
 * f = 0 is the identity, f = +-R/4 with 4 | R an exact quarter turn; no period limit, and the frequency error is at
 * most R / 2^33.
 * Filter.  z_i = mix_i(x), z_i[n] = 0 for n < 0.  Output m is emitted at e_m = m M + M - 1:
 *     A = sum_{j<T} h[j] z_i[e_m - j] (exact);  y = S ? (A + 2^(S-1)) >> S : A;  saturated to int16
 * (the rule of rxb200_fm_mix_create_ddc word for word).
 * Passes.  With B = buf_len / 2, outputs [p B, (p+1) B) of hop i are hop i's buffer in pass p, counted from create or
 * reset.  A call must cover whole passes: n_int16 a multiple of M * buf_len (else RXB200_EUNSUPPORTED, and nothing
 * changes); n_int16 == 0 is a no-op.  A call of P passes accumulates exactly what
 * rxb200_power_accumulate(member, bufs, P, 0, n_hops) would with bufs[p][i] = pass p of hop i.  power_ddc_kernel writes
 * those buffers pass-major into a scratch buffer of the handle, which a long call fills in groups of passes of at most
 * RXB200_POWER_MIX_SCRATCH_BYTES (at least one pass per group); the bytes are the same as with one group. */
#define RXB200_POWER_MIX_SCRATCH_BYTES (64u << 20)
typedef struct rxb200_power_mix rxb200_power_mix;
/* Refusals, all before any device is touched: those of rxb200_power_create for the params; RXB200_EINVAL for NULL
 * offsets, R <= 0 or any |f_i| >= R/2; those of rxb200_fm_mix_create_ddc for the ddc. */
int rxb200_power_mix_create(const rxb200_power_params *params, const int *window_coefs, const int16_t *sinewave,
                            int capture_rate, const int *offsets_hz /* n_hops */, const rxb200_ddc *ddc,
                            int device, rxb200_power_mix **out);
void rxb200_power_mix_destroy(rxb200_power_mix *m);
/* The inner rxb200_power handle, for rxb200_power_read / _read_db / _reset / _last_path / _kernel_ms / _stream (the DDC
 * runs on its stream).  rxb200_power_reset on it zeroes only the accumulators (csv_dbm's side effect): the phases and
 * the filter history carry on, since a capture stream is continuous across reports. */
rxb200_power *rxb200_power_mix_member(rxb200_power_mix *m);
/* Back to the state right after create: phases, filter history, pass count and accumulators. */
int rxb200_power_mix_reset(rxb200_power_mix *m);
/* cs16: HOST pointer to n_int16 int16 of the capture. */
int rxb200_power_mix_accumulate(rxb200_power_mix *m, const int16_t *cs16, size_t n_int16);
/* Same with a DEVICE capture (4-byte aligned), asynchronous on the member's stream unless sync != 0. */
int rxb200_power_mix_accumulate_device(rxb200_power_mix *m, const int16_t *d_cs16, size_t n_int16, int sync);
/* Device time (CUDA events on the member's stream) of the DDC launches of the last call, summed, in milliseconds;
 * synchronises. */
int rxb200_power_mix_kernel_ms(rxb200_power_mix *m, float *ms);
/* The NCO table: 2 * 65536 int32, (c, s) pairs. */
int rxb200_nco_table(int32_t *table);
/* The DDC alone on DEVICE pointers, stateless, on `stream`: the samples before d_src are zero, d_src[i] is capture
 * sample n0 + i for the NCO of (R, f), and floor(n_complex / M) outputs go to d_dst, e_m counted from d_src.  Both
 * pointers 4-byte aligned.  Asynchronous. */
int rxb200_power_ddc_device(int capture_rate, int offset_hz, unsigned long long n0, const rxb200_ddc *ddc,
                            const int16_t *d_src, size_t n_complex, int16_t *d_dst, void *stream);
/* The channel filter the rx_power shell's capture mode uses: a Blackman-windowed sinc with cutoff 1/(2M) cycles per
 * sample over T taps (odd, 1..8191), quantised to round(2^shift g_j / sum g) (shift 0..30) with the centre tap
 * corrected so that sum h = 2^shift exactly.  Pure host arithmetic. */
int rxb200_ddc_lowpass(int decim, int n_taps, int shift, int32_t *taps);

/* ---- wide sweeps in tiles (DESIGN.md section 4.5, "Wide sweeps in tiles")
 * A sweep wider than one capture is cut into tiles of consecutive hops; the radio is tuned once per tile and the tile's
 * hops are taken from one burst, a fresh capture after the retune.  The tiling of a plan for captures of at most
 * max_capture_rate Hz, with r = plan->rate, s = freq_step, F0 = first_freq and n = n_hops:
 *   Mcap = min(4096, floor(min(max_capture_rate, 2^31 - 1) / r)); Mcap < 1 is refused (RXB200_EINVAL).
 *   A run of k hops is centred at its first hop plus c(k) = floor((k - 1) s / 2) and needs
 *   Mreq(k) = ceil((2 max(c(k), (k - 1) s - c(k)) + r) / r), the capture mode's rule for the same hops.
 *   hmax is the largest k <= n with Mreq(k) <= Mcap (k = 1 always fits).
 *   n_tiles = ceil(n / hmax), h = ceil(n / n_tiles): no tile is empty, since (n_tiles - 1) h <= (n_tiles - 1) hmax < n.
 *   M = Mreq(h), R = M r, T = min(8191, 32 M + 1).
 *   Tile t holds hops [t h, min((t+1) h, n)) and is centred at F0 + t h s + c(len_t); hop i's offset is its frequency
 *   minus its tile's centre, so |f_i| < R/2.
 * With one tile this is exactly the centre, offsets, M, R and T of the shell's capture mode.  Pure host arithmetic. */
typedef struct rxb200_power_tiling {
	int n_tiles;
	int hops_per_tile;   /* h: tile t holds hops [t h, min((t+1) h, n_hops)) */
	int decim;           /* M */
	int n_taps;          /* T = min(8191, 32 M + 1), the capture mode's filter length */
	int capture_rate;    /* R = M * plan->rate */
} rxb200_power_tiling;
/* offsets_hz: n_hops ints, each hop's offset from its tile's centre, or NULL.  RXB200_EINVAL for NULL plan or out, a
 * plan with n_hops < 1, rate < 1 or freq_step < 0, and Mcap < 1. */
int rxb200_power_plan_tiles(const rxb200_power_plan *plan, long long max_capture_rate,
                            rxb200_power_tiling *out, int *offsets_hz /* n_hops, may be NULL */);
/* Tile t's hop range and centre (Hz); RXB200_EINVAL for a NULL argument or t outside [0, n_tiles). */
int rxb200_power_tile(const rxb200_power_plan *plan, const rxb200_power_tiling *tl, int t,
                      int *hop_begin, int *hop_end, int64_t *centre_hz);
/* Bursts.  A burst is one self-contained capture, not a continuation of the handle's stream: n_int16 = 2G + P M buf_len
 * int16 with P >= 1, where the lead G = M ceil((T - 1) / M) complex samples (rxb200_power_mix_lead) primes the filter.
 * Any other length is RXB200_EUNSUPPORTED; a hop range other than 0 <= hb < he <= n_hops, a NULL pointer or a device
 * pointer that is not 4-byte aligned is RXB200_EINVAL; a refused call changes nothing.
 * For hop i in [hb, he), n counts from the burst's first sample (the lead included) and z_i is the NCO rule above at
 * that n.  Output m is emitted at e_m = G + m M + M - 1 with the filter rule above word for word; every index it reads
 * is >= 0, so no zeros enter.  Outputs [p B, (p+1) B) are pass p of hop i, and the call accumulates what
 * rxb200_power_accumulate(member, bufs, P, hb, he) would.  Equivalently they are outputs G/M + u of
 * rxb200_power_ddc_device(R, f_i, 0, ddc, burst, n_complex).  A burst neither reads nor moves the handle's sample count
 * or filter history: continuous rxb200_power_mix_accumulate calls before and after it see one unbroken stream.
 * The offsets at create may be relative to different tile centres; create's rule |f_i| < R/2 is unchanged. */
int rxb200_power_mix_lead(const rxb200_power_mix *m);   /* G, or RXB200_EINVAL for NULL */
/* cs16: HOST pointer to the burst, staged through the handle's device buffer; synchronous. */
int rxb200_power_mix_accumulate_burst(rxb200_power_mix *m, int hop_begin, int hop_end,
                                      const int16_t *cs16, size_t n_int16);
/* Same with a DEVICE burst (4-byte aligned), asynchronous on the member's stream unless sync != 0. */
int rxb200_power_mix_accumulate_burst_device(rxb200_power_mix *m, int hop_begin, int hop_end,
                                             const int16_t *d_cs16, size_t n_int16, int sync);

/* ======================================================================== rx_sdr (SURVEY.md §8f row 4)
 * The pointwise sample-format conversions of rx_sdr's recorder loop (src/rtl_sdr.c:348-391):
 *   RXB200_CVT_CS16_CS8  : (uint8_t)(int)(x/32767.0*128.0+0.4)       per int16 (:367-370)
 *   RXB200_CVT_CS16_CU8  : (uint8_t)(x/32767.0*128.0+127.4)           per int16 (:375-378)
 *   RXB200_CVT_CS16_CF32 : x * 1.0f / SHRT_MAX                        per int16 (:383-386)
 *   RXB200_CVT_CS12_CS16 : 3 packed bytes -> (I, Q) int16             per complex element (:354-362)
 * and the widening of a device's 8-bit formats, the input stage of the capture handles ("capture handles in a device's
 * own format" below), exact, per byte b:
 *   RXB200_CVT_CS8_CS16  : (int16)((int8)b << 8)
 *   RXB200_CVT_CU8_CS16  : (int16)(((int)b - 128) << 8)
 * (4 is RXB200_SDR_OUT_CS16, an rx_sdr output format, and no conversion.)
 * n_elems counts COMPLEX elements.  Host pointers; bandwidth-bound, one kernel. */
#define RXB200_CVT_CS16_CS8  0
#define RXB200_CVT_CS16_CU8  1
#define RXB200_CVT_CS16_CF32 2
#define RXB200_CVT_CS12_CS16 3
#define RXB200_CVT_CS8_CS16  5
#define RXB200_CVT_CU8_CS16  6
int rxb200_sdr_convert(int kind, const void *src, size_t n_elems, void *dst, int device);
/* Same with device pointers on `stream` (a cudaStream_t, may be NULL).  Asynchronous.  Alignment, else RXB200_EINVAL
 * before any CUDA call:
 *   RXB200_CVT_CS16_CS8, _CS16_CU8, _CS16_CF32 : d_src and d_dst 16-byte aligned
 *   RXB200_CVT_CS12_CS16, _CS8_CS16, _CU8_CS16 : d_dst 4-byte aligned (one 32-bit store per element); d_src any (16-byte
 *                                                vectors when both are 16-byte aligned) */
int rxb200_sdr_convert_device(int kind, const void *d_src, size_t n_elems, void *d_dst, void *stream);

/* ---- rx_sdr channels of one capture (DESIGN.md section 4.6)
 * An I/Q down-converter handle records C channels of ONE wideband CS16 capture at rate R (Hz), channel c at an integer
 * offset f_c with |f_c| < R/2, each as its own decimated stream in a recorded format.  Indices n count capture samples
 * from create or reset across calls.  It has one of three front stages:
 *   Single stage (rxb200_sdr_mix_create, one rxb200_ddc (M, T, h, S)): channel c is the rx_power NCO rule of
 *     "rx_power hops of one capture" (word w_c, rxb200_nco_table, the mixer's rounding and wrap) followed by the filter
 *     rule: output q is output q of rxb200_power_ddc_device(R, f_c, 0, ddc, .) over the whole capture since create or
 *     reset.  The NCO has no period limit, so any integer offset works.
 *   Two stages (rxb200_sdr_mix_create_two_stage, K bins, coarse d1 and fine d2, M = M1 M2): channel c is the rule of
 *     "two-stage mixing handles": output q is output q of rxb200_two_stage_device at n0 = 0 over the whole capture.
 *   Raster (rxb200_sdr_mix_create_raster, K bins, channel c bin k_c, one rxb200_ddc (M, T, h, S)): channel c is the rule
 *     of "raster mixing handles": output q is output q of rxb200_raster_device(K, bins, 0, ddc, .) over the whole
 *     capture.  Channel c sits at k_c R / K for whatever capture rate R the capture has; the handle needs none.  Its
 *     DFT's epilogue (raster_dft_kernel) writes the format.
 * The rule.  Output q of channel c is the stateless rule's output q over the concatenated capture since create or
 * reset, so the bytes never depend on how the capture is cut into calls.  A call covering capture samples [n0, n0 + n)
 * returns the floor((n0 + n) / M) - floor(n0 / M) outputs emitted in it (rxb200_sdr_mix_decimated_len); any even
 * n_int16 is accepted, including calls with no output, which still advance the count and the histories.
 * Formats.  format RXB200_SDR_OUT_CS16 writes the rule's int16 I/Q pairs (4 bytes per output); RXB200_CVT_CS16_CS8,
 * _CU8 (2 bytes) and _CF32 (8 bytes) write rx_sdr's conversion of that int16 exactly as rxb200_sdr_convert defines it.
 * The kernels write the format directly, with no CS16 pass in between.  Rows are channel-major: channel c's call
 * output q is element c * out_stride + q of out, an output buffer of out_cap elements.
 * Refusals, all before anything is enqueued, and a refused call changes nothing: RXB200_EINVAL for a NULL handle,
 * capture or output, a bad format, odd n_int16, out_stride above RXB200_SDR_MIX_MAX_STRIDE, and (device entry) a capture
 * that is not 4-byte aligned or an output not aligned to min(element, 4) bytes; RXB200_ECAPACITY when out_stride or
 * out_cap is too small for the call's outputs (out_stride >= n_out, (C - 1) out_stride + n_out <= out_cap).
 * The handle carries the capture count and the histories (the filter's last T - 1 raw samples, or the coarse stage's
 * raw history and each bin's fine history), and a call's next histories become live only when it succeeds.  A host
 * call stages its capture and outputs through the device in groups of at most RXB200_SDR_MIX_SCRATCH_BYTES, each group
 * a device call of its own that commits its count and histories when it succeeds (so a CUDA failure in a later group
 * leaves the earlier groups' outputs written and their state live; reset starts over), and a
 * two-stage or raster call runs its (coarse) frames in groups under RXB200_RASTER_SCRATCH_BYTES; the bytes are the
 * same as with one group. */
#define RXB200_SDR_OUT_CS16 4
#define RXB200_SDR_MIX_SCRATCH_BYTES (64u << 20)
#define RXB200_SDR_MIX_MAX_STRIDE (1u << 30)
typedef struct rxb200_sdr_mix rxb200_sdr_mix;
/* Refusals, all before any device is touched: RXB200_EINVAL for NULL offsets or out, n_channels < 1, R <= 0 or any
 * |f_c| >= R/2; those of rxb200_fm_mix_create_ddc for the ddc. */
int rxb200_sdr_mix_create(int capture_rate, const int *offsets_hz /* n_channels */, int n_channels,
                          const rxb200_ddc *ddc, int device, rxb200_sdr_mix **out);
/* Refusals, all before any device is touched: those of rxb200_fm_mix_create_two_stage but the params'. */
int rxb200_sdr_mix_create_two_stage(int capture_rate, int n_bins, const int *offsets_hz /* n_channels */,
                                    int n_channels, const rxb200_ddc *coarse, const rxb200_ddc *fine, int device,
                                    rxb200_sdr_mix **out);
/* Refusals, all before any device is touched: RXB200_EINVAL for NULL out; those of rxb200_raster_device for K, bins
 * and the ddc (K outside [3, 4096], NULL bins, n_channels < 1, a bin outside [0, K), the ddc's own, sum |h| >= 2^22). */
int rxb200_sdr_mix_create_raster(int n_bins, const int *bins /* n_channels */, int n_channels, const rxb200_ddc *ddc,
                                 int device, rxb200_sdr_mix **out);
void rxb200_sdr_mix_destroy(rxb200_sdr_mix *m);
/* the count and every history back to the state right after create */
int rxb200_sdr_mix_reset(rxb200_sdr_mix *m);
/* *n_out: the outputs per channel the next call of n_int16 capture int16 returns */
int rxb200_sdr_mix_decimated_len(const rxb200_sdr_mix *m, size_t n_int16, size_t *n_out);
/* HOST capture and output; synchronous.  *n_out (may be NULL) receives the outputs per channel. */
int rxb200_sdr_mix_process(rxb200_sdr_mix *m, const int16_t *cs16, size_t n_int16, int format, void *out,
                           size_t out_cap, size_t out_stride, size_t *n_out);
/* DEVICE capture and output, asynchronous on the handle's stream unless sync != 0. */
int rxb200_sdr_mix_process_device(rxb200_sdr_mix *m, const int16_t *d_cs16, size_t n_int16, int format, void *d_out,
                                  size_t out_cap, size_t out_stride, size_t *n_out, int sync);
/* Device time (CUDA events on the handle's stream) of the down-converter kernels of the last call (of a host call's
 * last group), in milliseconds; synchronises. */
int rxb200_sdr_mix_kernel_ms(rxb200_sdr_mix *m, float *ms);
/* the handle's cudaStream_t */
void *rxb200_sdr_mix_stream(rxb200_sdr_mix *m);
/* The plan of the rx_sdr shell's capture mode for K tuned frequencies t_k (Hz) and a per-channel rate s (rx_sdr's -s):
 * the rule of rxb200_fm_plan_capture with c = s (fc, o_k, M, R = M s, T = min(8191, 32 M + 1), the filter
 * rxb200_ddc_lowpass(M, T, 15) at S = 15) and its refusals, but no offset is refused for a mixer table's period, since
 * the handle mixes with the NCO.  The two-stage plan is rxb200_fm_plan_capture_two_stage and the raster plan
 * rxb200_fm_plan_capture_raster, each with chain rate s. */
int rxb200_sdr_plan_capture(const int64_t *tuned_hz /* n_channels */, int n_channels, int sample_rate,
                            long long max_capture_rate, rxb200_fm_capture_plan *out, int *offsets_hz /* n_channels */);

/* ======================================================================== capture from a device at its own rate
 * (DESIGN.md section 4.7)  Every capture plan above asks the device for exactly R = M c.  Many receivers run only at a
 * few fixed rates, or round what they are asked for; a device that delivers R' != R moves every channel by
 * o (1 - R'/R) and scales the chain rate by R'/R.  A rational resampler takes the device's stream at the rate it really
 * runs at, R_dev, to the plan's R exactly, so every front stage above runs unchanged on its output.
 * The rule.  A resampler has an up factor L and a down factor N (R / R_dev = L / N, 1 <= L, N), J taps per phase
 * (1..1024, J L <= 2^22), a prototype h of J L int32 taps and a rounding shift S (0..62).  Let x[n] be the device's
 * CS16 samples, n counted from create or reset across calls, x[n] = 0 for n < 0.  For output m >= 0:
 *     t = m N,  q = floor(t / L),  p = t mod L;
 *     A = sum_{j<J} h[p + j L] x[q - j]   (exact, I and Q separately);
 *     y = S ? (A + 2^(S-1)) >> S : A   (arithmetic), saturated to [-32768, 32767].
 * Output m is emitted by device sample q.  A call over device samples [n0, n0 + c) returns the
 * ceil((n0 + c) L / N) - ceil(n0 L / N) outputs whose q falls in it (computed in 128-bit integers: no count wraps), so
 * the bytes never depend on how the stream is cut into calls.
 * Anchors.  L = N = 1, J = 1, h = {2^15}, S = 15 is the identity.  L = 1, N = M: output m is output m of
 * rxb200_ddc_device at offset 0 with the same M, taps and shift over the stream with M - 1 zeros prepended (the DDC
 * emits at m M + M - 1, this rule at m M).
 * resample_kernel accumulates in int32 when max_p sum_j |h[p + j L]| * 32768 + 2^(S-1) < 2^31, else in int64.  A CTA
 * owns consecutive outputs, stages the device samples they read once in shared memory, and holds the taps phase-major
 * ([L][J]) in shared memory when they fit (J L <= 12288), else reads them through the caches. */
typedef struct rxb200_resampler {
	int up;                /* L */
	int down;              /* N */
	int taps_per_phase;    /* J */
	const int32_t *taps;   /* h[0..J L), the prototype at rate L R_dev: phase p is h[p], h[p + L], ..., h[p + (J-1) L] */
	int shift;             /* S */
} rxb200_resampler;
/* The prototype filter: a Blackman-windowed sinc of J L taps at the prototype rate L R_dev, cutoff 1 / (2 max(L, N))
 * cycles per prototype sample (min(R, R_dev) / 2 Hz), scaled so that each phase sums to about 2^15 and rounded; then
 * each phase's sum is corrected to exactly 2^15 on that phase's largest-magnitude tap (the first of equals), so at
 * S = 15 a constant input comes out exactly constant once q >= J - 1.  Window w_i = 0.42 - 0.5 cos a + 0.08 cos 2a,
 * a = 2 pi (i + 1) / (J L + 1).  RXB200_EINVAL for NULL taps, L or N < 1, J outside [1, 1024] or J L > 2^22.  Pure host
 * arithmetic. */
int rxb200_resample_lowpass(int up, int down, int taps_per_phase, int32_t *taps /* J L */);
/* The resampler from a device rate R_dev to a plan's rate R for channels spanning `span` Hz around the centre (2A + c,
 * A the largest |offset|, c the chain rate):
 *   G = ceil(R_dev / 32), the guard band the transition needs; D = min(R, R_dev) - span, refused when D < G
 *     (RXB200_EINVAL; the message names the span, R_dev and the largest span that fits, min(R, R_dev) - G);
 *   L = R / gcd(R, R_dev), N = R_dev / gcd(R, R_dev);  J = 8 ceil(ceil(6 R_dev / D) / 8), so 8 <= J <= 192;
 *   J L > 2^22 is refused (RXB200_EUNSUPPORTED, the message names L/N);  S = 15, taps rxb200_resample_lowpass(L, N, J).
 * out->taps is set to NULL: the caller designs the J L taps.  L = N = 1 means no resampler is needed.  Also
 * RXB200_EINVAL for a NULL out, a rate outside [1, 2^31 - 1] or a negative span.  Pure host arithmetic.
 * Worked examples.  span = 2A + c, and R = M c with M = ceil((2A + c + G) / c): the decimation a capture plan needs so
 * that the guard band fits (the capture planners above choose M = ceil((2A + c) / c), which leaves no room for it on
 * these sets; DESIGN.md section 4.7):
 *   set                                          R_dev        M, R             L/N          J     J L
 *   7 NOAA channels, rx_fm NBFM (c = 1.008 M)    2.4 M        2, 2.016 M       21/25        24    504
 *   the same                                     2.5 M        2, 2.016 M       504/625      24    12 096
 *   100 FM stations, wbfm (c = 1.02 M)           30.72 M      22, 22.44 M      187/256      136   25 432
 *   the same                                     20 M         refused: span 21.02 MHz > 20 M - 625 k
 *   4 rx_sdr channels 100-100.95 MHz, -s 250k    2.4 M        6, 1.5 M         5/8          48    240
 *   100 FM stations, rx_sdr raster, -s 250k      30.72 M      85, 21.25 M      2125/3072    192   408 000 */
int rxb200_plan_resample(long long device_rate, long long rate, long long span, rxb200_resampler *out);
/* A resampler handle carries the device-sample count and the last J - 1 raw samples between calls; a call's next
 * history and count become live only when it succeeds, and a refused call changes nothing.  Refusals of create, all
 * before any device is touched: RXB200_EINVAL for a NULL resampler, taps or out, L or N < 1, J outside [1, 1024],
 * J L > 2^22, S outside [0, 62] and max_p sum |h_p| * 32768 + 2^(S-1) >= 2^63 (which the other bounds already keep
 * below 2^62).  The taps are copied. */
#define RXB200_RESAMPLE_SCRATCH_BYTES (64u << 20)
typedef struct rxb200_resample rxb200_resample;
int rxb200_resample_create(const rxb200_resampler *rs, int device, rxb200_resample **out);
void rxb200_resample_destroy(rxb200_resample *r);
/* the count and the history back to the state right after create */
int rxb200_resample_reset(rxb200_resample *r);
/* *n_out: the outputs the next call of n_int16 device int16 returns */
int rxb200_resample_out_len(const rxb200_resample *r, size_t n_int16, size_t *n_out);
/* HOST stream and output, synchronous: n_int16 int16 (even) in, *n_out (may be NULL) complex outputs to out, which
 * holds out_cap complex outputs.  RXB200_EINVAL for a NULL handle, stream or output or an odd n_int16;
 * RXB200_ECAPACITY when out_cap is below the call's outputs.  The call stages the stream through the device in groups
 * of at most RXB200_RESAMPLE_SCRATCH_BYTES, each a device call that commits its count and history when it succeeds;
 * the bytes are those of one group. */
int rxb200_resample_process(rxb200_resample *r, const int16_t *cs16, size_t n_int16, int16_t *out, size_t out_cap,
                            size_t *n_out);
/* The same on DEVICE pointers (both 4-byte aligned, else RXB200_EINVAL), asynchronous on the handle's stream unless
 * sync != 0. */
int rxb200_resample_process_device(rxb200_resample *r, const int16_t *d_cs16, size_t n_int16, int16_t *d_out,
                                   size_t out_cap, size_t *n_out, int sync);
/* the handle's cudaStream_t */
void *rxb200_resample_stream(rxb200_resample *r);
/* Device time (CUDA events on the handle's stream) of the resample_kernel launches of the last call (of a host call's
 * last group), in milliseconds; synchronises. */
int rxb200_resample_kernel_ms(rxb200_resample *r, float *ms);
/* The resampler alone on DEVICE pointers, stateless, on `stream`: d_src[i] is device sample n0 + i, the samples before
 * d_src are zero, and the ceil((n0 + n_complex) L / N) - ceil(n0 L / N) outputs whose q falls in
 * [n0, n0 + n_complex) go to d_dst.  Both pointers 4-byte aligned.  The refusals of rxb200_resample_create.
 * Asynchronous. */
int rxb200_resample_device(const rxb200_resampler *rs, unsigned long long n0, const int16_t *d_src, size_t n_complex,
                           int16_t *d_dst, void *stream);
/* The fewest device samples c that a call starting at device sample n0 needs for n_out outputs: the least c with
 * ceil((n0 + c) L / N) - ceil(n0 L / N) >= n_out (0 for n_out = 0), computed in 128-bit integers.  Output m is emitted
 * by device sample floor(m N / L), so c = floor((m0 + n_out - 1) N / L) + 1 - n0 with m0 = ceil(n0 L / N).  When L <= N
 * each device sample emits at most one output, so the call's count is exactly n_out: a reader that needs one block of
 * n_out capture samples reads exactly c device samples.  RXB200_EINVAL for NULL n_in, L or N < 1, or c >= 2^64.  Pure
 * host arithmetic. */
int rxb200_resample_in_len(int up, int down, unsigned long long n0, size_t n_out, size_t *n_in);

/* ---- capture handles at a device rate (DESIGN.md section 4.7)
 * rxb200_fm_mix_set_device_rate, rxb200_sdr_mix_set_device_rate and rxb200_power_mix_set_device_rate attach a resampler
 * (the rule above) to a capture handle of any kind, ahead of its front stage.  After the call every host and device
 * entry of the handle takes device-rate CS16: the handle's capture is the resampler's output over the device stream
 * since create or reset, and a call over device samples [n0, n0 + c) hands the front the ceil((n0 + c) L / N) -
 * ceil(n0 L / N) capture samples those device samples emit.  So a handle's bytes are exactly those of an
 * rxb200_resample handle followed by the same handle without a resampler on its output, however the device stream is
 * cut into calls.  What follows the device-sample count:
 *   rxb200_fm_mix: a call's shape is that of its capture samples (a read is one read of them; a chunked call's
 *     chunk_int16 counts capture int16 as before); _decimated_len and _max_output take device int16;
 *   rxb200_sdr_mix: _decimated_len takes device int16; a host call stages device samples in groups whose device-rate
 *     upload, resampled capture and output rows together fit RXB200_SDR_MIX_SCRATCH_BYTES;
 *   rxb200_power_mix: a call must resample to whole passes (else RXB200_EUNSUPPORTED, and nothing changes); bursts,
 *     capture-rate captures of their own, are refused (RXB200_EUNSUPPORTED): device-rate bursts take
 *     rxb200_power_mix_set_burst_device_rate instead;
 *   every handle: reset clears the resampler's count and history and keeps it attached; a refused call changes nothing;
 *     _kernel_ms includes resample_kernel; an odd n_int16 gets the code the handle gives it without a resampler
 *     (RXB200_EUNSUPPORTED for rx_fm and rx_power, RXB200_EINVAL for rx_sdr).
 * The resampler runs on the handle's stream into a capture-rate scratch buffer in device memory (4 bytes per capture
 * sample of a call, or of a host call's group).  rx_fm and rx_sdr commit its history and count with the front's, per
 * call or per host group.  rx_power resamples a whole call ahead of its pass groups and commits the resampler once
 * that is enqueued, before the groups commit theirs; a CUDA failure in a later group (RXB200_ECUDA) therefore leaves
 * the resampler's count ahead of the passes taken, and rxb200_power_mix_reset starts over, as after any failed call.
 * Refusals: RXB200_EINVAL for a NULL handle, or a handle that has taken any sample since create or reset or already has
 * a resampler; then those of rxb200_resample_create.  All come before any device work.  The taps are copied. */
int rxb200_fm_mix_set_device_rate(rxb200_fm_mix *m, const rxb200_resampler *rs);
int rxb200_sdr_mix_set_device_rate(rxb200_sdr_mix *m, const rxb200_resampler *rs);
int rxb200_power_mix_set_device_rate(rxb200_power_mix *m, const rxb200_resampler *rs);

/* ---- capture handles in a device's own format (DESIGN.md section 4.8)
 * Many receivers deliver narrower samples than CS16: 8-bit signed I/Q (CS8), 8-bit unsigned (CU8) or packed 12-bit
 * (CS12).  rxb200_fm_mix_set_input_format, rxb200_sdr_mix_set_input_format and rxb200_power_mix_set_input_format make
 * every host and device entry of a capture handle of any kind (stream calls and bursts alike) take that format.  Each
 * element is widened to one CS16 pair exactly, with no rounding:
 *   RXB200_IN_CS16 : 4 bytes, unchanged (the default)
 *   RXB200_IN_CS8  : 2 bytes, I and Q = (int16)((int8)b << 8)          (RXB200_CVT_CS8_CS16)
 *   RXB200_IN_CU8  : 2 bytes, I and Q = (int16)(((int)b - 128) << 8)   (RXB200_CVT_CU8_CS16)
 *   RXB200_IN_CS12 : 3 bytes b0 b1 b2, I = (int16)((b1 << 12) | (b0 << 4)), Q = (int16)((b2 << 8) | (b1 & 0xf0))
 *                    (RXB200_CVT_CS12_CS16)
 * A handle fed bytes b in format F gives exactly the bytes it gives when fed the widening of b as CS16, however the
 * stream is cut into calls: the widening runs on the handle's stream into a CS16 scratch buffer in device memory (4
 * bytes per sample of a call, or of a host call's group), ahead of everything else, and the resampler (when attached)
 * and the front stage run on it unchanged.  A driver's own CS16 conversion (an RTL driver's lookup table, say) may
 * differ from this rule; the handle matches the widened stream, not any driver.
 * Lengths keep their meaning: n_int16 counts I and Q components, two per complex element, so a call's buffer holds
 * n_int16 / 2 elements of the format (n_int16 bytes for CS8 and CU8, 3 n_int16 / 2 bytes for CS12), passed as the same
 * const int16_t * (callers cast).  Every length helper (_max_output, _decimated_len, _burst_in_len,
 * rxb200_resample_in_len) gives what it gives for CS16.  Device entries take a CS8, CU8 or CS12 capture at any byte
 * address (CS16 keeps its 4-byte rule).  Host entries copy only the format's bytes to the device; the groups of a host
 * call (RXB200_SDR_MIX_SCRATCH_BYTES, counting the upload and the widened samples) are cut at element boundaries, and
 * the bytes are the same as with one group.  Reset keeps the format.  The format and the resampler are independent:
 * set either first.  _kernel_ms includes the widening.
 * Refusals, before any device work: RXB200_EINVAL for a NULL handle or an unknown format, and RXB200_EINVAL for a
 * handle that has taken any sample since create or reset (as _set_device_rate).  A refused call changes nothing. */
#define RXB200_IN_CS16 0
#define RXB200_IN_CS8  1
#define RXB200_IN_CU8  2
#define RXB200_IN_CS12 3
int rxb200_fm_mix_set_input_format(rxb200_fm_mix *m, int fmt);
int rxb200_sdr_mix_set_input_format(rxb200_sdr_mix *m, int fmt);
int rxb200_power_mix_set_input_format(rxb200_power_mix *m, int fmt);

/* ---- capture plans at a device rate
 * The capture planners above with one more argument, the device rate R_dev (Hz) the shell's resampler starts from.
 * Each follows its own planner's rule, with one change: G = ceil(R_dev / 32), the guard band rxb200_plan_resample needs,
 * and the decimation floor leaves it, M = ceil((2 A + c + G) / c) instead of ceil((2 A + c) / c).  The centre, the
 * offsets, T, the raster's K and bins and the two-stage split M' = 4 ceil(M / 4) follow from that M as before, so
 * rxb200_plan_resample(R_dev, R, 2 A + c) fits whenever R <= R_dev.
 * Refusals, pure host arithmetic: RXB200_EINVAL for R_dev outside [1, 2^31 - 1], first; then every refusal of the
 * planner in its order (the arguments, the cap, 2^31 - 1 and the decimation bound, the two-stage M' < 8, the raster's
 * K > 4096, the mixer table's); and RXB200_EUNSUPPORTED for R > R_dev, right after the cap's refusal (the message names
 * R and R_dev): the shells only resample down.
 * Worked examples (each also in rxb200_plan_resample's table):
 *   set                                          planner    R_dev     M    R           resampler L/N
 *   7 NOAA channels, rx_fm NBFM (c = 1.008 M)    fm         2.4 M     2    2 016 000   21/25
 *   4 rx_sdr channels 100-100.95 MHz, -s 250k    sdr        2.4 M     6    1 500 000   5/8
 *   100 FM stations, wbfm (c = 1.02 M)           fm         30.72 M   22   22 440 000  187/256 */
int rxb200_fm_plan_capture_at(const int64_t *tuned_hz /* n_channels */, int n_channels, int chain_rate,
                              long long max_capture_rate, long long device_rate, rxb200_fm_capture_plan *out,
                              int *offsets_hz /* n_channels */);
int rxb200_fm_plan_capture_two_stage_at(const int64_t *tuned_hz /* n_channels */, int n_channels, int chain_rate,
                                        long long max_capture_rate, long long device_rate,
                                        rxb200_fm_two_stage_plan *out, int *offsets_hz /* n_channels */);
int rxb200_fm_plan_capture_raster_at(const int64_t *tuned_hz /* n_channels */, int n_channels, int chain_rate,
                                     long long max_capture_rate, long long device_rate, rxb200_fm_raster_plan *out,
                                     int *bins /* n_channels */);
int rxb200_sdr_plan_capture_at(const int64_t *tuned_hz /* n_channels */, int n_channels, int sample_rate,
                               long long max_capture_rate, long long device_rate, rxb200_fm_capture_plan *out,
                               int *offsets_hz /* n_channels */);

/* ---- rx_power plans at a device rate (DESIGN.md section 4.7)
 * The capture mode's plan, with r = plan->rate, s = freq_step, F0 = first_freq and n = n_hops: the centre
 * fc = F0 + floor((n - 1) s / 2), hop i's offset f_i = F0 + i s - fc, span = 2 max |f_i|, M = ceil((span + r) / r),
 * R = M r and T = min(32 M + 1, 8191), in out (centre_hz, decim, capture_rate, n_taps).  Refused (RXB200_EINVAL):
 * R > max_capture_rate, R > 2^31 - 1 or M > 4096, the message "the span needs a capture rate of R Hz"; a NULL plan or
 * out, n_hops < 1, rate < 1 or freq_step < 0.  offsets_hz (n_hops ints) may be NULL.  Pure host arithmetic. */
int rxb200_power_plan_capture(const rxb200_power_plan *plan, long long max_capture_rate, rxb200_fm_capture_plan *out,
                              int *offsets_hz /* n_hops, may be NULL */);
/* The same at a device rate R_dev, with the guard band G = ceil(R_dev / 32) of rxb200_plan_resample in the decimation
 * floor, M = ceil((span + r + G) / r), so rxb200_plan_resample(R_dev, R, span + r) fits whenever R <= R_dev.
 * Refusals: RXB200_EINVAL for R_dev outside [1, 2^31 - 1], first; then those of rxb200_power_plan_capture; then
 * RXB200_EUNSUPPORTED for R > R_dev (the message names R and R_dev). */
int rxb200_power_plan_capture_at(const rxb200_power_plan *plan, long long max_capture_rate, long long device_rate,
                                 rxb200_fm_capture_plan *out, int *offsets_hz /* n_hops, may be NULL */);
/* The tiling of rxb200_power_plan_tiles at a device rate R_dev: Mcap = min(4096, floor(min(max_capture_rate, R_dev,
 * 2^31 - 1) / r)) and Mreq(k) = ceil((2 max(c(k), (k - 1) s - c(k)) + r + G) / r), G = ceil(R_dev / 32); the rest of
 * that rule unchanged.  Tiles shrink until each fits: no tile runs above R_dev, and rxb200_plan_resample(R_dev, R,
 * 2 max(c, (len - 1) s - c) + r) fits every tile of len hops.  Refusals (RXB200_EINVAL): R_dev outside [1, 2^31 - 1],
 * first; those of rxb200_power_plan_tiles; and Mreq(1) > Mcap, a device too slow for a tile of one hop. */
int rxb200_power_plan_tiles_at(const rxb200_power_plan *plan, long long max_capture_rate, long long device_rate,
                               rxb200_power_tiling *out, int *offsets_hz /* n_hops, may be NULL */);
/* Bursts at a device rate.  rxb200_power_mix_set_burst_device_rate attaches a resampler (L, N, J taps per phase) for
 * bursts only, right after create or reset, on a handle without rxb200_power_mix_set_device_rate's resampler (the two
 * exclude each other; RXB200_EINVAL otherwise, then the refusals of rxb200_resample_create; the taps are copied).
 * After it, rxb200_power_mix_accumulate_burst and _accumulate_burst_device take DEVICE-rate bursts; the stream entries
 * (_accumulate, _accumulate_device) still take capture-rate samples, as before.
 * The burst rule.  A burst's capture is the stateless resampler rule over the burst's device samples, n0 = 0 with zeros
 * before the burst.  Its first E = ceil((J - 1) L / N) outputs, those whose window reaches before the burst, are
 * dropped, so no zeros enter; the remaining outputs must be exactly a capture-rate burst of the rule above, the lead G
 * plus P >= 1 whole passes (E + G + P M buf_len / 2 outputs), else RXB200_EUNSUPPORTED and nothing changes.  So the
 * call accumulates what rxb200_resample_device(rs, 0, burst) followed, from output E on, by the capture-rate burst
 * call would.  A burst still neither reads nor moves the handle's sample count or filter history. */
int rxb200_power_mix_set_burst_device_rate(rxb200_power_mix *m, const rxb200_resampler *rs);
/* *n_int16: the device int16 of one burst of `passes` passes: 2 rxb200_resample_in_len(L, N, 0, E + G + passes M
 * buf_len / 2), exact when L <= N (the planners only make such resamplers); on a handle without a burst device rate,
 * the capture-rate burst 2 G + passes M buf_len.  RXB200_EINVAL for a NULL argument or passes < 1. */
int rxb200_power_mix_burst_in_len(const rxb200_power_mix *m, int passes, size_t *n_int16);

#ifdef __cplusplus
}
#endif
#endif /* RXB200_H */
