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
 * unless sync != 0.  n_pcm is computed on the host (closed form) and valid at return. */
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
/* Device time (CUDA events on the handle's stream) of the last process call's main kernels, in
 * milliseconds: the split kernel on the row path, the fused kernel's main pass (not its per-chunk
 * reduction pre-passes), or the front and back kernels on the stream path.  Synchronises the stream. */
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

/* ======================================================================== rx_sdr (SURVEY.md §8f row 4)
 * The pointwise sample-format conversions of rx_sdr's recorder loop (src/rtl_sdr.c:348-391):
 *   RXB200_CVT_CS16_CS8  : (uint8_t)(int)(x/32767.0*128.0+0.4)       per int16 (:367-370)
 *   RXB200_CVT_CS16_CU8  : (uint8_t)(x/32767.0*128.0+127.4)           per int16 (:375-378)
 *   RXB200_CVT_CS16_CF32 : x * 1.0f / SHRT_MAX                        per int16 (:383-386)
 *   RXB200_CVT_CS12_CS16 : 3 packed bytes -> (I, Q) int16             per complex element (:354-362)
 * n_elems counts COMPLEX elements.  Host pointers; bandwidth-bound, one kernel. */
#define RXB200_CVT_CS16_CS8  0
#define RXB200_CVT_CS16_CU8  1
#define RXB200_CVT_CS16_CF32 2
#define RXB200_CVT_CS12_CS16 3
int rxb200_sdr_convert(int kind, const void *src, size_t n_elems, void *dst, int device);
/* Same with device pointers on `stream` (a cudaStream_t, may be NULL). */
int rxb200_sdr_convert_device(int kind, const void *d_src, size_t n_elems, void *d_dst, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* RXB200_H */
