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
 * post_downsample.  rxb200_fm_process_device wants d_cs16 32-byte aligned, or 4-byte aligned for
 * a call without passes whose chunk or length is not a multiple of 16 int16. */
int rxb200_fm_process(rxb200_fm *h, const int16_t *cs16, size_t n_int16, size_t chunk_int16,
                      int16_t *pcm, size_t pcm_stride, size_t *n_pcm, int *chunk_result_len);

/* Same with DEVICE pointers (inputs already resident in HBM); asynchronous on the handle's stream
 * unless sync != 0.  n_pcm is computed on the host (closed form) and valid at return. */
int rxb200_fm_process_device(rxb200_fm *h, const int16_t *d_cs16, size_t n_int16, size_t chunk_int16,
                             int16_t *d_pcm, size_t pcm_stride, size_t *n_pcm, int sync);

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

/* window_coefs: N ints (the global window_coefs table); sinewave: 3N/4 int16 (the global Sinewave)
 * or NULL to build it with rxb200_sine_table. */
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
