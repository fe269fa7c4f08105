/* sdr_util.h — small host helpers shared by the drop-in shells rx_fm_b200 / rx_power_b200 / rx_sdr_b200.
 * Own implementation of what rx_tools keeps in src/convenience/ (suffix parsing, device/stream
 * bring-up); behaviourally equivalent, not copied.  And the capture-mode plan of rx_fm_b200 and rx_sdr_b200. */
#ifndef RXB_SDR_UTIL_H
#define RXB_SDR_UTIL_H
#include <stddef.h>
#include <stdint.h>
#include <SoapySDR/Device.h>
#include <SoapySDR/Formats.h>
#include "rxb200.h"

double parse_scaled(const char *s);    /* 100M, 24k, 1.2G   (convenience.c:65-90)  */
double parse_seconds(const char *s);   /* 10s, 5m, 1h       (convenience.c:92-117) */
double parse_fraction(const char *s);  /* 28.5% -> 0.285    (convenience.c:119-136) */

/* makeStrArgs + an RX stream of `format` (SOAPY_SDR_CS16 unless RXB200_DEVICE_FORMAT says otherwise) on `channel`;
 * prints like the reference's verbose_* helpers. Returns 0 on success. */
int sdr_open(const char *query, size_t channel, const char *format, SoapySDRDevice **dev, SoapySDRStream **stream);
void sdr_close(SoapySDRDevice *dev, SoapySDRStream *stream);
/* gain: NULL = automatic, "30" overall, or "LNA=20,VGA=10" per element */
void sdr_set_gain(SoapySDRDevice *dev, size_t channel, const char *gain_str);

/* Capture mode (RXB200_CAPTURE_RATE): every channel from one capture, through a front stage of one of three kinds. */
enum capture_kind { CAPTURE_SINGLE, CAPTURE_RASTER, CAPTURE_TWO_STAGE };
struct capture_plan {
	int64_t centre_hz;     /* fc */
	int capture_rate;      /* R */
	int decim;             /* the total decimation: M, or M1 M2 for two stages */
	int n_bins;            /* K (raster, two stages) */
	long long span;        /* 2 A + c: the channels' span around the centre, A the largest |t_k - fc| */
	rxb200_ddc ddc;        /* the filter, the coarse one for two stages */
	rxb200_ddc fine;       /* two stages: the fine filter */
	char banner[256];      /* the "Capture mode: ..." line the shell prints */
};
/* The plan of kind for the n tuned frequencies at chain rate chain_rate under the cap cap_env (RXB200_CAPTURE_RATE's
 * value): single, rxb200_sdr_plan_capture's when nco (rx_sdr mixes with the NCO) else rxb200_fm_plan_capture's;
 * raster, rxb200_fm_plan_capture_raster's; two stages, rxb200_fm_plan_capture_two_stage's; each through its _at
 * planner when device_rate is not 0.  chans receives the n offsets (the bins for a raster).  The filters' taps are
 * rxb200_ddc_lowpass's, freed by capture_plan_release.  A refused plan is reported on stderr and returns nonzero, with
 * nothing to release. */
int capture_plan(enum capture_kind kind, const int64_t *tuned, int n, int chain_rate, const char *cap_env, int nco,
                 long long device_rate, struct capture_plan *p, int *chans);
void capture_plan_release(struct capture_plan *p);

/* Capture at the device's own rate (RXB200_DEVICE_RATE, DESIGN.md section 4.7).
 * device_rate_env: the variable's value, 0 when it is unset; -1, reported on stderr, when it is set but `allowed` is 0
 * (none of the variables named by `needs` is set) or it is not a whole number of Hz in [1, 2^31 - 1]. */
long long device_rate_env(int allowed, const char *needs);
/* setSampleRate(rate), then the rate the device reports, rounded to whole Hz; -1, reported on stderr, when that is not
 * a rate in [1, 2^31 - 1] Hz (a driver that does not report its rate returns 0) */
long long sdr_device_rate(SoapySDRDevice *dev, size_t channel, long long rate);
/* The resampler from device_rate to a plan's rate for channels spanning span Hz (rxb200_plan_resample), its taps
 * rxb200_resample_lowpass's on the heap (free rs->taps; NULL when L = N = 1, no resampler needed), and the banner line
 * "Device rate: ...".  Nonzero, reported on stderr, when the span leaves no room for the resampler. */
int device_resampler(long long device_rate, long long rate, long long span, rxb200_resampler *rs);
/* the capture samples the device samples [n0, n0 + c) emit through an L/N resampler */
size_t resample_out_count(int up, int down, unsigned long long n0, size_t c);

/* Capture in the device's own sample format (RXB200_DEVICE_FORMAT, DESIGN.md section 4.8).
 * device_format_env: the variable's value as RXB200_IN_CS16, _CS8, _CU8 or _CS12, with its SoapySDR format name at
 * *name; RXB200_IN_CS16 and SOAPY_SDR_CS16 when it is unset; -1, reported on stderr, when it is set but `allowed` is 0
 * (none of the variables named by `needs` is set) or it is not one of CS16, CS8, CU8, CS12. */
int device_format_env(int allowed, const char *needs, const char **name);
/* bytes per complex element of an RXB200_IN_* format */
size_t device_format_bytes(int in_fmt);
#endif
