/* Declarations-only stand-in for <SoapySDR/Device.h>; see Version.h.
 * Only the 0.8 C entry points that rx_tools calls are declared. */
#pragma once
#include <stddef.h>
#include <stdbool.h>
#include <stdint.h>

#define SOAPY_SDR_TX 0
#define SOAPY_SDR_RX 1

#define SOAPY_SDR_END_BURST (1 << 1)
#define SOAPY_SDR_HAS_TIME (1 << 2)
#define SOAPY_SDR_END_ABRUPT (1 << 3)
#define SOAPY_SDR_ONE_PACKET (1 << 4)
#define SOAPY_SDR_MORE_FRAGMENTS (1 << 5)

#define SOAPY_SDR_TIMEOUT (-1)
#define SOAPY_SDR_STREAM_ERROR (-2)
#define SOAPY_SDR_CORRUPTION (-3)
#define SOAPY_SDR_OVERFLOW (-4)
#define SOAPY_SDR_NOT_SUPPORTED (-5)
#define SOAPY_SDR_TIME_ERROR (-6)
#define SOAPY_SDR_UNDERFLOW (-7)

#ifdef __cplusplus
extern "C" {
#endif

typedef struct SoapySDRDevice SoapySDRDevice;
typedef struct SoapySDRStream SoapySDRStream;

typedef struct {
	size_t size;
	char **keys;
	char **vals;
} SoapySDRKwargs;

typedef struct {
	double minimum;
	double maximum;
	double step;
} SoapySDRRange;

SoapySDRKwargs SoapySDRKwargs_fromString(const char *markup);
void SoapySDRKwargs_clear(SoapySDRKwargs *args);

const char *SoapySDRDevice_lastError(void);
SoapySDRDevice *SoapySDRDevice_makeStrArgs(const char *args);
int SoapySDRDevice_unmake(SoapySDRDevice *device);

char *SoapySDRDevice_getDriverKey(const SoapySDRDevice *device);
char *SoapySDRDevice_getHardwareKey(const SoapySDRDevice *device);
SoapySDRKwargs SoapySDRDevice_getHardwareInfo(const SoapySDRDevice *device);
size_t SoapySDRDevice_getNumChannels(const SoapySDRDevice *device, const int direction);

SoapySDRStream *SoapySDRDevice_setupStream(SoapySDRDevice *device, const int direction,
	const char *format, const size_t *channels, const size_t numChans, const SoapySDRKwargs *args);
int SoapySDRDevice_closeStream(SoapySDRDevice *device, SoapySDRStream *stream);
int SoapySDRDevice_activateStream(SoapySDRDevice *device, SoapySDRStream *stream,
	const int flags, const long long timeNs, const size_t numElems);
int SoapySDRDevice_deactivateStream(SoapySDRDevice *device, SoapySDRStream *stream,
	const int flags, const long long timeNs);
int SoapySDRDevice_readStream(SoapySDRDevice *device, SoapySDRStream *stream,
	void * const *buffs, const size_t numElems, int *flags, long long *timeNs, const long timeoutUs);

int SoapySDRDevice_setAntenna(SoapySDRDevice *device, const int direction, const size_t channel, const char *name);
char **SoapySDRDevice_listAntennas(const SoapySDRDevice *device, const int direction, const size_t channel, size_t *length);
char **SoapySDRDevice_listGains(const SoapySDRDevice *device, const int direction, const size_t channel, size_t *length);
char **SoapySDRDevice_listFrequencies(const SoapySDRDevice *device, const int direction, const size_t channel, size_t *length);
double *SoapySDRDevice_listSampleRates(const SoapySDRDevice *device, const int direction, const size_t channel, size_t *length);
double *SoapySDRDevice_listBandwidths(const SoapySDRDevice *device, const int direction, const size_t channel, size_t *length);

int SoapySDRDevice_setGainMode(SoapySDRDevice *device, const int direction, const size_t channel, const bool automatic);
int SoapySDRDevice_setGain(SoapySDRDevice *device, const int direction, const size_t channel, const double value);
int SoapySDRDevice_setGainElement(SoapySDRDevice *device, const int direction, const size_t channel, const char *name, const double value);

int SoapySDRDevice_setFrequency(SoapySDRDevice *device, const int direction, const size_t channel, const double frequency, const SoapySDRKwargs *args);
double SoapySDRDevice_getFrequency(const SoapySDRDevice *device, const int direction, const size_t channel);
int SoapySDRDevice_setFrequencyCorrection(SoapySDRDevice *device, const int direction, const size_t channel, const double value);
int SoapySDRDevice_setSampleRate(SoapySDRDevice *device, const int direction, const size_t channel, const double rate);
double SoapySDRDevice_getSampleRate(const SoapySDRDevice *device, const int direction, const size_t channel);
int SoapySDRDevice_setBandwidth(SoapySDRDevice *device, const int direction, const size_t channel, const double bw);
double SoapySDRDevice_getBandwidth(const SoapySDRDevice *device, const int direction, const size_t channel);

int SoapySDRDevice_writeSetting(SoapySDRDevice *device, const char *key, const char *value);
char *SoapySDRDevice_readSetting(const SoapySDRDevice *device, const char *key);

#ifdef __cplusplus
}
#endif
