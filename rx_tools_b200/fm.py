"""rx_fm path — host-side mirror of the reference's interface (src/rtl_fm.c).

``FmParams`` carries the ``struct demod_state`` configuration fields under the reference's own names
(src/rtl_fm.c:124-159); ``derive_params`` is ``main()`` + ``optimal_settings()`` (:1224-1415, :960-997);
``FmDemod.full_demod`` is "``rtlsdr_callback`` + ``full_demod`` once per chunk" (:828-863, :759-824)
executed by the fused sm_90a kernel behind ``rxb200_fm_process`` (include/rxb200.h).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, fields
from typing import Optional

import numpy as np

from . import _lib

MODE_FM, MODE_AM, MODE_USB, MODE_LSB, MODE_RAW = range(5)
ATAN_STD, ATAN_FAST, ATAN_LUT, ATAN_ALE = range(4)
MAXIMUM_BUF_LENGTH = 262144          # src/rtl_fm.c:80-82


@dataclass
class FmParams:
    mode: int = MODE_FM
    downsample: int = 1
    downsample_passes: int = 0
    comp_fir_size: int = 0
    custom_atan: int = ATAN_STD
    output_scale: int = 1
    post_downsample: int = 1
    deemph: int = 0
    deemph_a: int = 0
    rate_out: int = 24000
    rate_out2: int = -1
    squelch_level: int = 0
    dc_block_audio: int = 0
    adc_block_const: int = 9
    dc_block_raw: int = 0
    rdc_block_const: int = 9
    offset_tuning: int = 0
    report_levels: int = 0

    def reference_fields(self) -> dict:
        """The fields that exist in the reference's demod_state (everything but library-only switches)."""
        return {f.name: int(getattr(self, f.name)) for f in fields(self) if f.name != "report_levels"}

    def to_c(self) -> _lib.FmParamsC:
        return _lib.FmParamsC(*[int(getattr(self, f.name)) for f in fields(self)])

    @classmethod
    def from_any(cls, other) -> "FmParams":
        return cls(**{f.name: int(getattr(other, f.name, 0)) for f in fields(cls)})


@dataclass
class Derived:
    params: FmParams
    capture_rate: int
    capture_freq_offset: int
    output_rate: int


def derive_params(mode: int = MODE_FM, rate_s: int = 0, rate_r: int = 0, use_F: int = 0, comp_fir_size: int = 0,
                  custom_atan: int = -1, post_downsample: int = 1, deemph: int = -1, time_constant_us: int = 75,
                  wbfm: int = 0, offset_tuning: int = 0, squelch_level: int = 0, dc_block_audio: int = 0,
                  dc_block_raw: int = 0, rdc_block_const: int = 0) -> Derived:
    """CLI-level values -> kernel parameters, as rx_fm's main() and optimal_settings() derive them."""
    cli = _lib.FmCliC(mode, wbfm, rate_s, rate_r, use_F, comp_fir_size, custom_atan, post_downsample, deemph,
                      time_constant_us, offset_tuning, squelch_level, dc_block_audio, dc_block_raw, rdc_block_const)
    out = _lib.FmDerivedC()
    _lib.check(_lib.lib().rxb200_fm_derive(C.byref(cli), C.byref(out)))
    return Derived(FmParams.from_any(out.params), out.capture_rate, out.capture_freq_offset, out.output_rate)


class FmDemod:
    """One handle = ``n_channels`` independent demod_state streams with identical parameters."""

    def __init__(self, params, device: int = 0, n_channels: int = 1):
        self.params = FmParams.from_any(params)
        self.n_channels = n_channels
        self._h = C.c_void_p()
        pc = self.params.to_c()
        _lib.check(_lib.lib().rxb200_fm_create(C.byref(pc), device, n_channels, C.byref(self._h)))

    def close(self) -> None:
        if _lib is not None and getattr(self, "_h", None) is not None and self._h:
            _lib.lib().rxb200_fm_destroy(self._h)
            self._h = None

    __del__ = close

    def reset(self) -> None:
        _lib.check(_lib.lib().rxb200_fm_reset(self._h))

    def tune(self, segment_len: int = 0, deemph_warmup: int = 0) -> None:
        _lib.check(_lib.lib().rxb200_fm_tune(self._h, segment_len, deemph_warmup))

    def max_output(self, n_int16: int, chunk_int16: int = MAXIMUM_BUF_LENGTH) -> int:
        return int(_lib.lib().rxb200_fm_max_output(self._h, n_int16, chunk_int16))

    def full_demod(self, cs16: np.ndarray, chunk_int16: int = MAXIMUM_BUF_LENGTH, return_chunks: bool = False):
        """Host arrays in, host arrays out.  cs16: int16[n_int16] (one channel) or
        int16[n_channels][n_int16].  Returns the concatenated ``demod.result`` per channel."""
        x = np.ascontiguousarray(cs16, dtype=np.int16)
        single = x.ndim == 1
        x2 = x.reshape(1, -1) if single else x
        assert x2.shape[0] == self.n_channels, (x2.shape, self.n_channels)
        n_int16 = x2.shape[1]
        cap = self.max_output(n_int16, chunk_int16) + 8
        out = np.empty((self.n_channels, cap), dtype=np.int16)
        n_chunks = max(1, -(-n_int16 // chunk_int16))
        lens = np.zeros(n_chunks, dtype=np.int32)
        n_pcm = C.c_size_t(0)
        _lib.check(_lib.lib().rxb200_fm_process(self._h, x2.ctypes.data, n_int16, chunk_int16, out.ctypes.data, cap,
                                                C.byref(n_pcm), lens.ctypes.data_as(C.POINTER(C.c_int))))
        res = out[:, :n_pcm.value].copy()
        res = res[0] if single else res
        return (res, lens) if return_chunks else res

    def process_device(self, d_in_ptr: int, n_int16: int, chunk_int16: int, d_out_ptr: int, out_stride: int,
                       sync: bool = False) -> int:
        """Device pointers (e.g. torch tensors' data_ptr()); returns PCM count per channel."""
        n_pcm = C.c_size_t(0)
        _lib.check(_lib.lib().rxb200_fm_process_device(self._h, d_in_ptr, n_int16, chunk_int16, d_out_ptr, out_stride,
                                                       C.byref(n_pcm), 1 if sync else 0))
        return int(n_pcm.value)

    def levels(self) -> np.ndarray:
        """rms() of every chunk of the last call, int32[n_channels][n_chunks] (needs report_levels;
        the ``sr`` of src/rtl_fm.c:792-806)."""
        cap = 1024
        while True:
            buf = np.zeros(cap, dtype=np.int32)
            n = C.c_size_t(0)
            rc = _lib.lib().rxb200_fm_levels(self._h, buf.ctypes.data_as(C.POINTER(C.c_int)), cap, C.byref(n))
            if rc == _lib.ECAPACITY:
                cap = int(n.value) * self.n_channels
                continue
            _lib.check(rc)
            return buf[:int(n.value) * self.n_channels].reshape(self.n_channels, int(n.value)).copy()

    @property
    def stream(self) -> int:
        return int(_lib.lib().rxb200_fm_stream(self._h) or 0)

    def kernel_ms(self) -> float:
        ms = C.c_float(0)
        _lib.check(_lib.lib().rxb200_fm_kernel_ms(self._h, C.byref(ms)))
        return float(ms.value)

    def stats(self) -> dict:
        s = _lib.FmStatsC()
        _lib.check(_lib.lib().rxb200_fm_last_stats(self._h, C.byref(s)))
        d = {f[0]: int(getattr(s, f[0])) for f in s._fields_}
        d["kernel"] = {1: "fm_split_kernel", 3: "fm_fused_kernel+fm_back_kernel"}.get(d["kernel_kind"], "fm_fused_kernel")
        return d


# ---- rx_sdr sample-format conversions (src/rtl_sdr.c:348-391) -------------------------------------------
CVT_CS16_CS8, CVT_CS16_CU8, CVT_CS16_CF32, CVT_CS12_CS16 = range(4)


def sdr_convert(kind: int, src: np.ndarray, device: int = 0) -> np.ndarray:
    """CS16 (int16 interleaved) -> CS8 / CU8 (uint8 bytes) / CF32 (float32), or packed CS12 (uint8, 3 bytes per
    complex element) -> CS16."""
    if kind == CVT_CS12_CS16:
        s = np.ascontiguousarray(src, dtype=np.uint8)
        n = s.size // 3
        out = np.empty(2 * n, dtype=np.int16)
    else:
        s = np.ascontiguousarray(src, dtype=np.int16)
        n = s.size // 2
        out = np.empty(2 * n, dtype=np.float32 if kind == CVT_CS16_CF32 else np.uint8)
    _lib.check(_lib.lib().rxb200_sdr_convert(kind, s.ctypes.data, n, out.ctypes.data, device))
    return out
