"""rx_sdr channels of one capture (``rxb200_sdr_mix_*``, include/rxb200.h "rx_sdr channels of one capture"): record the
I/Q of several channels of ONE wideband CS16 capture, each down-converted, decimated and written in rx_sdr's recorded
format, with the capture count and the filter histories carried between calls."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _lib
from .fm import CVT_CS16_CF32, CVT_CS16_CS8, CVT_CS16_CU8, CapturePlan, _ddc_c, _plan_call, _ptr

OUT_CS16 = 4
FORMATS = {"CS16": OUT_CS16, "CS8": CVT_CS16_CS8, "CU8": CVT_CS16_CU8, "CF32": CVT_CS16_CF32}
ELEM_BYTES = {OUT_CS16: 4, CVT_CS16_CS8: 2, CVT_CS16_CU8: 2, CVT_CS16_CF32: 8}
# the numpy dtype of one component (I or Q) of each format
DTYPES = {OUT_CS16: np.int16, CVT_CS16_CS8: np.uint8, CVT_CS16_CU8: np.uint8, CVT_CS16_CF32: np.float32}


def plan_sdr_capture(tuned_hz, sample_rate: int, max_rate: int, device_rate: Optional[int] = None):
    """The rx_sdr shell's capture plan (``rxb200_sdr_plan_capture``, or ``_at`` with a device_rate): (CapturePlan, each
    channel's offset).  It is ``fm.plan_capture`` with chain rate sample_rate, but takes any offset (the handle mixes
    with the NCO)."""
    t = np.ascontiguousarray(tuned_hz, dtype=np.int64).reshape(-1)
    offs = np.zeros(max(t.size, 1), dtype=np.int32)
    out = _lib.FmCapturePlanC()
    _plan_call("rxb200_sdr_plan_capture", t, sample_rate, max_rate, device_rate, out, offs)
    return CapturePlan(int(out.centre_hz), out.decim, out.capture_rate, out.n_taps), [int(v) for v in offs[:t.size]]


class SdrMix:
    """``len(offsets_hz)`` channels of ONE CS16 capture at ``capture_rate``.  ddc = (decim, taps, shift): the single
    stage (``rxb200_sdr_mix_create``), channel c the rx_power NCO rule then the filter.  two_stage = (n_bins, coarse,
    fine) instead: the two-stage rule (``rxb200_sdr_mix_create_two_stage``).  raster = (n_bins, bins) with ddc: the
    raster rule (``rxb200_sdr_mix_create_raster``), channel c bin bins[c] of an n_bins-bin raster over the capture;
    capture_rate and offsets_hz are then None.  Every call takes the capture, int16 [n_int16], and returns the call's
    outputs in format fmt (``FORMATS``) as a [n_channels][2 n_out] array of the format's component type."""

    def __init__(self, capture_rate: Optional[int] = None, offsets_hz=None, ddc=None, two_stage=None, device: int = 0,
                 raster=None):
        if (ddc is None) == (two_stage is None):
            raise ValueError("give exactly one of ddc and two_stage")
        self.device = device
        self._h = C.c_void_p()
        L = _lib.lib()
        if raster is not None:
            if ddc is None or capture_rate is not None or offsets_hz is not None:
                raise ValueError("a raster handle takes a ddc and bins, no capture_rate or offsets_hz")
            n_bins, bins = raster
            b = np.ascontiguousarray(bins, dtype=np.int32).reshape(-1)
            self.capture_rate, self.offsets_hz, self.n_channels = None, None, int(b.size)
            d, _t = _ddc_c(ddc)
            self.decim = int(ddc[0])
            _lib.check(L.rxb200_sdr_mix_create_raster(n_bins, _ptr(b), self.n_channels, C.byref(d), device,
                                                      C.byref(self._h)))
            return
        offs = np.ascontiguousarray(offsets_hz, dtype=np.int32).reshape(-1)
        self.capture_rate, self.offsets_hz, self.n_channels = capture_rate, offs.tolist(), int(offs.size)
        if ddc is not None:
            d, _t = _ddc_c(ddc)
            self.decim = int(ddc[0])
            _lib.check(L.rxb200_sdr_mix_create(capture_rate, _ptr(offs), self.n_channels, C.byref(d), device,
                                               C.byref(self._h)))
        else:
            n_bins, coarse, fine = two_stage
            d1, _t1 = _ddc_c(coarse)
            d2, _t2 = _ddc_c(fine)
            self.decim = int(coarse[0]) * int(fine[0])
            _lib.check(L.rxb200_sdr_mix_create_two_stage(capture_rate, n_bins, _ptr(offs), self.n_channels, C.byref(d1),
                                                         C.byref(d2), device, C.byref(self._h)))

    def close(self) -> None:
        if self._h:
            _lib.lib().rxb200_sdr_mix_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def reset(self) -> None:
        _lib.check(_lib.lib().rxb200_sdr_mix_reset(self._h))

    def set_device_rate(self, up: int, down: int, taps, shift: int = 15) -> None:
        """Attach a resampler right after create or reset (``rxb200_sdr_mix_set_device_rate``): from then on every call
        takes device-rate CS16."""
        from .resample import _rs_c
        rs, _t = _rs_c(up, down, taps, shift)
        _lib.check(_lib.lib().rxb200_sdr_mix_set_device_rate(self._h, C.byref(rs)))

    def set_input_format(self, fmt) -> None:
        """The capture's format right after create or reset (``rxb200_sdr_mix_set_input_format``): ``_lib.IN_*`` or its
        name.  From then on every call takes the format's raw bytes (uint8) for CS8, CU8 and CS12, widened to CS16 on
        the GPU; n_int16 still counts two per complex element."""
        fmt = _lib.IN_FORMATS.get(fmt, fmt)
        _lib.check(_lib.lib().rxb200_sdr_mix_set_input_format(self._h, fmt))
        self._in_fmt = fmt

    def decimated_len(self, n_int16: int) -> int:
        n = C.c_size_t(0)
        _lib.check(_lib.lib().rxb200_sdr_mix_decimated_len(self._h, n_int16, C.byref(n)))
        return int(n.value)

    def process(self, cs16: np.ndarray, fmt=OUT_CS16) -> np.ndarray:
        """One host call: the capture's outputs, [n_channels][2 n_out] of the format's component type."""
        fmt = FORMATS.get(fmt, fmt)
        x, n_int16 = _lib.in_array(cs16, getattr(self, "_in_fmt", _lib.IN_CS16))
        n = self.decimated_len(n_int16)
        out = np.zeros((self.n_channels, 2 * max(n, 1)), dtype=DTYPES[fmt])
        got = C.c_size_t(0)
        _lib.check(_lib.lib().rxb200_sdr_mix_process(self._h, x.ctypes.data, n_int16, fmt, out.ctypes.data, out.size // 2,
                                                     out.shape[1] // 2, C.byref(got)))
        assert got.value == n
        return out[:, :2 * n]

    def process_device(self, d_cs16: int, n_int16: int, fmt: int, d_out: int, out_cap: int, out_stride: int,
                       sync: int = 1) -> int:
        """One call on device pointers (``rxb200_sdr_mix_process_device``); returns the outputs per channel."""
        got = C.c_size_t(0)
        _lib.check(_lib.lib().rxb200_sdr_mix_process_device(self._h, d_cs16, n_int16, FORMATS.get(fmt, fmt), d_out,
                                                            out_cap, out_stride, C.byref(got), sync))
        return int(got.value)

    def kernel_ms(self) -> float:
        ms = C.c_float(0)
        _lib.check(_lib.lib().rxb200_sdr_mix_kernel_ms(self._h, C.byref(ms)))
        return float(ms.value)

    @property
    def stream(self) -> int:
        return int(_lib.lib().rxb200_sdr_mix_stream(self._h) or 0)
