"""Capture from a device at its own rate (``rxb200_resample_*``, include/rxb200.h "capture from a device at its own
rate"): a rational resampler that takes a device's CS16 stream at the rate it runs at, R_dev, to a capture plan's rate
R = R_dev L / N by an exact integer polyphase rule, carrying the device-sample count and the filter history between
calls so that a stream made of many calls is one stream."""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple

import numpy as np

from . import _lib


class ResamplePlan(NamedTuple):
    up: int               # L
    down: int             # N
    taps_per_phase: int   # J
    shift: int            # S


def lowpass(up: int, down: int, taps_per_phase: int) -> np.ndarray:
    """The prototype filter ``rxb200_resample_lowpass``: int32 [J L], every phase h[p::L] summing to exactly 2^15."""
    t = np.zeros(int(up) * int(taps_per_phase), dtype=np.int32)
    _lib.check(_lib.lib().rxb200_resample_lowpass(int(up), int(down), int(taps_per_phase),
                                                  t.ctypes.data_as(C.POINTER(C.c_int32))))
    return t


def plan_resample(device_rate: int, rate: int, span: int) -> ResamplePlan:
    """``rxb200_plan_resample``: (L, N, J, S) from the device rate to the plan's rate for channels spanning span Hz."""
    out = _lib.ResamplerC()
    _lib.check(_lib.lib().rxb200_plan_resample(int(device_rate), int(rate), int(span), C.byref(out)))
    return ResamplePlan(out.up, out.down, out.taps_per_phase, out.shift)


def out_count(n0: int, n_complex: int, up: int, down: int) -> int:
    """The outputs of a call over device samples [n0, n0 + n_complex): ceil((n0 + c) L / N) - ceil(n0 L / N)."""
    return -(-(n0 + n_complex) * up // down) + (-(n0 * up) // down)


def in_len(up: int, down: int, n0: int, n_out: int) -> int:
    """``rxb200_resample_in_len``: the fewest device samples from n0 that emit at least n_out outputs."""
    n = C.c_size_t(0)
    _lib.check(_lib.lib().rxb200_resample_in_len(int(up), int(down), int(n0), int(n_out), C.byref(n)))
    return int(n.value)


def _rs_c(up, down, taps, shift):
    t = np.ascontiguousarray(taps, dtype=np.int32).reshape(-1)
    J = t.size // int(up) if int(up) > 0 else 0
    return _lib.ResamplerC(int(up), int(down), int(J), t.ctypes.data_as(C.POINTER(C.c_int32)), int(shift)), t


def resample_device(up: int, down: int, taps, shift: int, n0: int, d_src_ptr: int, n_complex: int, d_dst_ptr: int,
                    stream: int = 0) -> None:
    """``rxb200_resample_device``: stateless, d_src[i] is device sample n0 + i, the samples before it zero."""
    rs, _t = _rs_c(up, down, taps, shift)
    _lib.check(_lib.lib().rxb200_resample_device(C.byref(rs), int(n0), d_src_ptr, int(n_complex), d_dst_ptr,
                                                 stream or None))


class Resampler:
    """One device stream resampled by up/down with the prototype taps (J = len(taps) / up per phase) and shift."""

    def __init__(self, up: int, down: int, taps, shift: int = 15, device: int = 0):
        self.up, self.down, self.shift, self.device = int(up), int(down), int(shift), device
        self._h = C.c_void_p()
        rs, _t = _rs_c(up, down, taps, shift)
        _lib.check(_lib.lib().rxb200_resample_create(C.byref(rs), device, C.byref(self._h)))

    def close(self) -> None:
        if self._h:
            _lib.lib().rxb200_resample_destroy(self._h)
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
        _lib.check(_lib.lib().rxb200_resample_reset(self._h))

    def out_len(self, n_int16: int) -> int:
        n = C.c_size_t(0)
        _lib.check(_lib.lib().rxb200_resample_out_len(self._h, n_int16, C.byref(n)))
        return int(n.value)

    def process(self, cs16: np.ndarray) -> np.ndarray:
        """One host call: int16 [n_int16] device samples in, int16 [2 n_out] resampled samples out."""
        x = np.ascontiguousarray(cs16, dtype=np.int16).reshape(-1)
        n = self.out_len(x.size)
        out = np.zeros(2 * max(n, 1), dtype=np.int16)
        got = C.c_size_t(0)
        _lib.check(_lib.lib().rxb200_resample_process(self._h, x.ctypes.data, x.size, out.ctypes.data, out.size // 2,
                                                      C.byref(got)))
        assert got.value == n
        return out[:2 * n]

    def process_device(self, d_cs16: int, n_int16: int, d_out: int, out_cap: int, sync: int = 1) -> int:
        """One call on device pointers (``rxb200_resample_process_device``); returns the outputs."""
        got = C.c_size_t(0)
        _lib.check(_lib.lib().rxb200_resample_process_device(self._h, d_cs16, n_int16, d_out, out_cap, C.byref(got),
                                                             sync))
        return int(got.value)

    def kernel_ms(self) -> float:
        ms = C.c_float(0)
        _lib.check(_lib.lib().rxb200_resample_kernel_ms(self._h, C.byref(ms)))
        return float(ms.value)

    @property
    def stream(self) -> int:
        return int(_lib.lib().rxb200_resample_stream(self._h) or 0)
