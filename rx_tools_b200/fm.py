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
# forms of disc_device (RXB200_DISC_*): the four discriminators, then the other device code a chain's samples run through
DISC_STD, DISC_FAST, DISC_LUT, DISC_ALE, DISC_ATAN2, DISC_STD_FP64, DISC_ROWS, DISC_STREAM, DISC_AM = range(9)
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


class _Handle:
    """What the four rx_fm handle kinds share: ``_prefix`` names their C entry points (``<prefix>_process`` ...), ``_h``
    holds the handle.  A subclass states how it is created, whether its input is per-channel streams
    (``_streams``: int16[n_int16] or int16[n_channels][n_int16]) or one capture (int16[n_int16]), and ``_bound``, the
    PCM per channel a call can make."""

    _prefix = ""
    _streams = True

    def _fn(self, name: str):
        return getattr(_lib.lib(), f"{self._prefix}_{name}")

    def close(self) -> None:
        if _lib is not None and getattr(self, "_h", None) is not None and self._h:
            self._fn("destroy")(self._h)
            self._h = None

    __del__ = close

    def reset(self) -> None:
        _lib.check(self._fn("reset")(self._h))

    def _input(self, cs16):
        """(the input as one C array, n_int16, whether a 1-D input of a one-channel stream handle returns 1-D)"""
        x = np.ascontiguousarray(cs16, dtype=np.int16)
        if not self._streams:
            x = x.reshape(-1)
            return x, x.size, False
        x2 = x.reshape(1, -1) if x.ndim == 1 else x
        assert x2.shape[0] == self.n_channels, (x2.shape, self.n_channels)
        return x2, x2.shape[1], x.ndim == 1

    def full_demod(self, cs16: np.ndarray, chunk_int16: int = MAXIMUM_BUF_LENGTH, return_chunks: bool = False):
        """Host arrays in, host arrays out (``<prefix>_process``): ``rtlsdr_callback`` + ``full_demod`` once per chunk.
        Returns the concatenated ``demod.result`` per channel, int16[n_channels][n_pcm] (int16[n_pcm] for a 1-D input
        of one channel stream), and with return_chunks the PCM count of each chunk."""
        x, n_int16, single = self._input(cs16)
        cap = self._bound(n_int16, chunk_int16) + 8
        out = np.empty((self.n_channels, cap), dtype=np.int16)
        lens = np.zeros(max(1, -(-n_int16 // chunk_int16)), dtype=np.int32)
        n_pcm = C.c_size_t(0)
        _lib.check(self._fn("process")(self._h, x.ctypes.data, n_int16, chunk_int16, out.ctypes.data, cap,
                                       C.byref(n_pcm), lens.ctypes.data_as(C.POINTER(C.c_int))))
        res = out[:, :n_pcm.value].copy()
        res = res[0] if single else res
        return (res, lens) if return_chunks else res

    def process_read(self, cs16: np.ndarray) -> np.ndarray:
        """One device read: ``rtlsdr_callback`` + ``full_demod`` once on the whole of it, whatever its length
        (``<prefix>_process_read``).  Shapes as ``full_demod``."""
        x, n_int16, single = self._input(cs16)
        cap = self._bound(n_int16, max(n_int16, 1)) + 8
        out = np.empty((self.n_channels, cap), dtype=np.int16)
        n_pcm = C.c_size_t(0)
        _lib.check(self._fn("process_read")(self._h, x.ctypes.data, n_int16, out.ctypes.data, cap, C.byref(n_pcm)))
        res = out[:, :n_pcm.value].copy()
        return res[0] if single else res

    def squelch_hits(self) -> np.ndarray:
        """demod.squelch_hits of every channel after the last call, int32[n_channels]."""
        h = np.zeros(self.n_channels, dtype=np.int32)
        _lib.check(self._fn("squelch_hits")(self._h, h.ctypes.data_as(C.POINTER(C.c_int))))
        return h

    def levels(self) -> np.ndarray:
        """rms() of every chunk of the last call, int32[n_channels][n_chunks] (needs report_levels; the ``sr`` of
        src/rtl_fm.c:792-806)."""
        fn, n = self._fn("levels"), C.c_size_t(0)
        rc = fn(self._h, np.zeros(1, np.int32).ctypes.data_as(C.POINTER(C.c_int)), 0, C.byref(n))
        if rc != _lib.ECAPACITY:
            _lib.check(rc)
        buf = np.zeros((self.n_channels, int(n.value)), dtype=np.int32)
        _lib.check(fn(self._h, buf.ctypes.data_as(C.POINTER(C.c_int)), buf.size, C.byref(n)))
        return buf


class _OneGpu(_Handle):
    """The device entry points of the single-GPU kinds (``FmDemod``, ``FmMix``)."""

    def process_device(self, d_in_ptr: int, n_int16: int, chunk_int16: int, d_out_ptr: int, out_stride: int,
                       sync: bool = False) -> int:
        """Device pointers (e.g. torch tensors' data_ptr()): the input and [n_channels][out_stride] PCM; returns the PCM
        count per channel."""
        n_pcm = C.c_size_t(0)
        _lib.check(self._fn("process_device")(self._h, d_in_ptr, n_int16, chunk_int16, d_out_ptr, out_stride,
                                              C.byref(n_pcm), 1 if sync else 0))
        return int(n_pcm.value)

    def process_read_device(self, d_in_ptr: int, n_int16: int, d_out_ptr: int, out_stride: int,
                            sync: bool = False) -> int:
        """``process_read`` on device pointers (4-byte alignment is enough); returns the PCM count per channel."""
        n_pcm = C.c_size_t(0)
        _lib.check(self._fn("process_read_device")(self._h, d_in_ptr, n_int16, d_out_ptr, out_stride, C.byref(n_pcm),
                                                   1 if sync else 0))
        return int(n_pcm.value)


def _devices(devices, n_dev):
    """A group's member ordinals as a C array (None: range(n_dev)) and its member count."""
    devs = None if devices is None else np.ascontiguousarray(devices, dtype=np.int32)
    return devs, len(devs) if devs is not None else int(n_dev or 1)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_int))


class FmDemod(_OneGpu):
    """One handle = ``n_channels`` independent demod_state streams with identical parameters."""

    _prefix = "rxb200_fm"

    def __init__(self, params, device: int = 0, n_channels: int = 1):
        self.params = FmParams.from_any(params)
        self.n_channels = n_channels
        self._h = C.c_void_p()
        pc = self.params.to_c()
        _lib.check(_lib.lib().rxb200_fm_create(C.byref(pc), device, n_channels, C.byref(self._h)))

    def tune(self, segment_len: int = 0, deemph_warmup: int = 0) -> None:
        _lib.check(_lib.lib().rxb200_fm_tune(self._h, segment_len, deemph_warmup))

    def max_output(self, n_int16: int, chunk_int16: int = MAXIMUM_BUF_LENGTH) -> int:
        return int(_lib.lib().rxb200_fm_max_output(self._h, n_int16, chunk_int16))

    _bound = max_output

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


class FmGroup(_Handle):
    """``n_channels`` streams split over several GPUs (``rxb200_fm_group_*``): member i owns a contiguous block of the
    channels and its own ``rxb200_fm`` handle; the group's results are byte for byte those of one ``FmDemod`` with all
    the channels.  devices: one CUDA ordinal per member (may repeat), or None for ``range(n_dev)``."""

    _prefix = "rxb200_fm_group"
    _g = property(lambda self: self._h)     # the handle under the name callers of earlier releases read

    def __init__(self, params, n_channels: int, devices=None, n_dev: Optional[int] = None):
        self.params = FmParams.from_any(params)
        self.n_channels = n_channels
        devs, self.n_dev = _devices(devices, n_dev)
        self._h = C.c_void_p()
        pc = self.params.to_c()
        _lib.check(_lib.lib().rxb200_fm_group_create(C.byref(pc), n_channels, self.n_dev, _ptr(devs), C.byref(self._h)))

    def member(self, i: int) -> int:
        """Member i's rxb200_fm handle as an integer, 0 for a member that owns no channel."""
        return int(_lib.lib().rxb200_fm_group_member(self._h, i) or 0)

    def _bound(self, n_int16: int, chunk_int16: int) -> int:
        return int(_lib.lib().rxb200_fm_max_output(C.c_void_p(self.member(0)), n_int16, chunk_int16))


# ---- several channels of one capture (rxb200_fm_mix_*) ------------------------------------------------------
def mix_table(capture_rate: int, offset_hz: int) -> np.ndarray:
    """The integer mixer of a channel offset_hz away from the centre of a capture at capture_rate:
    int32[period][2] of (c, s) in Q15 with unity 2^15 (``rxb200_fm_mix_table``)."""
    period = C.c_size_t(0)
    rc = _lib.lib().rxb200_fm_mix_table(capture_rate, offset_hz, None, 0, C.byref(period))
    if rc != _lib.ECAPACITY:
        _lib.check(rc)
    t = np.zeros((int(period.value), 2), dtype=np.int32)
    _lib.check(_lib.lib().rxb200_fm_mix_table(capture_rate, offset_hz, t.ctypes.data_as(C.POINTER(C.c_int32)), t.size,
                                              C.byref(period)))
    return t


def mix_device(capture_rate: int, offset_hz: int, phase: int, d_src_ptr: int, n_complex: int, d_dst_ptr: int,
               stream: int = 0) -> None:
    """The mixer alone on device pointers (``rxb200_mix_device``), asynchronous on ``stream``."""
    _lib.check(_lib.lib().rxb200_mix_device(capture_rate, offset_hz, phase, d_src_ptr, n_complex, d_dst_ptr,
                                            stream or None))


def _ddc_c(ddc):
    """(decim, taps, shift) -> (rxb200_ddc, the int32 taps it points at, to be kept alive for the call)."""
    decim, taps, shift = ddc
    t = np.ascontiguousarray(taps, dtype=np.int32).reshape(-1)
    return _lib.DdcC(int(decim), int(t.size), t.ctypes.data_as(C.POINTER(C.c_int32)), int(shift)), t


def ddc_device(capture_rate: int, offset_hz: int, phase: int, ddc, d_src_ptr: int, n_complex: int, d_dst_ptr: int,
               stream: int = 0) -> None:
    """The down-converter alone on device pointers (``rxb200_ddc_device``), asynchronous on ``stream``: zero samples
    before d_src, the mixer from entry phase mod L, floor(n_complex / decim) outputs.  ddc: (decim, taps, shift)."""
    d, _t = _ddc_c(ddc)
    _lib.check(_lib.lib().rxb200_ddc_device(capture_rate, offset_hz, phase, C.byref(d), d_src_ptr, n_complex, d_dst_ptr,
                                            stream or None))


def disc_device(form: int, quads, stream: int = 0):
    """One discriminator alone on the device (``rxb200_fm_disc_device``): quads is a contiguous int32 CUDA tensor
    [n][4] of (ar, aj, br, bj); returns the int32 [n] results, a new tensor on the same device, written asynchronously
    on ``stream``.  form: DISC_*."""
    assert quads.dim() == 2 and quads.shape[1] == 4 and quads.is_contiguous() and quads.element_size() == 4
    out = quads.new_empty((quads.shape[0],))
    _lib.check(_lib.lib().rxb200_fm_disc_device(form, quads.data_ptr(), quads.shape[0], out.data_ptr(), stream or None))
    return out


class FmMix(_OneGpu):
    """``len(offsets_hz)`` channels of ONE CS16 capture at ``capture_rate`` (``rxb200_fm_mix_*``): channel k is
    ``FmDemod`` run on the capture mixed down by ``offsets_hz[k]`` with ``mix_table``; the mixers' phases carry across
    calls.  Every call takes the one capture, int16[n_int16], and returns int16[n_channels][n_pcm].
    ddc = (decim, taps, shift): a decimating handle (``rxb200_fm_mix_create_ddc``), each channel filtered by the int32
    taps, rounded by the shift and decimated by decim before the chain."""

    _prefix = "rxb200_fm_mix"
    _streams = False
    _m = property(lambda self: self._h)     # the handle under the name callers of earlier releases read

    def __init__(self, params, capture_rate: int, offsets_hz, device: int = 0, ddc=None):
        self.params = FmParams.from_any(params)
        self.capture_rate = capture_rate
        offs = np.ascontiguousarray(offsets_hz, dtype=np.int32)
        self.offsets_hz = offs.tolist()
        self.n_channels = len(offs)
        self.ddc = ddc
        self._h = C.c_void_p()
        pc = self.params.to_c()
        if ddc is None:
            _lib.check(_lib.lib().rxb200_fm_mix_create(C.byref(pc), capture_rate, _ptr(offs), self.n_channels, device,
                                                       C.byref(self._h)))
        else:
            d, _t = _ddc_c(ddc)
            _lib.check(_lib.lib().rxb200_fm_mix_create_ddc(C.byref(pc), capture_rate, _ptr(offs), self.n_channels,
                                                           C.byref(d), device, C.byref(self._h)))

    def member(self) -> int:
        """The inner rxb200_fm handle (one channel per mixed stream) as an integer."""
        return int(_lib.lib().rxb200_fm_mix_member(self._h) or 0)

    def max_output(self, n_int16: int, chunk_int16: int = MAXIMUM_BUF_LENGTH) -> int:
        """A bound on the PCM per channel of a call of n_int16 capture int16, at any phase
        (``rxb200_fm_mix_max_output``)."""
        return int(_lib.lib().rxb200_fm_mix_max_output(self._h, n_int16, chunk_int16))

    _bound = max_output

    def decimated_len(self, n_int16: int) -> int:
        """int16 per channel the next call of n_int16 capture int16 hands the chain (``rxb200_fm_mix_decimated_len``)."""
        n = C.c_size_t(0)
        _lib.check(_lib.lib().rxb200_fm_mix_decimated_len(self._h, n_int16, C.byref(n)))
        return int(n.value)

    def stats(self) -> dict:
        s = _lib.FmStatsC()
        _lib.check(_lib.lib().rxb200_fm_last_stats(C.c_void_p(self.member()), C.byref(s)))
        return {f[0]: int(getattr(s, f[0])) for f in s._fields_}

    @property
    def stream(self) -> int:
        return int(_lib.lib().rxb200_fm_stream(C.c_void_p(self.member())) or 0)

    def mix_ms(self) -> float:
        """Device time of the last call's fm_mix_kernel (fm_ddc_kernel for a decimating handle)."""
        ms = C.c_float(0)
        _lib.check(_lib.lib().rxb200_fm_mix_kernel_ms(self._h, C.byref(ms)))
        return float(ms.value)

    def kernel_ms(self) -> float:
        """Device time of the last call's chain kernels (``rxb200_fm_kernel_ms`` of the member)."""
        ms = C.c_float(0)
        _lib.check(_lib.lib().rxb200_fm_kernel_ms(C.c_void_p(self.member()), C.byref(ms)))
        return float(ms.value)


class FmMixGroup(_Handle):
    """The channels of ONE capture split over several GPUs (``rxb200_fm_mix_group_*``): member i is a ``FmMix`` on its
    own GPU with a contiguous block of the offsets, and every member gets a copy of the capture; the group's results
    are byte for byte those of one ``FmMix`` with all the offsets.  devices: one CUDA ordinal per member (may repeat),
    or None for ``range(n_dev)``.  ddc = (decim, taps, shift): decimating members (``rxb200_fm_mix_group_create_ddc``),
    byte for byte one ``FmMix`` with that ddc."""

    _prefix = "rxb200_fm_mix_group"
    _streams = False
    _g = property(lambda self: self._h)     # the handle under the name callers of earlier releases read

    def __init__(self, params, capture_rate: int, offsets_hz, devices=None, n_dev: Optional[int] = None, ddc=None):
        self.params = FmParams.from_any(params)
        self.capture_rate = capture_rate
        offs = np.ascontiguousarray(offsets_hz, dtype=np.int32)
        self.offsets_hz = offs.tolist()
        self.n_channels = len(offs)
        self.ddc = ddc
        devs, self.n_dev = _devices(devices, n_dev)
        self._h = C.c_void_p()
        pc = self.params.to_c()
        if ddc is None:
            _lib.check(_lib.lib().rxb200_fm_mix_group_create(C.byref(pc), capture_rate, _ptr(offs), self.n_channels,
                                                             self.n_dev, _ptr(devs), C.byref(self._h)))
        else:
            d, _t = _ddc_c(ddc)
            _lib.check(_lib.lib().rxb200_fm_mix_group_create_ddc(C.byref(pc), capture_rate, _ptr(offs), self.n_channels,
                                                                 C.byref(d), self.n_dev, _ptr(devs), C.byref(self._h)))

    def member(self, i: int) -> int:
        """Member i's rxb200_fm_mix handle as an integer, 0 for a member that owns no channel."""
        return int(_lib.lib().rxb200_fm_mix_group_member(self._h, i) or 0)

    def inner(self, i: int) -> int:
        """The inner rxb200_fm handle of member i (``rxb200_fm_mix_member``), 0 for a member that owns no channel."""
        m = self.member(i)
        return int(_lib.lib().rxb200_fm_mix_member(C.c_void_p(m)) or 0) if m else 0

    def _bound(self, n_int16: int, chunk_int16: int) -> int:
        return int(_lib.lib().rxb200_fm_mix_max_output(C.c_void_p(self.member(0)), n_int16, chunk_int16))


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
