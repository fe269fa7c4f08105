"""rx_power path — host-side mirror of the reference's interface (src/rtl_power.c).

``plan_range`` is ``frequency_range()`` (:431-543), ``window_table``/``sine_table`` are the tables
``main()`` builds (:1028, :1034-1037), ``PowerScanner.scanner`` is n passes of ``scanner()`` (:670-772)
over hop buffers, executed by the batched sm_90a kernel behind ``rxb200_power_accumulate``
(include/rxb200.h); ``csv_rows`` is ``csv_dbm()`` (:774-817).  ``PowerMix`` takes every hop of a sweep from one
wideband capture through an NCO down-converter on the GPU (``rxb200_power_mix_*``); ``plan_tiles`` cuts a sweep wider
than one capture into tiles, each taken from one burst (``PowerMix.accumulate_burst``).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np

from . import _lib
from .fm import _ddc_c

WINDOWS = {"rectangle": 0, "hamming": 1, "blackman": 2, "blackman-harris": 3, "hann-poisson": 4,
           "youssef": 5, "kaiser": 6, "bartlett": 7, "hann": 8}


def atofs(s: str) -> float:
    """'k'/'M'/'G' suffixed number (convenience.c:65-90)."""
    s = s.strip()
    mult = {"g": 1e9, "G": 1e9, "m": 1e6, "M": 1e6, "k": 1e3, "K": 1e3}.get(s[-1:] if s else "", None)
    if mult is not None:
        return float(s[:-1]) * mult
    return float(s)


@dataclass
class Plan:
    n_hops: int
    bin_e: int
    buf_len: int
    downsample: int
    downsample_passes: int
    comp_fir_size: int
    boxcar: int
    peak_hold: int
    rate: int
    crop: float
    first_freq: int
    freq_step: int
    bin_size_hz: float

    def to_c(self) -> _lib.PowerParamsC:
        return _lib.PowerParamsC(self.n_hops, self.bin_e, self.buf_len, self.downsample, self.downsample_passes,
                                 self.comp_fir_size, self.boxcar, self.peak_hold)

    def hop_freq(self, i: int) -> int:
        return self.first_freq + i * self.freq_step


def plan_range(freq_arg: str, crop: float = 0.0, boxcar: int = 1, comp_fir_size: int = 0, peak_hold: int = 0) -> Plan:
    lo, hi, step = freq_arg.split(":")
    out = _lib.PowerPlanC()
    _lib.check(_lib.lib().rxb200_power_plan_range(int(atofs(lo)), int(atofs(hi)), int(atofs(step)), crop, boxcar,
                                                  comp_fir_size, peak_hold, C.byref(out)))
    p = out.params
    return Plan(p.n_hops, p.bin_e, p.buf_len, p.downsample, p.downsample_passes, p.comp_fir_size, p.boxcar,
                p.peak_hold, out.rate, out.crop, out.first_freq, out.freq_step, out.bin_size_hz)


def window_table(name_or_id, length: int) -> np.ndarray:
    wid = WINDOWS[name_or_id] if isinstance(name_or_id, str) else int(name_or_id)
    t = np.empty(length, dtype=np.int32)
    _lib.check(_lib.lib().rxb200_window_table(wid, length, t.ctypes.data_as(C.POINTER(C.c_int))))
    return t


def sine_table(log2_n: int) -> np.ndarray:
    t = np.empty(max((1 << log2_n) * 3 // 4, 1), dtype=np.int16)
    _lib.check(_lib.lib().rxb200_sine_table(log2_n, t.ctypes.data_as(C.POINTER(C.c_int16))))
    return t


class PowerScanner:
    def __init__(self, plan: Plan, window: Sequence[int] | str = "rectangle", device: int = 0,
                 sinewave: Optional[np.ndarray] = None):
        self.plan = plan
        n = 1 << plan.bin_e
        self.window = window_table(window, n) if isinstance(window, str) else np.ascontiguousarray(window, np.int32)
        assert self.window.size == n
        self._h = C.c_void_p()
        pc = plan.to_c()
        sw = None if sinewave is None else np.ascontiguousarray(sinewave, np.int16).ctypes.data_as(C.POINTER(C.c_int16))
        _lib.check(_lib.lib().rxb200_power_create(C.byref(pc), self.window.ctypes.data_as(C.POINTER(C.c_int)), sw,
                                                  device, C.byref(self._h)))

    def close(self) -> None:
        if _lib is not None and getattr(self, "_h", None) is not None and self._h:
            _lib.lib().rxb200_power_destroy(self._h)
            self._h = None

    __del__ = close

    def scanner(self, hop_bufs: np.ndarray, n_pass: int, hop_begin: int = 0, hop_end: Optional[int] = None) -> None:
        """hop_bufs: int16[n_pass][hop_end-hop_begin][buf_len] (host)."""
        hop_end = self.plan.n_hops if hop_end is None else hop_end
        hb = np.ascontiguousarray(hop_bufs, dtype=np.int16).reshape(-1)
        assert hb.size == n_pass * (hop_end - hop_begin) * self.plan.buf_len
        _lib.check(_lib.lib().rxb200_power_accumulate(self._h, hb.ctypes.data, n_pass, hop_begin, hop_end))

    def scanner_device(self, d_ptr: int, n_pass: int, hop_begin: int = 0, hop_end: Optional[int] = None,
                       sync: bool = False) -> None:
        hop_end = self.plan.n_hops if hop_end is None else hop_end
        _lib.check(_lib.lib().rxb200_power_accumulate_device(self._h, d_ptr, n_pass, hop_begin, hop_end,
                                                             1 if sync else 0))

    def read(self):
        n = 1 << self.plan.bin_e
        avg = np.zeros((self.plan.n_hops, n), dtype=np.int64)
        samples = np.zeros(self.plan.n_hops, dtype=np.int32)
        _lib.check(_lib.lib().rxb200_power_read(self._h, avg.ctypes.data_as(C.POINTER(C.c_int64)),
                                                samples.ctypes.data_as(C.POINTER(C.c_int))))
        return avg, samples

    def read_db(self):
        """csv_dbm's numbers computed on the device (src/rtl_power.c:783-811): float64[n_hops][row_len], samples."""
        row_len = _lib.check(_lib.lib().rxb200_power_row_len(self.plan.bin_e, self.plan.crop))
        db = np.zeros((self.plan.n_hops, row_len), dtype=np.float64)
        samples = np.zeros(self.plan.n_hops, dtype=np.int32)
        _lib.check(_lib.lib().rxb200_power_read_db(self._h, self.plan.rate, self.plan.crop,
                                                   db.ctypes.data_as(C.POINTER(C.c_double)), row_len,
                                                   samples.ctypes.data_as(C.POINTER(C.c_int))))
        return db, samples

    def csv_rows_device(self, tstr: str = "2026-01-01, 00:00:00") -> str:
        """The CSV text of csv_dbm() over every hop with the dB values computed on the device."""
        db, samples = self.read_db()
        buf = C.create_string_buffer(64 + 16 * (db.shape[1] + 8))
        lines = []
        for i in range(self.plan.n_hops):
            row = np.ascontiguousarray(db[i])
            r = _lib.check(_lib.lib().rxb200_power_format_db_row(row.ctypes.data_as(C.POINTER(C.c_double)), self.plan.bin_e,
                                                                 self.plan.hop_freq(i), self.plan.rate, self.plan.downsample,
                                                                 self.plan.crop, int(samples[i]), buf, len(buf)))
            lines.append(tstr + ", " + buf.raw[:r].decode())
        return "".join(lines)

    def reset(self) -> None:
        _lib.check(_lib.lib().rxb200_power_reset(self._h))

    def last_path(self) -> dict:
        """What the last scanner call ran (rxb200_power_last_path): kernel is one of "none", "rms", "fft8", "generic",
        "big_load", "big_decim"."""
        out = _lib.PowerPathC()
        _lib.check(_lib.lib().rxb200_power_last_path(self._h, C.byref(out)))
        d = {n: int(getattr(out, n)) for n, _ in out._fields_}
        d["kernel"] = _lib.POWER_PATHS[d["kernel"]]
        return d

    def kernel_ms(self) -> float:
        ms = C.c_float(0)
        _lib.check(_lib.lib().rxb200_power_kernel_ms(self._h, C.byref(ms)))
        return float(ms.value)

    def gather(self, comm: "Comm", sync: bool = True) -> None:
        """The collation before the report (src/rtl_power.c:1047-1050 walks every hop): ONE in-place NCCL all-gather of
        the accumulator rows inside the library; afterwards read()/read_db() see every rank's hops."""
        _lib.check(_lib.lib().rxb200_power_gather(self._h, comm._c, 1 if sync else 0))

    @property
    def device_avg_ptr(self) -> int:
        return int(_lib.lib().rxb200_power_device_avg(self._h) or 0)

    @property
    def stream(self) -> int:
        return int(_lib.lib().rxb200_power_stream(self._h) or 0)

    def csv_rows(self, avg: np.ndarray, samples: np.ndarray, tstr: str = "2026-01-01, 00:00:00") -> str:
        """csv_dbm() over every hop (src/rtl_power.c:1047-1050): returns the CSV text."""
        return csv_rows(self.plan, avg, samples, tstr)


def csv_rows(plan: Plan, avg: np.ndarray, samples: np.ndarray, tstr: str = "2026-01-01, 00:00:00") -> str:
    n = 1 << plan.bin_e
    buf = C.create_string_buffer(64 + 16 * (n + 8))
    lines = []
    a = np.array(avg, dtype=np.int64, copy=True).reshape(plan.n_hops, n)
    for i in range(plan.n_hops):
        row = np.ascontiguousarray(a[i])
        r = _lib.check(_lib.lib().rxb200_power_format_row(row.ctypes.data_as(C.POINTER(C.c_int64)), plan.bin_e,
                                                          plan.hop_freq(i), plan.rate, plan.downsample, plan.crop,
                                                          int(samples[i]), buf, len(buf)))
        lines.append(tstr + ", " + buf.raw[:r].decode())
    return "".join(lines)


class PowerMix(PowerScanner):
    """Every hop of a sweep from ONE wideband capture (``rxb200_power_mix_*``): hop i is the capture mixed down by
    offsets_hz[i] with a phase-accumulator NCO, filtered and decimated by ddc = (M, taps, S), and every buf_len / 2
    outputs of it are one hop buffer of the inner rx_power handle (the member).  read, read_db, csv_rows_device and
    last_path are the member's; reset() brings the whole handle back to create, reset_accumulators() zeroes only the
    accumulators (the phases and the filter history carry on, as across the reports of a continuous capture)."""

    def __init__(self, plan: Plan, capture_rate: int, offsets_hz: Sequence[int], ddc,
                 window: Sequence[int] | str = "rectangle", device: int = 0, sinewave: Optional[np.ndarray] = None):
        self.plan = plan
        n = 1 << plan.bin_e
        self.window = window_table(window, n) if isinstance(window, str) else np.ascontiguousarray(window, np.int32)
        assert self.window.size == n
        self.capture_rate, self.ddc = int(capture_rate), ddc
        self.offsets = np.ascontiguousarray(offsets_hz, dtype=np.int32)
        assert self.offsets.size == plan.n_hops
        self._m = C.c_void_p()
        pc = plan.to_c()
        d, _t = _ddc_c(ddc)
        sw = None if sinewave is None else np.ascontiguousarray(sinewave, np.int16).ctypes.data_as(C.POINTER(C.c_int16))
        _lib.check(_lib.lib().rxb200_power_mix_create(C.byref(pc), self.window.ctypes.data_as(C.POINTER(C.c_int)), sw,
                                                      self.capture_rate,
                                                      self.offsets.ctypes.data_as(C.POINTER(C.c_int)), C.byref(d),
                                                      device, C.byref(self._m)))
        self._h = C.c_void_p(_lib.lib().rxb200_power_mix_member(self._m))

    def close(self) -> None:
        if _lib is not None and getattr(self, "_m", None) is not None and self._m:
            _lib.lib().rxb200_power_mix_destroy(self._m)
            self._m = None
            self._h = None

    __del__ = close

    @property
    def pass_int16(self) -> int:
        """Capture int16 per pass: decim * buf_len."""
        return int(self.ddc[0]) * self.plan.buf_len

    def accumulate(self, capture: np.ndarray) -> None:
        """capture: int16 CS16 (host), a whole number of passes; uint8 bytes after set_input_format(CS8, CU8, CS12)."""
        x, n_int16 = _lib.in_array(capture, getattr(self, "_in_fmt", _lib.IN_CS16))
        _lib.check(_lib.lib().rxb200_power_mix_accumulate(self._m, x.ctypes.data, n_int16))

    def accumulate_device(self, d_ptr: int, n_int16: int, sync: bool = False) -> None:
        _lib.check(_lib.lib().rxb200_power_mix_accumulate_device(self._m, d_ptr, n_int16, 1 if sync else 0))

    def reset(self) -> None:
        _lib.check(_lib.lib().rxb200_power_mix_reset(self._m))

    def reset_accumulators(self) -> None:
        _lib.check(_lib.lib().rxb200_power_reset(self._h))

    def set_device_rate(self, up: int, down: int, taps, shift: int = 15) -> None:
        """Attach a resampler right after create or reset (``rxb200_power_mix_set_device_rate``): from then on every
        accumulate takes device-rate CS16 that resamples to whole passes."""
        from .resample import _rs_c
        rs, _t = _rs_c(up, down, taps, shift)
        _lib.check(_lib.lib().rxb200_power_mix_set_device_rate(self._m, C.byref(rs)))

    def set_input_format(self, fmt) -> None:
        """The capture's format right after create or reset (``rxb200_power_mix_set_input_format``): ``_lib.IN_*`` or
        its name.  From then on every accumulate and burst takes the format's raw bytes (uint8) for CS8, CU8 and CS12,
        widened to CS16 on the GPU; n_int16 still counts two per complex element."""
        fmt = _lib.IN_FORMATS.get(fmt, fmt)
        _lib.check(_lib.lib().rxb200_power_mix_set_input_format(self._m, fmt))
        self._in_fmt = fmt

    def set_burst_device_rate(self, up: int, down: int, taps, shift: int = 15) -> None:
        """Attach a resampler for bursts only, right after create or reset (``rxb200_power_mix_set_burst_device_rate``):
        from then on every burst is device-rate CS16 (``burst_in_len``), resampled statelessly with its first
        ceil((J - 1) L / N) outputs dropped; accumulate still takes capture-rate samples."""
        from .resample import _rs_c
        rs, _t = _rs_c(up, down, taps, shift)
        _lib.check(_lib.lib().rxb200_power_mix_set_burst_device_rate(self._m, C.byref(rs)))

    def burst_in_len(self, n_pass: int = 1) -> int:
        """int16 of one burst of n_pass passes as the handle takes it (``rxb200_power_mix_burst_in_len``): device int16
        with a burst device rate, else burst_int16(n_pass)."""
        n = C.c_size_t(0)
        _lib.check(_lib.lib().rxb200_power_mix_burst_in_len(self._m, int(n_pass), C.byref(n)))
        return int(n.value)

    def kernel_ms(self) -> float:
        """Device time of the last call's DDC launches (ms)."""
        ms = C.c_float(0)
        _lib.check(_lib.lib().rxb200_power_mix_kernel_ms(self._m, C.byref(ms)))
        return float(ms.value)

    def accumulate_ms(self) -> float:
        """Device time of the member's last accumulate kernel (ms)."""
        return PowerScanner.kernel_ms(self)

    @property
    def lead(self) -> int:
        """G = M ceil((T - 1) / M): the complex samples at the front of a burst that prime the filter."""
        return _lib.check(_lib.lib().rxb200_power_mix_lead(self._m))

    def burst_int16(self, n_pass: int = 1) -> int:
        """Capture int16 of a burst of n_pass passes: 2 G + n_pass M buf_len."""
        return 2 * self.lead + n_pass * self.pass_int16

    def accumulate_burst(self, hop_begin: int, hop_end: int, capture: np.ndarray) -> None:
        """One burst (host int16 CS16: the lead, then whole passes) for hops [hop_begin, hop_end).  The handle's
        carried phases and filter history are left as they are."""
        x, n_int16 = _lib.in_array(capture, getattr(self, "_in_fmt", _lib.IN_CS16))
        _lib.check(_lib.lib().rxb200_power_mix_accumulate_burst(self._m, hop_begin, hop_end, x.ctypes.data, n_int16))

    def accumulate_burst_device(self, hop_begin: int, hop_end: int, d_ptr: int, n_int16: int,
                                sync: bool = False) -> None:
        _lib.check(_lib.lib().rxb200_power_mix_accumulate_burst_device(self._m, hop_begin, hop_end, d_ptr, n_int16,
                                                                       1 if sync else 0))


@dataclass
class Tiling:
    """rxb200_power_tiling: n_tiles tiles of up to hops_per_tile hops, each taken from one capture at capture_rate
    (decim times the hop rate) through a filter of n_taps taps."""
    n_tiles: int
    hops_per_tile: int
    decim: int
    n_taps: int
    capture_rate: int


def _plan_c(plan: Plan) -> _lib.PowerPlanC:
    return _lib.PowerPlanC(plan.to_c(), plan.rate, plan.crop, plan.first_freq, plan.freq_step, plan.bin_size_hz)


def _power_plan_call(name: str, pc, max_rate: int, device_rate: Optional[int], out, offs) -> None:
    """``name`` without a device rate, ``name_at`` (the guard band in the decimation floor) with one."""
    args = [C.byref(pc), int(max_rate)]
    if device_rate is not None:
        name += "_at"
        args.append(int(device_rate))
    _lib.check(getattr(_lib.lib(), name)(*args, C.byref(out), offs.ctypes.data_as(C.POINTER(C.c_int))))


def plan_capture(plan: Plan, max_rate: int, device_rate: Optional[int] = None):
    """The rx_power shell's capture-mode plan (``rxb200_power_plan_capture``, or ``_at`` with a device_rate):
    (fm.CapturePlan of the centre, M, R = M rate and T, each hop's offset from the centre)."""
    from .fm import CapturePlan
    out = _lib.FmCapturePlanC()
    offs = np.zeros(plan.n_hops, dtype=np.int32)
    _power_plan_call("rxb200_power_plan_capture", _plan_c(plan), max_rate, device_rate, out, offs)
    return CapturePlan(int(out.centre_hz), out.decim, out.capture_rate, out.n_taps), [int(v) for v in offs]


def plan_tiles(plan: Plan, max_rate: int, device_rate: Optional[int] = None):
    """The tiling of a sweep for captures of at most max_rate Hz (``rxb200_power_plan_tiles``, or ``_at`` with a
    device_rate, whose tiles shrink to fit it): (Tiling, each tile's (hop_begin, hop_end, centre_hz), each hop's offset
    from its tile's centre)."""
    pc = _plan_c(plan)
    tl = _lib.PowerTilingC()
    offs = np.zeros(plan.n_hops, dtype=np.int32)
    _power_plan_call("rxb200_power_plan_tiles", pc, max_rate, device_rate, tl, offs)
    tiles = []
    for t in range(tl.n_tiles):
        b, e, c = C.c_int(0), C.c_int(0), C.c_int64(0)
        _lib.check(_lib.lib().rxb200_power_tile(C.byref(pc), C.byref(tl), t, C.byref(b), C.byref(e), C.byref(c)))
        tiles.append((b.value, e.value, c.value))
    return (Tiling(tl.n_tiles, tl.hops_per_tile, tl.decim, tl.n_taps, tl.capture_rate), tiles,
            [int(v) for v in offs])


def nco_table() -> np.ndarray:
    """The NCO table (``rxb200_nco_table``): int32[65536][2] of (c, s)."""
    t = np.empty((65536, 2), dtype=np.int32)
    _lib.check(_lib.lib().rxb200_nco_table(t.ctypes.data_as(C.POINTER(C.c_int32))))
    return t


def ddc_lowpass(decim: int, n_taps: int, shift: int) -> np.ndarray:
    """The capture mode's channel filter (``rxb200_ddc_lowpass``): int32[n_taps] summing to 2^shift."""
    t = np.empty(n_taps, dtype=np.int32)
    _lib.check(_lib.lib().rxb200_ddc_lowpass(decim, n_taps, shift, t.ctypes.data_as(C.POINTER(C.c_int32))))
    return t


def power_ddc_device(capture_rate: int, offset_hz: int, n0: int, ddc, d_src_ptr: int, n_complex: int, d_dst_ptr: int,
                     stream: int = 0) -> None:
    """The NCO down-converter alone on device pointers (``rxb200_power_ddc_device``), asynchronous on ``stream``: zero
    samples before d_src, d_src[i] is capture sample n0 + i, floor(n_complex / decim) outputs.  ddc: (decim, taps, S)."""
    d, _t = _ddc_c(ddc)
    _lib.check(_lib.lib().rxb200_power_ddc_device(capture_rate, offset_hz, n0, C.byref(d), d_src_ptr, n_complex,
                                                  d_dst_ptr, stream or None))


def shard(n_hops: int, n_ranks: int, rank: int):
    """Contiguous hop range [begin, end) of `rank` (rxb200_power_shard)."""
    b, e = C.c_int(0), C.c_int(0)
    _lib.check(_lib.lib().rxb200_power_shard(n_hops, n_ranks, rank, C.byref(b), C.byref(e)))
    return b.value, e.value


class Comm:
    """One rank's NCCL communicator, owned by librxb200 (include/rxb200.h: rxb200_comm_*)."""

    def __init__(self, n_ranks: int, rank: int, unique_id: bytes, device: int):
        assert len(unique_id) == 128
        self._c = C.c_void_p()
        buf = C.create_string_buffer(unique_id, 128)
        _lib.check(_lib.lib().rxb200_comm_create(n_ranks, rank, buf, device, C.byref(self._c)))
        self.n_ranks, self.rank = n_ranks, rank

    @staticmethod
    def unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        _lib.check(_lib.lib().rxb200_comm_unique_id(buf))
        return buf.raw

    def close(self) -> None:
        if _lib is not None and getattr(self, "_c", None) is not None and self._c:
            _lib.lib().rxb200_comm_destroy(self._c)
            self._c = None

    __del__ = close


class PowerGroup:
    """All ranks in one process: n_dev GPUs, hops sharded, one all-gather before the report (what the drop-in
    rx_power_b200 shell uses when RXB200_GPUS > 1)."""

    def __init__(self, plan: Plan, window: Sequence[int] | str = "rectangle", n_dev: int = 1):
        self.plan = plan
        n = 1 << plan.bin_e
        self.window = window_table(window, n) if isinstance(window, str) else np.ascontiguousarray(window, np.int32)
        self._g = C.c_void_p()
        pc = plan.to_c()
        _lib.check(_lib.lib().rxb200_power_group_create(C.byref(pc), self.window.ctypes.data_as(C.POINTER(C.c_int)), None,
                                                        n_dev, None, C.byref(self._g)))
        self.n_dev = n_dev

    def close(self) -> None:
        if _lib is not None and getattr(self, "_g", None) is not None and self._g:
            _lib.lib().rxb200_power_group_destroy(self._g)
            self._g = None

    __del__ = close

    def scanner(self, hop_bufs: np.ndarray, n_pass: int, hop_begin: int = 0, hop_end: Optional[int] = None) -> None:
        hop_end = self.plan.n_hops if hop_end is None else hop_end
        hb = np.ascontiguousarray(hop_bufs, dtype=np.int16).reshape(-1)
        assert hb.size == n_pass * (hop_end - hop_begin) * self.plan.buf_len
        _lib.check(_lib.lib().rxb200_power_group_accumulate(self._g, hb.ctypes.data, n_pass, hop_begin, hop_end))

    def gather(self) -> None:
        _lib.check(_lib.lib().rxb200_power_group_gather(self._g))

    def read(self, member: int = 0):
        n = 1 << self.plan.bin_e
        avg = np.zeros((self.plan.n_hops, n), dtype=np.int64)
        samples = np.zeros(self.plan.n_hops, dtype=np.int32)
        h = _lib.lib().rxb200_power_group_member(self._g, member)
        _lib.check(_lib.lib().rxb200_power_read(h, avg.ctypes.data_as(C.POINTER(C.c_int64)),
                                                samples.ctypes.data_as(C.POINTER(C.c_int))))
        return avg, samples

    def reset(self) -> None:
        _lib.check(_lib.lib().rxb200_power_group_reset(self._g))
