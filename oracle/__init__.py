"""oracle — CPU checkers for the rx_tools hot path.  TEST INFRASTRUCTURE ONLY.

Two implementations behind one Python face:

* ``port``  (``librx_oracle.so``, built from ``rx_oracle.c``): our own plain-C restatement of
  the reference algorithm; always buildable, travels to the GPU box.
* ``ref``   (``_ref/libref_fm.so`` / ``_ref/libref_power.so``): the UNMODIFIED reference
  sources compiled where they lie under ``/root/reference`` (``oracle/Makefile``); exists
  only if it was built in the authoring container (the built files travel with gpurun).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl
reference`` legs may import this package.  The product (``rx_tools_b200``) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass, fields
from typing import Optional, Sequence

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PORT_SO = os.path.join(HERE, "librx_oracle.so")
REF_FM_SO = os.path.join(HERE, "_ref", "libref_fm.so")
REF_POWER_SO = os.path.join(HERE, "_ref", "libref_power.so")
REF_SDR_BIN = os.path.join(HERE, "_ref", "rx_sdr_ref")
REFERENCE_ROOT = "/root/reference"

MODE_FM, MODE_AM, MODE_USB, MODE_LSB, MODE_RAW = range(5)
ATAN_STD, ATAN_FAST, ATAN_LUT, ATAN_ALE = range(4)


def build(force: bool = False) -> None:
    """Compile the port (always) and the reference harness (when /root/reference exists)."""
    args = ["make", "-C", HERE, "-s"]
    if force:
        args.append("-B")
    subprocess.run(args + ["librx_oracle.so"], check=True)
    if os.path.exists(os.path.join(REFERENCE_ROOT, "src", "rtl_fm.c")):
        subprocess.run(args + ["ref"], check=True)


def have_ref() -> bool:
    return os.path.exists(REF_FM_SO) and os.path.exists(REF_POWER_SO)


class FmParamsC(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "mode", "downsample", "downsample_passes", "comp_fir_size", "custom_atan", "output_scale",
        "post_downsample", "deemph", "deemph_a", "rate_out", "rate_out2", "squelch_level",
        "dc_block_audio", "adc_block_const", "dc_block_raw", "rdc_block_const", "offset_tuning")]


@dataclass
class FmParams:
    """Derived rx_fm DSP parameters = the demod_state config fields (src/rtl_fm.c:124-159)."""
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

    def to_c(self) -> FmParamsC:
        return FmParamsC(*[int(getattr(self, f.name)) for f in fields(self)])

    @classmethod
    def from_c(cls, c: FmParamsC) -> "FmParams":
        return cls(**{f.name: int(getattr(c, f.name)) for f in fields(cls)})


class PowerParamsC(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "bin_e", "buf_len", "downsample", "downsample_passes", "comp_fir_size", "boxcar", "peak_hold")]


@dataclass
class PowerParams:
    bin_e: int
    buf_len: int = 16384
    downsample: int = 1
    downsample_passes: int = 0
    comp_fir_size: int = 0
    boxcar: int = 1
    peak_hold: int = 0

    def to_c(self) -> PowerParamsC:
        return PowerParamsC(*[int(getattr(self, f.name)) for f in fields(self)])


class RefPlanC(C.Structure):
    _fields_ = [("tune_count", C.c_int), ("bin_e", C.c_int), ("buf_len", C.c_int),
                ("downsample", C.c_int), ("downsample_passes", C.c_int), ("rate", C.c_int),
                ("crop", C.c_double)]


def _i16(a) -> np.ndarray:
    a = np.ascontiguousarray(a, dtype=np.int16)
    return a


def _p16(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_int16))


WINDOWS = {"rectangle": 0, "hamming": 1, "blackman": 2, "blackman-harris": 3, "hann-poisson": 4,
           "youssef": 5, "kaiser": 6, "bartlett": 7, "hann": 8}


# --------------------------------------------------------------------------- port
class Port:
    """ctypes face of librx_oracle.so (rx_oracle.c)."""

    def __init__(self) -> None:
        if not os.path.exists(PORT_SO):
            build()
        L = C.CDLL(PORT_SO)
        L.orx_fm_new.restype = C.c_void_p
        L.orx_fm_new.argtypes = [C.POINTER(FmParamsC)]
        L.orx_fm_free.argtypes = [C.c_void_p]
        L.orx_fm_run.restype = C.c_long
        L.orx_fm_run.argtypes = [C.c_void_p, C.POINTER(C.c_int16), C.c_size_t, C.c_size_t,
                                 C.POINTER(C.c_int16), C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.orx_fm_run_levels.restype = C.c_long
        L.orx_fm_run_levels.argtypes = [C.c_void_p, C.POINTER(C.c_int16), C.c_size_t, C.c_size_t, C.POINTER(C.c_int)]
        L.orx_fm_time.restype = C.c_double
        L.orx_fm_time.argtypes = [C.c_void_p, C.POINTER(C.c_int16), C.c_size_t, C.c_size_t, C.c_int,
                                  C.POINTER(C.c_long)]
        L.orx_scale_sample.restype = C.c_int16
        L.orx_scale_sample.argtypes = [C.c_int16]
        L.orx_deemph_a.restype = C.c_int
        L.orx_deemph_a.argtypes = [C.c_int, C.c_int]
        L.orx_build_atan_table.argtypes = [C.POINTER(C.c_int)]
        L.orx_droop9.argtypes = [C.c_int, C.POINTER(C.c_int)]
        L.orx_sine_table.argtypes = [C.c_int, C.POINTER(C.c_int16)]
        L.orx_window_table.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_int)]
        L.orx_fix_fft.restype = C.c_int
        L.orx_fix_fft.argtypes = [C.POINTER(C.c_int16), C.c_int, C.POINTER(C.c_int16), C.c_int]
        L.orx_power_scan.argtypes = [C.POINTER(PowerParamsC), C.POINTER(C.c_int), C.POINTER(C.c_int16),
                                     C.POINTER(C.c_int16), C.c_int, C.c_int,
                                     C.POINTER(C.c_int64), C.POINTER(C.c_int)]
        L.orx_power_time.restype = C.c_double
        L.orx_power_time.argtypes = L.orx_power_scan.argtypes + [C.c_int]
        for name in ("orx_disc_std", "orx_disc_fast", "orx_disc_ale"):
            getattr(L, name).restype = C.c_int
            getattr(L, name).argtypes = [C.c_int] * 4
        L.orx_fast_atan2.restype = C.c_int
        L.orx_fast_atan2.argtypes = [C.c_int, C.c_int]
        self.L = L

    # ---- rx_fm
    def fm_run(self, params: FmParams, cs16: np.ndarray, chunk_int16: int = 262144,
               return_chunks: bool = False):
        x = _i16(cs16)
        pc = params.to_c()
        h = self.L.orx_fm_new(C.byref(pc))
        n_chunks = (x.size + chunk_int16 - 1) // chunk_int16
        out = np.empty(x.size + 64, dtype=np.int16)
        lens = np.zeros(max(n_chunks, 1), dtype=np.int32)
        hits = np.zeros(max(n_chunks, 1), dtype=np.int32)
        try:
            n = self.L.orx_fm_run(h, _p16(x), x.size, chunk_int16, _p16(out), out.size,
                                  lens.ctypes.data_as(C.POINTER(C.c_int)),
                                  hits.ctypes.data_as(C.POINTER(C.c_int)))
        finally:
            self.L.orx_fm_free(h)
        if n < 0:
            raise RuntimeError(f"orx_fm_run failed: {n}")
        res = out[:n].copy()
        return (res, lens[:n_chunks], hits[:n_chunks]) if return_chunks else res

    def fm_levels(self, params: FmParams, cs16: np.ndarray, chunk_int16: int = 262144) -> np.ndarray:
        """Per-chunk rms() that feeds the -L statistics (src/rtl_fm.c:792-806)."""
        x = _i16(cs16)
        pc = params.to_c()
        h = self.L.orx_fm_new(C.byref(pc))
        n_chunks = (x.size + chunk_int16 - 1) // chunk_int16
        lv = np.zeros(max(n_chunks, 1), dtype=np.int32)
        try:
            n = self.L.orx_fm_run_levels(h, _p16(x), x.size, chunk_int16, lv.ctypes.data_as(C.POINTER(C.c_int)))
        finally:
            self.L.orx_fm_free(h)
        if n < 0:
            raise RuntimeError(f"orx_fm_run_levels failed: {n}")
        return lv[:n_chunks]

    def fm_time(self, params: FmParams, cs16: np.ndarray, chunk_int16: int, repeats: int = 1) -> float:
        x = _i16(cs16)
        pc = params.to_c()
        h = self.L.orx_fm_new(C.byref(pc))
        nout = C.c_long(0)
        try:
            return float(self.L.orx_fm_time(h, _p16(x), x.size, chunk_int16, repeats, C.byref(nout)))
        finally:
            self.L.orx_fm_free(h)

    def scale_table(self) -> np.ndarray:
        """scaled value for every int16 input, index = x + 32768."""
        return np.array([self.L.orx_scale_sample(v) for v in range(-32768, 32768)], dtype=np.int16)

    def atan_table(self) -> np.ndarray:
        t = np.empty(131072, dtype=np.int32)
        self.L.orx_build_atan_table(t.ctypes.data_as(C.POINTER(C.c_int)))
        return t

    def droop9(self, row: int) -> np.ndarray:
        t = np.zeros(10, dtype=np.int32)
        if self.L.orx_droop9(row, t.ctypes.data_as(C.POINTER(C.c_int))) != 0:
            raise ValueError(row)
        return t

    def deemph_a(self, rate_out: int, tc_us: int = 75) -> int:
        return int(self.L.orx_deemph_a(rate_out, tc_us))

    # ---- rx_power
    def sine_table(self, log2n: int) -> np.ndarray:
        t = np.empty((1 << log2n) * 3 // 4, dtype=np.int16)
        self.L.orx_sine_table(log2n, _p16(t))
        return t

    def window_table(self, name_or_id, length: int) -> np.ndarray:
        wid = WINDOWS[name_or_id] if isinstance(name_or_id, str) else int(name_or_id)
        t = np.empty(length, dtype=np.int32)
        self.L.orx_window_table(wid, length, t.ctypes.data_as(C.POINTER(C.c_int)))
        return t

    def fix_fft(self, iq: np.ndarray, m: int, log2_wave: Optional[int] = None) -> np.ndarray:
        log2_wave = m if log2_wave is None else log2_wave
        buf = _i16(iq).copy()
        sine = self.sine_table(log2_wave)
        r = self.L.orx_fix_fft(_p16(buf), m, _p16(sine), log2_wave)
        if r != 0:
            raise RuntimeError("fix_fft size")
        return buf

    def power_scan(self, params: PowerParams, window: np.ndarray, hop_bufs: np.ndarray,
                   n_pass: int, n_hops: int, avg: Optional[np.ndarray] = None,
                   samples: Optional[np.ndarray] = None, sine: Optional[np.ndarray] = None):
        """sine: a caller's Sinewave table (3N/4 int16), else the one sine_table() builds."""
        n = 1 << params.bin_e
        hb = _i16(hop_bufs).reshape(-1)
        assert hb.size == n_pass * n_hops * params.buf_len
        win = np.ascontiguousarray(window, dtype=np.int32)
        if sine is None:
            sine = self.sine_table(max(params.bin_e, 1))
        else:
            sine = _i16(sine)
            assert sine.size >= n * 3 // 4
        avg = np.zeros((n_hops, n), dtype=np.int64) if avg is None else avg
        samples = np.zeros(n_hops, dtype=np.int32) if samples is None else samples
        pc = params.to_c()
        self.L.orx_power_scan(C.byref(pc), win.ctypes.data_as(C.POINTER(C.c_int)), _p16(sine), _p16(hb),
                              n_pass, n_hops, avg.ctypes.data_as(C.POINTER(C.c_int64)),
                              samples.ctypes.data_as(C.POINTER(C.c_int)))
        return avg, samples

    def power_time(self, params: PowerParams, window: np.ndarray, hop_bufs: np.ndarray,
                   n_pass: int, n_hops: int, repeats: int = 1) -> float:
        n = 1 << params.bin_e
        hb = _i16(hop_bufs).reshape(-1)
        win = np.ascontiguousarray(window, dtype=np.int32)
        sine = self.sine_table(max(params.bin_e, 1))
        avg = np.zeros((n_hops, n), dtype=np.int64)
        samples = np.zeros(n_hops, dtype=np.int32)
        pc = params.to_c()
        return float(self.L.orx_power_time(C.byref(pc), win.ctypes.data_as(C.POINTER(C.c_int)), _p16(sine),
                                           _p16(hb), n_pass, n_hops,
                                           avg.ctypes.data_as(C.POINTER(C.c_int64)),
                                           samples.ctypes.data_as(C.POINTER(C.c_int)), repeats))


# --------------------------------------------------------------------------- reference
class RefFm:
    """ctypes face of _ref/libref_fm.so — the unmodified reference rx_fm DSP.  The reference keeps
    its state in globals, so one process can host ONE stream at a time; ``run`` reconfigures."""

    def __init__(self) -> None:
        L = C.CDLL(REF_FM_SO)
        L.ref_fm_configure.argtypes = [C.POINTER(FmParamsC)]
        L.ref_fm_run.restype = C.c_long
        L.ref_fm_run.argtypes = [C.POINTER(C.c_int16), C.c_size_t, C.c_size_t, C.POINTER(C.c_int16),
                                 C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.ref_fm_run_levels.restype = C.c_long
        L.ref_fm_run_levels.argtypes = [C.POINTER(C.c_int16), C.c_size_t, C.c_size_t, C.POINTER(C.c_int)]
        L.ref_fm_time.restype = C.c_double
        L.ref_fm_time.argtypes = [C.POINTER(C.c_int16), C.c_size_t, C.c_size_t, C.c_int, C.POINTER(C.c_long)]
        L.ref_fm_derive.argtypes = [C.c_int] * 11 + [C.POINTER(FmParamsC), C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.ref_fm_atan_lut.restype = C.c_int
        L.ref_fm_atan_lut.argtypes = [C.POINTER(C.c_int), C.c_int]
        L.ref_fm_cic9.argtypes = [C.c_int, C.POINTER(C.c_int)]
        self.L = L

    def run(self, params: FmParams, cs16: np.ndarray, chunk_int16: int = 262144, return_chunks: bool = False):
        x = _i16(cs16)
        pc = params.to_c()
        if self.L.ref_fm_configure(C.byref(pc)) != 0:
            raise ValueError("bad params")
        n_chunks = (x.size + chunk_int16 - 1) // chunk_int16
        out = np.empty(x.size + 64, dtype=np.int16)
        lens = np.zeros(max(n_chunks, 1), dtype=np.int32)
        hits = np.zeros(max(n_chunks, 1), dtype=np.int32)
        n = self.L.ref_fm_run(_p16(x), x.size, chunk_int16, _p16(out), out.size,
                              lens.ctypes.data_as(C.POINTER(C.c_int)), hits.ctypes.data_as(C.POINTER(C.c_int)))
        if n < 0:
            raise RuntimeError(f"ref_fm_run failed: {n}")
        res = out[:n].copy()
        return (res, lens[:n_chunks], hits[:n_chunks]) if return_chunks else res

    def levels(self, params: FmParams, cs16: np.ndarray, chunk_int16: int = 262144) -> np.ndarray:
        x = _i16(cs16)
        pc = params.to_c()
        if self.L.ref_fm_configure(C.byref(pc)) != 0:
            raise ValueError("bad params")
        n_chunks = (x.size + chunk_int16 - 1) // chunk_int16
        lv = np.zeros(max(n_chunks, 1), dtype=np.int32)
        n = self.L.ref_fm_run_levels(_p16(x), x.size, chunk_int16, lv.ctypes.data_as(C.POINTER(C.c_int)))
        if n < 0:
            raise RuntimeError(f"ref_fm_run_levels failed: {n}")
        return lv[:n_chunks]

    def time(self, params: FmParams, cs16: np.ndarray, chunk_int16: int, repeats: int = 1) -> float:
        x = _i16(cs16)
        pc = params.to_c()
        self.L.ref_fm_configure(C.byref(pc))
        nout = C.c_long(0)
        return float(self.L.ref_fm_time(_p16(x), x.size, chunk_int16, repeats, C.byref(nout)))

    def derive(self, mode=MODE_FM, rate_s=0, rate_r=0, use_F=0, comp_fir_size=0, custom_atan=-1,
               post_downsample=1, deemph=-1, time_constant_us=75, wbfm=0, offset_tuning=0):
        out = FmParamsC()
        cap = C.c_int(0)
        off = C.c_int(0)
        self.L.ref_fm_derive(mode, rate_s, rate_r, use_F, comp_fir_size, custom_atan, post_downsample,
                             deemph, time_constant_us, wbfm, offset_tuning, C.byref(out), C.byref(cap), C.byref(off))
        return FmParams.from_c(out), int(cap.value), int(off.value)

    def atan_table(self) -> np.ndarray:
        t = np.empty(131072, dtype=np.int32)
        self.L.ref_fm_atan_lut(t.ctypes.data_as(C.POINTER(C.c_int)), t.size)
        return t

    def cic9(self, row: int) -> np.ndarray:
        t = np.zeros(10, dtype=np.int32)
        self.L.ref_fm_cic9(row, t.ctypes.data_as(C.POINTER(C.c_int)))
        return t


class RefPower:
    """ctypes face of _ref/libref_power.so — the unmodified reference rx_power scanner."""

    def __init__(self) -> None:
        L = C.CDLL(REF_POWER_SO)
        L.ref_power_setup.argtypes = [C.c_char_p, C.c_double, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.POINTER(C.c_int), C.POINTER(RefPlanC)]
        L.ref_power_tables.restype = C.c_int
        L.ref_power_tables.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_int16)]
        L.ref_power_scan.argtypes = [C.POINTER(C.c_int16), C.c_int]
        L.ref_power_time.restype = C.c_double
        L.ref_power_time.argtypes = [C.POINTER(C.c_int16), C.c_int, C.c_int]
        L.ref_power_get.argtypes = [C.POINTER(C.c_int64), C.POINTER(C.c_int)]
        L.ref_power_hop_freq.restype = C.c_longlong
        L.ref_power_hop_freq.argtypes = [C.c_int]
        L.ref_power_csv.argtypes = [C.c_char_p, C.c_char_p]
        L.ref_fix_fft.argtypes = [C.POINTER(C.c_int16), C.c_int, C.c_int]
        self.L = L
        self.plan: Optional[RefPlanC] = None

    def setup(self, freq_arg: str, crop: float = 0.0, boxcar: int = 1, comp_fir_size: int = 0,
              peak_hold: int = 0, window="rectangle", custom_window: Optional[Sequence[int]] = None):
        plan = RefPlanC()
        cw = None
        if custom_window is not None:
            cw_arr = np.ascontiguousarray(custom_window, dtype=np.int32)
            cw = cw_arr.ctypes.data_as(C.POINTER(C.c_int))
        wid = WINDOWS[window] if isinstance(window, str) else int(window)
        r = self.L.ref_power_setup(freq_arg.encode(), crop, boxcar, comp_fir_size, peak_hold, wid & 7, cw,
                                   C.byref(plan))
        if r != 0:
            raise RuntimeError("ref_power_setup failed")
        self.plan = plan
        return plan

    def tables(self):
        n = 1 << self.plan.bin_e
        win = np.empty(n, dtype=np.int32)
        sine = np.empty(max(n * 3 // 4, 1), dtype=np.int16)
        self.L.ref_power_tables(win.ctypes.data_as(C.POINTER(C.c_int)), _p16(sine))
        return win, sine

    def hop_freqs(self) -> np.ndarray:
        return np.array([self.L.ref_power_hop_freq(i) for i in range(self.plan.tune_count)], dtype=np.int64)

    def scan(self, hop_bufs: np.ndarray, n_pass: int):
        hb = _i16(hop_bufs).reshape(-1)
        assert hb.size == n_pass * self.plan.tune_count * self.plan.buf_len
        got = self.L.ref_power_scan(_p16(hb), n_pass)
        assert got == n_pass * self.plan.tune_count, got
        return self.get()

    def time(self, hop_bufs: np.ndarray, n_pass: int, repeats: int = 1) -> float:
        hb = _i16(hop_bufs).reshape(-1)
        return float(self.L.ref_power_time(_p16(hb), n_pass, repeats))

    def get(self):
        n = 1 << self.plan.bin_e
        avg = np.zeros((self.plan.tune_count, n), dtype=np.int64)
        samples = np.zeros(self.plan.tune_count, dtype=np.int32)
        self.L.ref_power_get(avg.ctypes.data_as(C.POINTER(C.c_int64)), samples.ctypes.data_as(C.POINTER(C.c_int)))
        return avg, samples

    def reset(self) -> None:
        self.L.ref_power_reset()

    def csv(self, path: str, tstr: str = "2026-01-01, 00:00:00") -> str:
        if self.L.ref_power_csv(path.encode(), tstr.encode()) != 0:
            raise OSError(path)
        with open(path) as f:
            return f.read()

    def fix_fft(self, iq: np.ndarray, m: int, log2_wave: Optional[int] = None) -> np.ndarray:
        buf = _i16(iq).copy()
        self.L.ref_fix_fft(_p16(buf), m, m if log2_wave is None else log2_wave)
        return buf


def ref_rx_sdr(src: np.ndarray, in_fmt: str, out_fmt: str, n_elems: int, block: int = 16384, workdir: str = "/tmp") -> bytes:
    """Run the reference's own rx_sdr executable (_ref/rx_sdr_ref = src/rtl_sdr.c's main() linked against the replay
    fake) over a capture and return the bytes it wrote: `rx_sdr -d driver=file,path=.. -I in_fmt -F out_fmt -n N -b B out`.
    The capture must hold MORE than n_elems elements (the recorder only stops on a read that over-delivers, :341-346)."""
    import tempfile
    with tempfile.TemporaryDirectory(dir=workdir) as td:
        cap, out = os.path.join(td, "cap.bin"), os.path.join(td, "out.bin")
        np.ascontiguousarray(src).tofile(cap)
        r = subprocess.run([REF_SDR_BIN, "-d", f"driver=file,path={cap}", "-I", in_fmt, "-F", out_fmt, "-n", str(n_elems),
                            "-b", str(block), out], capture_output=True, timeout=120)
        if r.returncode != 0:
            raise RuntimeError(r.stderr.decode()[-500:])
        with open(out, "rb") as f:
            return f.read()


_port: Optional[Port] = None


def port() -> Port:
    global _port
    if _port is None:
        _port = Port()
    return _port
