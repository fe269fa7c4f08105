"""Cases of the tests of rx_power hops of one capture (rxb200_power_mix_*): a numpy model of the NCO down-converter (the
exact-integer frequency word, the library's own NCO table, then fm_ddc.ddc_model's filter arithmetic over the NCO-mixed
stream), the capture plan the rx_power shell derives from a sweep plan in capture mode, and the named shapes.

Hop i of a power mixing handle is what the reference's scanner() accumulates from hop buffers made of the decimated
stream of mix_i(capture): pass p of hop i is outputs [p B, (p+1) B), B = buf_len / 2.  The oracles run on the model's hop
buffers ([P][n_hops][buf_len], pass-major), and the library runs on the capture itself.
"""
import hashlib

import numpy as np

import fm_ddc as fdd
import power_paths
from rx_tools_b200 import power

IDENTITY = np.array([[32768, 0]], dtype=np.int32)     # a one-entry mixer table that leaves every sample as it is
_NCO = None


def nco_table():
    global _NCO
    if _NCO is None:
        _NCO = power.nco_table()
    return _NCO


def nco_word(rate, f):
    """w = floor((f 2^32 + floor(R/2)) / R) mod 2^32, with Python's floor division."""
    return ((int(f) << 32) + int(rate) // 2) // int(rate) % (1 << 32)


def nco_mix(cs16, rate, f, n0=0):
    """The NCO mixer: int16[2c] CS16 -> int16[2c]; sample k is capture sample n0 + k, phase (n0 + k) w mod 2^32."""
    x = np.asarray(cs16, dtype=np.int16).reshape(-1, 2).astype(np.int64)
    w = np.uint64(nco_word(rate, f))
    n = (np.uint64(int(n0) % (1 << 32)) + np.arange(x.shape[0], dtype=np.uint64)) & np.uint64(0xffffffff)
    theta = (n * w) & np.uint64(0xffffffff)                              # < 2^64 before the mask: no wrap loss
    j = (((theta + np.uint64(32768)) & np.uint64(0xffffffff)) >> np.uint64(16)).astype(np.int64)
    t = nco_table()
    c, s = t[j, 0].astype(np.int64), t[j, 1].astype(np.int64)
    out = np.empty_like(x)
    out[:, 0] = (x[:, 0] * c - x[:, 1] * s + (1 << 14)) >> 15
    out[:, 1] = (x[:, 0] * s + x[:, 1] * c + (1 << 14)) >> 15
    return out.astype(np.int16).reshape(-1)                            # int64 -> int16 wraps, like the kernel's stores


def ddc(cs16, rate, f, dd, n0=0, hist=None):
    """The DDC of one hop over c samples whose first is capture sample n0, emission points counted from that sample:
    (int16[2 floor(c/M)], the new history of mixed samples); hist: the mixed history before the call (None: zeros)."""
    decim, taps, shift = dd
    z = nco_mix(cs16, rate, f, n0)
    return fdd.ddc_model(z, IDENTITY, taps, decim, shift, 0, hist)


class Model:
    """The handle's state in numpy: the sample count and each hop's (mixed) filter history."""

    def __init__(self, rate, offsets, dd, buf_len):
        self.rate, self.offsets, self.dd, self.buf_len = int(rate), list(offsets), dd, int(buf_len)
        self.pos, self.hist = 0, [None] * len(self.offsets)

    def hop_buffers(self, cs16):
        """int16[P][n_hops][buf_len] of a call of whole passes (so every call starts on an emission boundary)."""
        x = np.asarray(cs16, dtype=np.int16).reshape(-1)
        assert x.size % (self.dd[0] * self.buf_len) == 0
        P = x.size // (self.dd[0] * self.buf_len)
        out = np.empty((P, len(self.offsets), self.buf_len), dtype=np.int16)
        for i, f in enumerate(self.offsets):
            y, self.hist[i] = ddc(x, self.rate, f, self.dd, self.pos, self.hist[i])
            out[:, i, :] = y.reshape(P, self.buf_len)
        self.pos += x.size // 2
        return out


def capture_plan(plan):
    """What the shell derives in capture mode: (centre F_c, offsets f_i, M, R, (M, taps, 15))."""
    n = plan.n_hops
    fc = plan.first_freq + ((n - 1) * plan.freq_step) // 2
    offs = [plan.hop_freq(i) - fc for i in range(n)]
    span = 2 * max(abs(f) for f in offs)
    M = max(1, -(-(span + plan.rate) // plan.rate))
    T = min(8191, 32 * M + 1)
    return fc, offs, M, M * plan.rate, (M, power.ddc_lowpass(M, T, 15), 15)


def capture(n_complex, rate, offsets, seed, amplitude=3000.0, noise=800):
    """A tone near each hop's offset (its own frequency within the hop and its own phase) over broadband noise."""
    rng = np.random.default_rng(seed)
    t = np.arange(n_complex, dtype=np.float64)
    z = np.zeros(n_complex, dtype=np.complex128)
    for k, f in enumerate(offsets[::max(1, len(offsets) // 8)]):
        fk = (f + rng.uniform(-0.3, 0.3) * rate / max(8, len(offsets))) / rate
        z += amplitude / (1 + k % 3) * np.exp(2j * np.pi * (fk * t + rng.uniform()))
    x = np.empty(2 * n_complex, dtype=np.int64)
    x[0::2] = np.rint(z.real)
    x[1::2] = np.rint(z.imag)
    x += rng.integers(-noise, noise + 1, size=x.size)
    return np.clip(x, -32768, 32767).astype(np.int16)


# name -> the command line (as rx_power takes it) and the run: passes, window, and an optional filter in place of the
# shell's (M from the capture plan, taps from rxb200_ddc_lowpass(M, T, S) with the given T and S)
SHAPES = {
    # the timing tool's plans: 88-108 MHz at 10 kHz (8 hops, R = 20 Msps) and 24-60 MHz cropped 28.5 % (18 hops)
    "fm_band": dict(freq="88M:108M:10k", crop=0.0, boxcar=1, fir=0, peak=0, window="hamming", n_pass=3),
    "hf_crop285": dict(freq="24M:60M:10k", crop=0.285, boxcar=1, fir=0, peak=0, window="blackman", n_pass=2),
    # a cropped plan whose periods the table mixer refuses (L up to 1 333 333 > 2^20)
    "uhf_crop25": dict(freq="430M:450M:10k", crop=0.25, boxcar=1, fir=0, peak=0, window="hann-poisson", n_pass=2),
    # one hop of a span below 1 MHz: the boxcar downsample 5, M = 1 and a 33-tap filter
    "small_boxcar": dict(freq="100M:100.5M:1k", crop=0.0, boxcar=1, fir=0, peak=0, window="blackman-harris", n_pass=3),
    # -F 9: fifth_order passes and the droop FIR
    "small_F9": dict(freq="100M:100.3M:1k", crop=0.0, boxcar=0, fir=9, peak=0, window="kaiser", n_pass=2),
    # -P peak hold
    "peak_hold": dict(freq="88M:98M:20k", crop=0.1, boxcar=1, fir=0, peak=1, window="rectangle", n_pass=3),
    # bin size >= 1 MHz: rms_power, bin_e = 0
    "rms": dict(freq="100M:110M:1M", crop=0.0, boxcar=1, fir=0, peak=0, window="rectangle", n_pass=2),
    # 260 hops at crop 0.99: two grid rows of the kernel; a short filter keeps the model's work small
    "hops260": dict(freq="100M:107.28M:10k", crop=0.99, boxcar=1, fir=0, peak=0, window="bartlett", n_pass=1,
                    taps=(17, 15)),
    # taps summing to 2^17 at S = 17: the 64-bit accumulator
    "wide_acc": dict(freq="88M:92M:10k", crop=0.0, boxcar=1, fir=0, peak=0, window="hamming", n_pass=2,
                     taps=(65, 17)),
}


def shape(name):
    """(plan, window, R, offsets, (M, taps, S)) of a named shape."""
    c = SHAPES[name]
    plan = power.plan_range(c["freq"], c["crop"], c["boxcar"], c["fir"], c["peak"])
    _, offs, M, R, dd = capture_plan(plan)
    if "taps" in c:
        T, S = c["taps"]
        dd = (M, power.ddc_lowpass(M, T, S), S)
    return plan, power.window_table(c["window"], 1 << plan.bin_e), R, offs, dd


def case_input(name, seed=0):
    """(plan, window, R, offsets, ddc, capture) of a named shape: exactly n_pass passes."""
    plan, win, R, offs, dd = shape(name)
    n_complex = SHAPES[name]["n_pass"] * dd[0] * plan.buf_len // 2
    return plan, win, R, offs, dd, capture(n_complex, R, offs, 1300 + seed + len(name))


def model_buffers(name, seed=0):
    plan, win, R, offs, dd, x = case_input(name, seed)
    return Model(R, offs, dd, plan.buf_len).hop_buffers(x)


def port_result(port, plan, win, hb):
    return port.power_scan(power_paths.oracle_params(plan), win, hb, hb.shape[0], plan.n_hops)


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()

