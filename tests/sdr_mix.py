"""Cases of the tests of rx_sdr I/Q down-converter handles (rxb200_sdr_mix_*): a numpy model of both front stages and of
rx_sdr's recorded formats, the capture planner's rule restated, and the named shapes.

The single stage is power_mix's per-hop model (the NCO mixer, then fm_ddc.ddc_model's filter) over the whole capture,
laid out channel-major; the two-stage model is fm_two_stage's.  The formats follow rx_sdr's conversions of the int16
(src/rtl_sdr.c:367-386): CS8 (uint8_t)(int)(x/32767.0*128.0+0.4), CU8 (uint8_t)(x/32767.0*128.0+127.4) and CF32
x * 1.0f / 32767, in fp64 and fp32 as there.
"""
import hashlib

import numpy as np

import fm_ddc as fdd
import fm_raster as frs
import fm_two_stage as fts
import power_mix as pmx
from rx_tools_b200 import power, sdr

FORMATS = ("CS16", "CS8", "CU8", "CF32")


def convert(y16, fmt):
    """int16[..., 2n] -> the format's components, as rx_sdr converts each int16."""
    y = np.asarray(y16, dtype=np.int16)
    if fmt == "CS16":
        return y.copy()
    if fmt == "CF32":
        return (y.astype(np.float32) * np.float32(1.0)) / np.float32(32767)
    v = y.astype(np.float64) / 32767.0 * 128.0 + (0.4 if fmt == "CS8" else 127.4)
    return np.trunc(v).astype(np.int64).astype(np.uint8)


def single_model(cs16, rate, offsets, dd):
    """The single-stage rule over a whole capture: int16[n_channels][2 floor(c / M)]."""
    x = np.asarray(cs16, dtype=np.int16).reshape(-1)
    n = x.size // 2 // int(dd[0])
    out = np.empty((len(offsets), 2 * n), np.int16)
    for c, f in enumerate(offsets):
        out[c] = pmx.ddc(x, rate, f, dd)[0][:2 * n]
    return out


def two_stage_model(cs16, rate, n_bins, offsets, coarse, fine):
    return fts.two_stage_model(cs16, rate, n_bins, offsets, coarse, fine)


def model(name, x=None):
    """(CS16 outputs [n_channels][2 n], decimation M) of a shape over its capture."""
    kind, rate, offs, stages = SHAPES[name][:4]
    x = case_capture(name) if x is None else x
    if kind == "single":
        return single_model(x, rate, offs, stages), int(stages[0])
    K, coarse, fine = stages
    return two_stage_model(x, rate, K, offs, coarse, fine), int(coarse[0]) * int(fine[0])


def plan_restated(tuned_hz, sample_rate, max_rate):
    """rxb200_sdr_plan_capture's rule: (fc, M, R, T, offsets) or None where it refuses (no table refusal)."""
    t = [int(v) for v in tuned_hz]
    tmin, tmax = min(t), max(t)
    g = 0
    for v in t:
        a, b = v - tmin, g
        while b:
            a, b = b, a % b
        g = a
    fc = tmin + g * ((tmax - tmin) // (2 * g)) if g else tmin
    A, c = max(fc - tmin, tmax - fc), int(sample_rate)
    M = -(-(2 * A + c) // c)
    R = M * c
    if R > max_rate or R > (1 << 31) - 1 or M > 256:
        return None
    return fc, M, R, min(8191, 32 * M + 1), [v - fc for v in t]


def _offsets(rate, n, seed):
    rng = np.random.default_rng(seed)
    lim = rate // 2 - 1
    return [int(v) for v in rng.choice(np.arange(-lim, lim), size=n, replace=False)]


def _plan20(n):
    """The shell's single-stage plan at 20 Msps for a 250 kHz channel rate: M = 80, T = 2561."""
    M = 80
    return (M, power.ddc_lowpass(M, min(8191, 32 * M + 1), 15), 15)


_C20 = fts.plan_stages(80)                  # two stages at 20 Msps: K = 40, M1 = 20, M2 = 4

# name -> (kind, capture rate, offsets, stages, complex samples of capture): stages is (M, h, S) for "single" and
# (K, coarse, fine) for "two"
SHAPES = {
    # 256 channels at arbitrary offsets of a 20 Msps plan, both kinds
    "single_20m_c256": ("single", 20_000_000, _offsets(20_000_000, 256, 11), _plan20(256), 80 * 300),
    "two_20m_c256": ("two", 20_000_000, _offsets(20_000_000, 256, 12), _C20, 80 * 300),
    # M = 1, T = 1, h = {1}, S = 0 at offset 0: the capture itself
    "identity": ("single", 1_000_000, [0], (1, np.array([1], np.int32), 0), 5000),
    # taps whose sum |h| 2^15 needs a 64-bit accumulator
    "wide_acc": ("single", 2_000_000, [123_457, -654_321], (4, np.array([1 << 20, -(1 << 19), 1 << 20, 7], np.int32), 21),
                 4000),
    # channels at +-(R/2 - 1)
    "band_edges": ("single", 4_000_000, [1_999_999, -1_999_999, 0], (8, fdd.lowpass(65, 0.06), 15), 8000),
    # K = 3 and K = 4096
    "two_k3": ("two", 1_008_000, [0, 335_999, -170_001, 1], (3, (3, frs.near_limit(17, 120e3 / 1.008e6), 33),
                                                            (2, fdd.lowpass(9, 0.2), 15)), 6000),
    "two_k4096": ("two", 2_048_000, [0, 250, -1_023_999, 1_023_999, 777_777],
                  (4096, (64, frs.near_limit(129, 0.5 / 64), 33), (2, fdd.lowpass(17, 0.2), 15)), 128 * 60),
}


def case_capture(name, seed=0):
    """The shape's capture: int16[2 n]; the identity shape's covers every int16 value."""
    kind, rate, offs, stages, n = SHAPES[name]
    rng = np.random.default_rng(900 + seed + len(name))
    return rng.integers(-32768, 32768, size=2 * n, dtype=np.int32).astype(np.int16)


def handle(name, device=0):
    kind, rate, offs, stages = SHAPES[name][:4]
    if kind == "single":
        return sdr.SdrMix(rate, offs, ddc=stages, device=device)
    return sdr.SdrMix(rate, offs, two_stage=stages, device=device)


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).view(np.uint8)).hexdigest()
