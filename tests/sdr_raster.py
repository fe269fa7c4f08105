"""Cases of the tests of rx_sdr raster I/Q handles (rxb200_sdr_mix_create_raster) and of the shells' raster capture plan
(rxb200_fm_plan_capture_raster): the planner's rule restated, the model (fm_raster's raster rule, then sdr_mix's
rx_sdr conversion of the int16) and the named shapes.
"""
import numpy as np

import fm_raster as frs
import sdr_mix as sm
from rx_tools_b200 import power, sdr

FORMATS = sm.FORMATS
convert = sm.convert
digest = sm.digest


def _gcd(a, b):
    while b:
        a, b = b, a % b
    return a


def plan_restated(tuned_hz, chain_rate, max_rate):
    """rxb200_fm_plan_capture_raster's rule: (fc, M, R, T, K, bins), or "rate" / "bins" where it refuses."""
    t = [int(v) for v in tuned_hz]
    tmin, tmax = min(t), max(t)
    g = 0
    for v in t:
        g = _gcd(v - tmin, g)
    fc = tmin + g * ((tmax - tmin) // (2 * g)) if g else tmin
    A, c = max(fc - tmin, tmax - fc), int(chain_rate)
    M = -(-(2 * A + c) // c)
    R = M * c
    if R > max_rate or R > (1 << 31) - 1 or M > 256:
        return "rate"
    K0 = R // _gcd(R, g) if g else 1
    K = K0 if K0 >= 3 else 3
    if K > 4096:
        return "bins"
    bins = []
    for v in t:
        o = v - fc
        assert (o * K) % R == 0
        bins.append((o * K // R) % K)
    return fc, M, R, min(8191, 32 * M + 1), K, bins


def model(name, x=None):
    """(CS16 outputs [n_channels][2 n] of the raster rule over the shape's whole capture, decimation M)."""
    K, bins, (M, taps, S) = SHAPES[name][:3]
    x = case_capture(name) if x is None else x
    return frs.raster_model(x, K, bins, taps, M, S)[0], int(M)


def _broadcast():
    """The FM broadcast band, one -f per station 88.1-107.9 MHz at 200 kHz, through rx_sdr -s 250k."""
    tuned = [88_100_000 + 200_000 * k for k in range(100)]
    fc, M, R, T, K, bins = plan_restated(tuned, 250_000, 25_000_000)
    assert (fc, M, R, T, K) == (97_900_000, 81, 20_250_000, 2593, 405)
    return K, bins, (M, power.ddc_lowpass(M, T, 15), 30)


def _k768(n_ch):
    """tools/fm_raster_time.py's raster: 19.2 Msps, 768 bins of 25 kHz, M = 64, the 2049-tap capture filter."""
    rng = np.random.default_rng(768 + n_ch)
    bins = sorted(int(b) for b in rng.choice(768, size=n_ch, replace=False))
    return 768, bins, (64, power.ddc_lowpass(64, 2049, 15), 30)


# name -> (K, bins, (M, taps, S), complex samples of capture)
SHAPES = {
    "broadcast_k405_c100": _broadcast() + (81 * 150 + 40,),
    "k768_c256": _k768(256) + (64 * 100 + 17,),
    # K = 3: every bin
    "k3": (3, [0, 1, 2], (3, np.array([5, -40, 900, 4000, 900, -40, 5], np.int32), 20), 3 * 700 + 2),
    # K = 4096 with sum |h| = 2^22 - 1 at S = 33: outputs that saturate
    "k4096_sat": (4096, [0, 1, 2048, 4095, 1234], (64, frs.near_limit(129, 0.5 / 64), 33), 64 * 90 + 5),
    # repeated bins, bin K/2 and bin 0
    "repeats_k64": (64, [0, 32, 5, 5, 0, 32, 63], (8, power.ddc_lowpass(8, 65, 15), 30), 8 * 500 + 3),
    # M = 1, T = 1, h = {1} at S = 15: bin 0 is the capture itself
    "unit_k5": (5, [0, 1, 4, 2], (1, np.array([1], np.int32), 15), 3001),
}


def case_capture(name, seed=0):
    """The shape's capture: full-scale int16[2 n]."""
    n = SHAPES[name][3]
    rng = np.random.default_rng(1900 + seed + len(name))
    return rng.integers(-32768, 32768, size=2 * n, dtype=np.int32).astype(np.int16)


def handle(name, device=0):
    K, bins, dd = SHAPES[name][:3]
    return sdr.SdrMix(ddc=dd, raster=(K, bins), device=device)
