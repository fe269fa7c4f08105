"""Capture plans at a device rate (include/rxb200.h, "capture plans at a device rate") restated in Python, the
closed form of rxb200_resample_in_len, and the header's worked examples.

Every _at planner is its planner with the decimation floor M = ceil((2A + c + G) / c), G = ceil(R_dev / 32), and one
more refusal, R > R_dev, right after the cap's.
"""
import math

import resample as rsm

FM, SDR, TWO_STAGE, RASTER = "fm", "sdr", "two_stage", "raster"
MIX_MAX_PERIOD = 1 << 20


def guard(R_dev):
    return rsm.ceil_div(R_dev, 32)


def plan_at(kind, tuned, c, cap, R_dev):
    """The _at planner of kind restated: a dict of the plan, or the refusal ("rate", "device", "m8", "bins", "period")."""
    t = [int(v) for v in tuned]
    tmin, tmax = min(t), max(t)
    g = 0
    for v in t:
        g = math.gcd(g, v - tmin)
    fc = tmin + g * ((tmax - tmin) // (2 * g)) if g else tmin
    offs = [v - fc for v in t]
    A = max(fc - tmin, tmax - fc)
    M = rsm.ceil_div(2 * A + c + guard(R_dev), c)
    if kind == TWO_STAGE:
        Mp = 4 * rsm.ceil_div(M, 4)
        R = Mp * c
        if Mp < 8 or R > cap or R > (1 << 31) - 1 or Mp > 256:
            return "m8" if Mp < 8 else "rate"
        if R > R_dev:
            return "device"
        M1 = Mp // 4
        return dict(fc=fc, R=R, K=2 * M1, M1=M1, T1=min(8191, 24 * M1 + 1), offsets=offs, span=2 * A + c)
    R = M * c
    if R > cap or R > (1 << 31) - 1 or M > 256:
        return "rate"
    if R > R_dev:
        return "device"
    T = min(8191, 32 * M + 1)
    if kind == RASTER:
        K = max(3, R // math.gcd(R, g) if g else 1)
        if K > 4096:
            return "bins"
        return dict(fc=fc, M=M, R=R, T=T, K=K, bins=[(o * K // R) % K for o in offs], span=2 * A + c)
    if kind == FM and any(R // math.gcd(R, abs(o)) > MIX_MAX_PERIOD for o in offs):
        return "period"
    return dict(fc=fc, M=M, R=R, T=T, offsets=offs, span=2 * A + c)


def in_len_rule(L, N, n0, n_out):
    """The fewest device samples c from n0 with out_count(n0, c) >= n_out, by its closed form."""
    if n_out == 0:
        return 0
    m0 = rsm.ceil_div(n0 * L, N)
    return (m0 + n_out - 1) * N // L + 1 - n0


# the header's worked examples: (kind, tuned Hz, chain rate, R_dev, M, R, L/N)
NOAA7 = [162_400_000 + 25_000 * k for k in range(7)]
SDR4 = [100_000_000, 100_025_000, 100_500_000, 100_950_000]
FM100 = [88_100_000 + 200_000 * k for k in range(100)]
WORKED = [
    (FM, NOAA7, 1_008_000, 2_400_000, 2, 2_016_000, (21, 25)),
    (SDR, SDR4, 250_000, 2_400_000, 6, 1_500_000, (5, 8)),
    (FM, FM100, 1_020_000, 30_720_000, 22, 22_440_000, (187, 256)),
]

