"""The rational resampler's rule (include/rxb200.h, "capture from a device at its own rate") as a numpy int64 model and
as a term-by-term Python-integer restatement, the planner restated, and the named plans.

Output m of a resampler (L up, N down, J taps per phase, prototype h of J L taps, shift S) over device samples x[n]
(x[n] = 0 for n < 0) is t = m N, q = floor(t / L), p = t mod L, A = sum_{j<J} h[p + j L] x[q - j], then the rounding
shift and int16 saturation.  A call over [n0, n0 + c) returns outputs ceil(n0 L / N) .. ceil((n0 + c) L / N) - 1.
"""
import math

import numpy as np


def ceil_div(a, b):
    return -(-a // b)


def out_count(n0, c, L, N):
    return ceil_div((n0 + c) * L, N) - ceil_div(n0 * L, N)


def _round_sat(A, S):
    y = A if S == 0 else (A + (1 << (S - 1))) >> S
    return np.clip(y, -32768, 32767)


def resample_model(cs16, L, N, taps, S, n0=0, hist=None):
    """One call over device samples [n0, n0 + c): int16 [2c] -> (int16 [2 n_out], the new history).

    hist: the J - 1 raw samples before the call as int16 [2(J - 1)] (None: zeros, the state after create or reset)."""
    x = np.asarray(cs16, dtype=np.int16).reshape(-1, 2).astype(np.int64)
    h = np.asarray(taps, dtype=np.int64).reshape(-1)
    J = h.size // L
    assert J * L == h.size
    H = J - 1
    hs = np.zeros((H, 2), np.int64) if hist is None else np.asarray(hist, np.int16).reshape(-1, 2).astype(np.int64)
    ext = np.concatenate([hs, x])
    c = x.shape[0]
    m0, n = ceil_div(n0 * L, N), out_count(n0, c, L, N)
    t0 = m0 * N
    q0, p0 = t0 // L - n0, t0 % L                               # Python integers: n0 may be near 2^64
    out = np.empty((n, 2), np.int64)
    jj = np.arange(J, dtype=np.int64)
    blk = max(1, (1 << 21) // J)
    for a in range(0, n, blk):
        i = np.arange(a, min(n, a + blk), dtype=np.int64)
        v = p0 + i * N
        q, p = q0 + v // L, v % L
        idx = q[:, None] + H - jj[None, :]                      # ext index of x[q - j]
        hp = h[p[:, None] + jj[None, :] * L]
        out[a:a + i.size, 0] = (hp * ext[idx, 0]).sum(1)
        out[a:a + i.size, 1] = (hp * ext[idx, 1]).sum(1)
    y = _round_sat(out, S).astype(np.int16).reshape(-1)
    new_hist = ext[ext.shape[0] - H:].astype(np.int16).reshape(-1) if H else np.zeros(0, np.int16)
    return y, new_hist


def resample_rule(cs16, L, N, taps, S, n0=0):
    """The rule term by term in Python integers, for a stream that is zero before n0 (small cases only)."""
    x = [tuple(int(v) for v in s) for s in np.asarray(cs16, dtype=np.int16).reshape(-1, 2)]
    h = [int(v) for v in np.asarray(taps).reshape(-1)]
    J = len(h) // L
    out = []
    for m in range(ceil_div(n0 * L, N), ceil_div((n0 + len(x)) * L, N)):
        t = m * N
        q, p = t // L, t % L
        assert n0 <= q < n0 + len(x)
        A = [0, 0]
        for j in range(J):
            k = q - j - n0
            if k >= 0:
                A[0] += h[p + j * L] * x[k][0]
                A[1] += h[p + j * L] * x[k][1]
        for a in A:
            y = a if S == 0 else (a + (1 << (S - 1))) >> S
            out.append(max(-32768, min(32767, y)))
    return np.array(out, dtype=np.int16)


def calls_model(cs16, L, N, taps, S, lens16):
    """The model over a sequence of calls cut at lens16 (cycled), concatenated."""
    x = np.asarray(cs16, dtype=np.int16).reshape(-1)
    parts, at, i, pos, hist = [], 0, 0, 0, None
    while at < x.size:
        n = min(lens16[i % len(lens16)], x.size - at)
        y, hist = resample_model(x[at:at + n], L, N, taps, S, pos, hist)
        parts.append(y)
        pos += n // 2
        at += n
        i += 1
    return np.concatenate(parts) if parts else np.zeros(0, np.int16)


def wide(taps, L, S):
    """Whether the library accumulates in 64 bits: max_p sum |h_p| * 32768 + 2^(S-1) >= 2^31."""
    h = np.abs(np.asarray(taps, dtype=np.int64))
    worst = max(int(h[p::L].sum()) for p in range(L))
    return worst * 32768 + ((1 << (S - 1)) if S else 0) >= (1 << 31)


def plan_rule(R_dev, R, span):
    """rxb200_plan_resample restated: (L, N, J, S), or None where it refuses a span that does not fit."""
    G = ceil_div(R_dev, 32)
    D = min(R, R_dev) - span
    if D < G:
        return None
    g = math.gcd(R, R_dev)
    L, N = R // g, R_dev // g
    J = 8 * ceil_div(ceil_div(6 * R_dev, D), 8)
    return L, N, J, 15


def response_db(taps, L, R_dev, span, R):
    """(worst passband deviation in dB over |f| <= span/2, worst stopband level in dB over |f| >= min(R, R_dev) -
    span/2) of the prototype at rate L R_dev, normalised to its DC gain."""
    h = np.asarray(taps, dtype=np.float64)
    nfft = 1 << max(20, int(np.ceil(np.log2(h.size * 16))))
    H = np.abs(np.fft.rfft(h, nfft))
    f = np.arange(H.size) * (L * R_dev) / nfft
    db = 20 * np.log10(np.maximum(H / H[0], 1e-30))
    pb, sb = f <= span / 2, f >= min(R, R_dev) - span / 2
    return float(np.abs(db[pb]).max()), float(db[sb].max())


# The named plans: (name, R_dev, R, span = 2A + c, L/N, J)
NAMED = [
    ("noaa7_nbfm_2.4M", 2_400_000, 2_016_000, 1_158_000, (21, 25), 24),
    ("noaa7_nbfm_2.5M", 2_500_000, 2_016_000, 1_158_000, (504, 625), 24),
    ("fm100_wbfm_30.72M", 30_720_000, 22_440_000, 21_020_000, (187, 256), 136),
    ("sdr4_250k_2.4M", 2_400_000, 1_500_000, 1_200_000, (5, 8), 48),
    ("fm100_sdr_raster_30.72M", 30_720_000, 21_250_000, 20_250_000, (2125, 3072), 192),
    ("fm100_wbfm_61.44M", 61_440_000, 23_460_000, 21_020_000, (391, 1024), 152),
]
# the same 100 stations on a 20 Msps device: refused, the span 21.02 MHz being above 20 M - 625 k
REFUSED = (20_000_000, 22_440_000, 21_020_000)
