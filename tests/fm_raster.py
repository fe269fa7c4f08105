"""Cases of the tests of raster mixing handles (rxb200_fm_mix_create_raster): a numpy model of the raster rule in int64
(every value stays below 2^53, so it is exact), the polyphase regrouping the kernels use, the named shapes with their
captures and read sequences, and the per-read decimated streams the reference and the port demodulate.

Channel c of a raster handle is bin k_c of a K-bin raster over the capture:
    A = sum_{j<T} h[j] x[e_m - j] tw[(k (e_m - j)) mod K],   y = S ? (A + 2^(S-1)) >> S : A,   out = sat16(y)
with tw the period-K table rxb200_fm_mix_table(K, 1) and e_m = m M + M - 1 counted from create or reset.
"""
import numpy as np

import fm_any_chunk as fac
import fm_ddc as fdd
import fm_mix as fmx
import fm_read as frd
from fm_any_chunk import with_
from rx_tools_b200 import fm, power


def table(n_bins):
    """tw: int32[K][2], the period-K table rxb200_fm_mix_table(K, 1)."""
    return fm.mix_table(n_bins, 1)


def sum_abs(taps):
    return int(np.abs(np.asarray(taps, dtype=np.int64)).sum())


def _finish(acc, shift):
    y = acc if shift == 0 else (acc + (1 << (shift - 1))) >> shift
    return np.clip(y, -32768, 32767).astype(np.int16)


def raster_model(cs16, n_bins, bins, taps, decim, shift, pos=0, hist=None, phase=None):
    """The raster rule over one call: int16[2c] capture -> (int16[n_channels][2 n_out], the new history).

    pos: capture samples before this call (emission points are global samples m M + M - 1); hist: the capture's last
    T - 1 complex samples before the call as int16[2(T - 1)] (None: zeros); phase: the residue mod K of the call's
    first sample's index (default pos mod K; the stateless entry's n0 mod K)."""
    x = np.asarray(cs16, dtype=np.int16).reshape(-1)
    taps = np.asarray(taps, dtype=np.int64)
    T, M, H, K = taps.size, int(decim), taps.size - 1, int(n_bins)
    assert sum_abs(taps) < (1 << 22)
    h = np.zeros(2 * H, np.int16) if hist is None else np.asarray(hist, dtype=np.int16).reshape(-1)
    assert h.size == 2 * H
    p0 = pos % K if phase is None else phase % K
    ext = np.concatenate([h, x]).reshape(-1, 2).astype(np.int64)
    res = (p0 - H + np.arange(ext.shape[0], dtype=np.int64)) % K            # each staged sample's index mod K
    tw = table(K).astype(np.int64)
    c = x.size // 2
    m0, m1 = pos // M, (pos + c) // M
    e = np.arange(m0, m1, dtype=np.int64) * M + M - 1 - pos                  # local emission points, in [0, c)
    hr = taps[::-1]
    out = np.empty((len(bins), e.size, 2), np.int64)
    for ci, k in enumerate(bins):
        t = tw[(int(k) * res) % K]
        z = np.empty_like(ext)
        z[:, 0] = ext[:, 0] * t[:, 0] - ext[:, 1] * t[:, 1]                 # |z| <= 2^31: exact, no rounding
        z[:, 1] = ext[:, 0] * t[:, 1] + ext[:, 1] * t[:, 0]
        win = np.lib.stride_tricks.sliding_window_view(z, T, axis=0)        # win[i] = z[i .. i + T), shape (., 2, T)
        blk = max(1, (1 << 21) // max(T, 1))
        for a in range(0, e.size, blk):
            out[ci, a:a + blk] = np.einsum("ukt,t->uk", win[e[a:a + blk]], hr)
    y = _finish(out, shift).reshape(len(bins), -1)
    full = np.concatenate([h, x])
    return y, (full[full.size - 2 * H:].copy() if H else np.zeros(0, np.int16))


def branch_sums(ext, taps, decim, n_bins, res0, n_out):
    """The polyphase branch sums: v[m][rho] (complex int64 [n_out][K][2]) over ext (int16[2 n], the staged samples,
    ext[i] of index residue (res0 + i) mod K), output m's window ending at ext sample m M + M - 1 + T - 1."""
    x = np.asarray(ext, dtype=np.int16).reshape(-1, 2).astype(np.int64)
    taps = np.asarray(taps, dtype=np.int64)
    T, M, K = taps.size, int(decim), int(n_bins)
    v = np.zeros((n_out, K, 2), np.int64)
    for m in range(n_out):
        end = m * M + M - 1 + T - 1
        for j in range(T):
            i = end - j
            v[m, (res0 + i) % K] += taps[j] * x[i]
    return v


def dft(v, n_bins, bins):
    """A_k[m] = sum_rho tw[(k rho) mod K] v_rho[m]: int64 [n_channels][n_out][2]."""
    tw = table(n_bins).astype(np.int64)
    rho = np.arange(n_bins)
    out = []
    for k in bins:
        t = tw[(int(k) * rho) % n_bins]
        re = v[:, :, 0] @ t[:, 0] - v[:, :, 1] @ t[:, 1]
        im = v[:, :, 0] @ t[:, 1] + v[:, :, 1] @ t[:, 0]
        out.append(np.stack([re, im], axis=-1))
    return np.stack(out)


def decimated_reads(x, n_bins, bins, ddc, lens16):
    """The model over a read sequence: per channel, the decimated stream of each read (possibly empty), in order."""
    decim, taps, shift = ddc
    out, pos, hist = [[] for _ in bins], 0, None
    for a, n in fac.seq_bounds(x.size, lens16):
        y, hist = raster_model(x[a:a + n], n_bins, bins, taps, decim, shift, pos, hist)
        for c in range(len(bins)):
            out[c].append(y[c])
        pos += n // 2
    return out


def near_limit(n_taps, cutoff, total=(1 << 22) - 1):
    """A low-pass whose sum |h| is exactly `total` (the centre tap takes the difference)."""
    h = fdd.lowpass(n_taps, cutoff, gain_bits=21).astype(np.int64)
    h[n_taps // 2] += total - sum_abs(h)
    assert sum_abs(h) == total and h[n_taps // 2] > 0
    return h.astype(np.int32)


def bin_offsets(rate, n_bins, bins):
    """The centre frequency of each bin in Hz (negative past K/2), for synthesising captures."""
    return [int(round(k * rate / n_bins)) if 2 * k <= n_bins else int(round((k - n_bins) * rate / n_bins)) for k in bins]


READS, READS_LONG = fdd.READS, fdd.READS_LONG
NBFM12 = fdd.NBFM12

# name -> (parameters, capture rate (for the capture only), K, bins, (M, taps, S), capture keyword arguments, reads).
# A raster sum carries the twiddles' 2^15 on top of the taps' gain, so Q15 unity-gain taps take S = 30.
SHAPES = {
    # DESIGN 4.4's timing plan as a raster: 19.2 Msps, 768 bins of 25 kHz, M = 64, 257 taps, a D = 12 lut NBFM chain
    "nbfm_k768_m64_t257": (NBFM12, 19_200_000, 768, [408, 767, 0, 1, 360],
                           (64, fdd.lowpass(257, 12500 / 19.2e6), 30), {}, READS_LONG),
    # the same through the rx_power shell's channel filter, 2049 taps
    "nbfm_k768_m64_t2049": (NBFM12, 19_200_000, 768, [408, 767, 0, 1, 360],
                            (64, power.ddc_lowpass(64, 2049, 15), 30), {}, READS_LONG),
    # fm2b's -F 9 chain at M = 8: 19.2 Msps, 64 bins of 300 kHz (-4.8 MHz, 0, 3 MHz)
    "fm2b_f9_k64_m8": (with_(frd.FM2B, offset_tuning=1), 19_200_000, 64, [48, 0, 10],
                       (8, fdd.lowpass(33, 120e3 / 19.2e6), 30), dict(deviation=75000.0), READS_LONG),
    # am and raw at M = 100: 2.4 Msps -> 24 kHz; K = 240 and K = 100, not powers of two
    "am_k240_m100": (with_(fac.AM, downsample=1, offset_tuning=1), 2_400_000, 240, [237, 1],
                     (100, fdd.lowpass(301, 6000 / 2.4e6), 30), {}, READS),
    "raw_k100_m100": (with_(fac.RAW, downsample=1, offset_tuning=1), 2_400_000, 100, [0, 1, 98],
                      (100, fdd.lowpass(201, 9000 / 2.4e6), 30), {}, READS),
    # squelch with -L: 4.032 Msps, 504 bins of 8 kHz (+-200 kHz), M = 4, D = 42 lut, channels that fall quiet half way
    "fm_lut_squelch_k504_m4": (with_(fac.FM24K_LUT, squelch_level=60, offset_tuning=1), 4_032_000, 504, [479, 25],
                               (4, fdd.lowpass(33, 80e3 / 4.032e6), 30), dict(quiet_half=True), READS_LONG),
    # K = 3 with sum |h| = 2^22 - 1 at S = 33: gain 16, outputs that saturate
    "raw_sat_k3_m3": (with_(fac.RAW, downsample=2, offset_tuning=1), 1_008_000, 3, [0, 1, 2],
                      (3, near_limit(17, 120e3 / 1.008e6), 33), dict(amplitude=4000.0), READS),
    # K = 4096: bins 0, 1, K/2, K - 1 and bin 1 again
    "raw_k4096_m64": (with_(fac.RAW, downsample=1, offset_tuning=1), 2_048_000, 4096, [0, 1, 2048, 4095, 1],
                      (64, fdd.lowpass(129, 0.5 / 64), 30), {}, READS),
}


def case_input(name, seed=0):
    """(params, K, bins, (M, taps, S), capture, reads) of a shape."""
    p, rate, K, bins, ddc, kw, reads = SHAPES[name]
    x = fmx.capture(fdd.n_complex_for(reads), rate, bin_offsets(rate, K, bins), 1300 + seed + len(name), **kw)
    return p, K, bins, ddc, x, reads
