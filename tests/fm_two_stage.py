"""Cases of the tests of two-stage mixing handles (rxb200_fm_mix_create_two_stage): a numpy model of the two-stage rule
in int64 built from fm_raster's model (the coarse stage) and an NCO mixer by word plus fm_ddc's filter arithmetic (the
fine stage), the bins and words in Python integers, the shell's two-stage capture plan, and the named shapes with their
captures and read sequences.

Channel c of a two-stage handle, at offset f_c of a capture at rate R, K coarse bins, coarse (M1, h1, S1), fine
(M2, h2, S2):
    b_c = floor((f_c K + floor(R/2)) / R) mod K,  N_c = (f_c K - b'_c R) M1,  w_c = floor((N_c 2^32 + floor(KR/2)) / KR)
    y_b = the raster rule for bin b with (M1, h1, S1);  z_c[m] = NCO-mix(y_{b_c}[m], phase m w_c);
    out_c[q] = sat16(shift_S2(sum_j h2[j] z_c[q M2 + M2 - 1 - j])).
"""
import numpy as np

import fm_any_chunk as fac
import fm_ddc as fdd
import fm_mix as fmx
import fm_raster as frs
import fm_read as frd
import power_mix as pmx
from fm_any_chunk import with_
from rx_tools_b200 import power


def bin_word(rate, n_bins, coarse_decim, f):
    """(b_c, w_c) of the rule, in Python integers (floor division)."""
    R, K, f = int(rate), int(n_bins), int(f)
    b = ((f * K + R // 2) // R) % K
    bp = b - K if 2 * b > K else b
    N = (f * K - bp * R) * int(coarse_decim)
    D = K * R
    return b, ((N << 32) + D // 2) // D % (1 << 32)


def nco_mix_word(cs16, word, n0=0):
    """The rx_power NCO mixer by word: sample k is mixed at phase (n0 + k) w mod 2^32 (as power_mix.nco_mix)."""
    x = np.asarray(cs16, dtype=np.int16).reshape(-1, 2).astype(np.int64)
    w = np.uint64(int(word))
    n = (np.uint64(int(n0) % (1 << 32)) + np.arange(x.shape[0], dtype=np.uint64)) & np.uint64(0xffffffff)
    theta = (n * w) & np.uint64(0xffffffff)
    j = (((theta + np.uint64(32768)) & np.uint64(0xffffffff)) >> np.uint64(16)).astype(np.int64)
    t = pmx.nco_table()
    c, s = t[j, 0].astype(np.int64), t[j, 1].astype(np.int64)
    out = np.empty_like(x)
    out[:, 0] = (x[:, 0] * c - x[:, 1] * s + (1 << 14)) >> 15
    out[:, 1] = (x[:, 0] * s + x[:, 1] * c + (1 << 14)) >> 15
    return out.astype(np.int16).reshape(-1)                            # int64 -> int16 wraps, like mix_one


def coarse_streams(cs16, n_bins, bins, coarse, n1, n0=0):
    """{bin: int16[2 n1]}: the first n1 coarse outputs of each distinct bin over cs16 (sample i is index n0 + i)."""
    M1, h1, S1 = coarse
    x = np.asarray(cs16, dtype=np.int16).reshape(-1)[:2 * n1 * int(M1)]
    return {b: frs.raster_model(x, n_bins, [b], h1, M1, S1, phase=n0 % n_bins)[0][0] for b in sorted(set(bins))}


def fine_stream(y, word, fine, m0=0):
    """The fine stage over one bin's coarse stream y (coarse output m mixed at phase (m0 + m) w)."""
    M2, h2, S2 = fine
    return fdd.ddc_model(nco_mix_word(y, word, m0), pmx.IDENTITY, h2, M2, S2)[0]


def two_stage_model(cs16, rate, n_bins, offsets, coarse, fine, n0=0):
    """The rule over a whole stream: int16[2c] -> int16[n_channels][2 floor(c / M)].  Sample i is capture index n0 + i
    (twiddles), zeros before it, coarse output m at i = m M1 + M1 - 1 mixed at phase (floor(n0 / M1) + m) w_c, fine
    output q at coarse output q M2 + M2 - 1 (the stateless entry's convention; n0 = 0 is a handle's whole stream)."""
    M1, M2 = int(coarse[0]), int(fine[0])
    c = np.asarray(cs16).size // 2
    n_out = c // (M1 * M2)
    out = np.empty((len(offsets), 2 * n_out), np.int16)
    if n_out == 0:
        return out
    bw = [bin_word(rate, n_bins, M1, f) for f in offsets]
    ys = coarse_streams(cs16, n_bins, [b for b, _ in bw], coarse, n_out * M2, n0)
    for ci, (b, w) in enumerate(bw):
        out[ci] = fine_stream(ys[b], w, fine, int(n0) // M1)
    return out


def decimated_reads(x, rate, n_bins, offsets, coarse, fine, lens16):
    """The model over a read sequence: per channel, the decimated stream of each read (possibly empty), in order."""
    M = int(coarse[0]) * int(fine[0])
    y = two_stage_model(x, rate, n_bins, offsets, coarse, fine)
    out, at = [[] for _ in offsets], 0
    for a, n in fac.seq_bounds(x.size, lens16):
        d = fdd.decimated_len(a // 2, n, M)
        for c in range(len(offsets)):
            out[c].append(y[c, at:at + d])
        at += d
    return out


def plan_stages(m_prime):
    """The shell's two-stage plan for M' (rxb200_fm_plan_capture_two_stage): (K, coarse, fine)."""
    M1 = m_prime // 4
    return (2 * M1, (M1, power.ddc_lowpass(M1, min(8191, 24 * M1 + 1), 15), 30),
            (4, power.ddc_lowpass(4, 129, 15), 15))


def plan_restated(tuned_hz, chain_rate, max_rate):
    """The planner's rule restated: (fc, R, K, M1, T1, offsets) or None where it refuses."""
    t = [int(v) for v in tuned_hz]
    tmin, tmax = min(t), max(t)
    g = 0
    for v in t:
        a, b = v - tmin, g
        while b:
            a, b = b, a % b
        g = a
    fc = tmin + g * ((tmax - tmin) // (2 * g)) if g else tmin
    A, c = max(fc - tmin, tmax - fc), int(chain_rate)
    M = -(-(2 * A + c) // c)
    Mp = 4 * (-(-M // 4))
    R = Mp * c
    if Mp < 8 or R > max_rate or R > (1 << 31) - 1 or Mp > 256:
        return None
    M1 = Mp // 4
    return fc, R, 2 * M1, M1, min(8191, 24 * M1 + 1), [v - fc for v in t]


def _offsets(rate, n, seed, margin):
    """n distinct integer offsets in (-R/2 + margin, R/2 - margin), none on a round number."""
    rng = np.random.default_rng(seed)
    lim = rate // 2 - margin
    return [int(v) for v in rng.choice(np.arange(-lim, lim), size=n, replace=False)]


READS, READS_LONG = fdd.READS, fdd.READS_LONG
NBFM12 = fdd.NBFM12
K19, C19, F19 = plan_stages(64)              # 19.2 Msps of a 300 kHz chain: M' = 64, K = 32, M1 = 16, 385 taps

# name -> (parameters, capture rate, K, offsets, coarse (M1, h1, S1), fine (M2, h2, S2), capture keyword arguments,
# reads).  The coarse sum carries the twiddles' 2^15 on top of the taps' gain, so Q15 unity-gain coarse taps take 30.
SHAPES = {
    # the shell's plan at 19.2 Msps for a 300 kHz NBFM chain, 256 channels at arbitrary offsets (a signal on every 16th)
    "nbfm_19m2_c256": (NBFM12, 19_200_000, K19, _offsets(19_200_000, 256, 7, 150_000), C19, F19,
                       dict(every=16), READS_LONG),
    # fm2b's -F 9 chain (2.4 Msps): M' = 8, K = 4 bins of 4.8 MHz, coarse rate 9.6 Msps
    "fm2b_f9": (with_(frd.FM2B, offset_tuning=1), 19_200_000) + plan_stages(8)[:1] +
               ([-4_812_345, 3_001_234, 17],) + plan_stages(8)[1:] + (dict(deviation=75000.0), READS_LONG),
    # am and raw at 24 kHz: M' = 100, K = 50 bins of 48 kHz at 2.4 Msps
    "am_m100": (with_(fac.AM, downsample=1, offset_tuning=1), 2_400_000) + plan_stages(100)[:1] +
               ([-1_187_003, 23_457],) + plan_stages(100)[1:] + ({}, READS),
    "raw_m100": (with_(fac.RAW, downsample=1, offset_tuning=1), 2_400_000) + plan_stages(100)[:1] +
                ([0, 311_111, -311_111, 1_199_999],) + plan_stages(100)[1:] + ({}, READS),
    # squelch with -L: 1.008 Msps chain, M' = 8 at 8.064 Msps, channels that fall quiet half way
    "fm_lut_squelch": (with_(fac.FM24K_LUT, squelch_level=60, offset_tuning=1), 8_064_000) + plan_stages(8)[:1] +
                      ([-3_500_001, 1_234_567],) + plan_stages(8)[1:] + (dict(quiet_half=True), READS_LONG),
    # K = 3 with sum |h1| = 2^22 - 1 at S1 = 33: gain 16, coarse outputs that saturate
    "raw_sat_k3": (with_(fac.RAW, downsample=2, offset_tuning=1), 1_008_000, 3, [0, 335_999, -170_001, 1],
                   (3, frs.near_limit(17, 120e3 / 1.008e6), 33), (2, fdd.lowpass(9, 0.2), 15),
                   dict(amplitude=4000.0), READS),
    # K = 4096 with sum |h1| = 2^22 - 1 at S1 = 33, M1 = 64, M2 = 2
    "raw_sat_k4096": (with_(fac.RAW, downsample=1, offset_tuning=1), 2_048_000, 4096,
                      [0, 250, -1_023_999, 1_023_999, 250, 777_777],
                      (64, frs.near_limit(129, 0.5 / 64), 33), (2, fdd.lowpass(17, 0.2), 15),
                      dict(amplitude=4000.0), READS),
    # channels exactly on bin centres (w = 0) and exactly on bin edges (ties round up): K = 48 bins of 48 kHz
    "raw_centres_edges": (with_(fac.RAW, downsample=1, offset_tuning=1), 2_304_000) + plan_stages(96)[:1] +
                         ([0, 48_000, -96_000, 1_104_000, 24_000, -24_000, 1_128_000, -1_128_000, 72_000],) +
                         plan_stages(96)[1:] + ({}, READS),
}


def case_input(name, seed=0):
    """(params, R, K, offsets, coarse, fine, capture, reads) of a shape."""
    p, rate, K, offs, coarse, fine, kw, reads = SHAPES[name]
    kw = dict(kw)
    every = kw.pop("every", 1)
    x = fmx.capture(fdd.n_complex_for(reads), rate, offs[::every], 1700 + seed + len(name), **kw)
    return p, rate, K, offs, coarse, fine, x, reads
