"""Cases of the tests of decimating mixing handles (rxb200_fm_mix_create_ddc): a numpy model of the digital down-converter
(the integer mixer of fm_mix.mix_model over the library's own table, then the decimating FIR with its rounding shift and
int16 saturation), windowed-sinc tap sets quantised to int32, the channel shapes with their captures and ragged read
sequences, and the per-read decimated streams the reference and the port demodulate.

Channel k of a decimating handle is the reference's rtlsdr_callback() + full_demod() on the decimated stream of
mix_k(capture): capture read r maps to one chain read of the outputs whose emission point e_m = m*M + M - 1 falls in
it.  Read lengths are not multiples of M, so the phase within M moves from read to read.
"""
import numpy as np

import fm_any_chunk as fac
import fm_mix as fmx
import fm_read as frd
from fm_any_chunk import M_FM, P, with_


def lowpass(n_taps, cutoff, gain_bits=15):
    """A Hamming-windowed sinc low-pass with its cutoff at `cutoff` times the capture rate, quantised to int32 taps
    whose sum is about 2^gain_bits (unity DC gain at shift gain_bits)."""
    j = np.arange(n_taps) - (n_taps - 1) / 2.0
    h = np.sinc(2.0 * cutoff * j) * np.hamming(n_taps) if n_taps > 1 else np.ones(1)
    return np.round(h / h.sum() * float(1 << gain_bits)).astype(np.int32)


def wide(taps, shift):
    """Whether the library accumulates in 64 bits: sum |h| * 32768 + 2^(S-1) >= 2^31."""
    return int(np.abs(taps.astype(np.int64)).sum()) * 32768 + ((1 << (shift - 1)) if shift else 0) >= (1 << 31)


def ddc_model(cs16, table, taps, decim, shift, pos=0, hist=None, table_phase=None):
    """The DDC over one call: int16[2c] capture -> (int16[2 * n_out] decimated stream, the new history).

    pos: capture samples before this call (emission points are global samples m*M + M - 1); hist: the raw capture's
    last T - 1 complex samples before the call as int16[2(T - 1)] (None: zeros, the state after create or reset);
    table_phase: the mixer entry of the call's first sample (default pos, as in a handle)."""
    x = np.asarray(cs16, dtype=np.int16).reshape(-1)
    taps = np.asarray(taps, dtype=np.int64)
    T, M, H = taps.size, int(decim), taps.size - 1
    h = np.zeros(2 * H, np.int16) if hist is None else np.asarray(hist, dtype=np.int16).reshape(-1)
    assert h.size == 2 * H
    tp = pos if table_phase is None else table_phase
    ext = np.concatenate([h, x])
    z = fmx.mix_model(ext, table, tp - H).reshape(-1, 2).astype(np.int64)   # entry (tp - H + i) mod L, zeros stay 0
    c = x.size // 2
    m0, m1 = pos // M, (pos + c) // M
    e = np.arange(m0, m1, dtype=np.int64) * M + M - 1 - pos                  # local emission points, in [0, c)
    out = np.empty((e.size, 2), dtype=np.int64)
    win = np.lib.stride_tricks.sliding_window_view(z, T, axis=0)            # win[i] = z[i .. i + T), shape (., 2, T)
    hr = taps[::-1]
    blk = max(1, (1 << 22) // max(T, 1))
    for a in range(0, e.size, blk):
        w = win[e[a:a + blk]]                                                # windows ending at e + H in ext
        out[a:a + blk] = np.einsum("ukt,t->uk", w, hr)
    y = out if shift == 0 else (out + (1 << (shift - 1))) >> shift
    y = np.clip(y, -32768, 32767).astype(np.int16).reshape(-1)
    return y, (ext[ext.size - 2 * H:].copy() if H else np.zeros(0, np.int16))


def decimated_reads(x, table, ddc, lens16):
    """The model over the read sequence: the decimated stream of each read (possibly empty), in order."""
    decim, taps, shift = ddc
    out, pos, hist = [], 0, None
    for a, n in fac.seq_bounds(x.size, lens16):
        y, hist = ddc_model(x[a:a + n], table, taps, decim, shift, pos, hist)
        out.append(y)
        pos += n // 2
    return out


def decimated_len(pos, n_int16, decim):
    """int16 the chain sees from a call of n_int16 capture int16 after pos capture samples."""
    c = n_int16 // 2
    return 2 * ((pos + c) // decim - pos // decim)


READS = [2 * 20011, 2 * 37, 2 * 6007, 2 * 33331]     # complex 20011, 37, 6007, 33331: none a multiple of any M below
READS_LONG = [2 * 20011, 2 * 6007, 2 * 33331]         # every read decimates past 2^P samples (fm2b's passes) and
                                                      # hands the chain at least one boxcar (the squelch at D = 42)

NBFM12 = with_(P(mode=M_FM, downsample=12, custom_atan=2, rate_out=25000), offset_tuning=1)   # 300 kHz -> 25 kHz, lut

# name -> (parameters, capture rate, offsets in Hz, (M, taps, S), capture keyword arguments, reads)
SHAPES = {
    # 19.2 Msps, M = 64, 257 taps, 300 kHz into a D = 12 lut NBFM chain, channels on a 25 kHz raster out to +-9 MHz
    "nbfm_m64_t257": (NBFM12, 19_200_000, [-9_000_000, -25000, 0, 25000, 9_000_000],
                      (64, lowpass(257, 12500 / 19.2e6), 15), {}, READS_LONG),
    # the same on READS: the 37-sample read decimates to 0 or 1 sample, a chain read that completes no boxcar
    "nbfm_m64_t257_short": (NBFM12, 19_200_000, [-9_000_000, -25000, 0, 25000, 9_000_000],
                            (64, lowpass(257, 12500 / 19.2e6), 15), {}, READS),
    # 19.2 Msps, M = 8 into fm2b's -F 9 chain (2.4 Msps, 3 passes), three broadcast channels
    "fm2b_f9_m8": (with_(frd.FM2B, offset_tuning=1), 19_200_000, [-4_800_000, 0, 3_000_000],
                   (8, lowpass(33, 120e3 / 19.2e6), 15), dict(deviation=75000.0), READS_LONG),
    # am and raw at M = 100: 2.4 Msps -> 24 kHz, chain D = 1
    "am_m100": (with_(fac.AM, downsample=1, offset_tuning=1), 2_400_000, [-30000, 10000],
                (100, lowpass(301, 6000 / 2.4e6), 15), {}, READS),
    "raw_m100": (with_(fac.RAW, downsample=1, offset_tuning=1), 2_400_000, [0, 24000, -48000],
                 (100, lowpass(201, 9000 / 2.4e6), 15), {}, READS),
    # squelch with -L: 4.032 Msps, M = 4 -> 1.008 Msps, D = 42 lut, channels that fall quiet half way
    "fm_lut_squelch_m4": (with_(fac.FM24K_LUT, squelch_level=60, offset_tuning=1), 4_032_000, [-200000, 200000],
                          (4, lowpass(33, 80e3 / 4.032e6), 15), dict(quiet_half=True), READS_LONG),
    # gain 16 through taps with sum |h| ~ 2^17 at S = 13: the 64-bit accumulator, and outputs that saturate
    "raw_wide_m3": (with_(fac.RAW, downsample=2, offset_tuning=1), 1_008_000, [0, 48000],
                    (3, lowpass(17, 120e3 / 1.008e6, gain_bits=17), 13), dict(amplitude=4000.0), READS),
}


def n_complex_for(lens16, extra=777):
    return fmx.n_complex_for(lens16, extra)


def case_input(name, seed=0):
    """(params, rate, offsets, (M, taps, S), capture, reads) of a shape."""
    p, rate, offs, ddc, kw, reads = SHAPES[name]
    return p, rate, offs, ddc, fmx.capture(n_complex_for(reads), rate, offs, 900 + seed + len(name), **kw), reads


def nonempty(reads):
    """The decimated reads the chain runs on (a read with no output runs no chain call) and their lengths."""
    keep = [r for r in reads if r.size]
    return np.concatenate(keep) if keep else np.zeros(0, np.int16), [int(r.size) for r in keep]
