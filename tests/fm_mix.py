"""Cases of the tests of several rx_fm channels of one capture (rxb200_fm_mix_*): wideband captures with a channel at
each offset, the channel shapes they are demodulated with (boxcar and fifth_order, fm / am / raw, the fp64 discriminator
with rotate16_90 left on, squelch with -L), the read sequences, and a numpy model of the integer mixer over the
library's own table (rx_tools_b200.fm.mix_table), so that the model and the library agree on every table entry.

Channel k of a mixing handle is the reference's rtlsdr_callback() + full_demod() on mix_model(capture, table_k): the
oracles run on the model's output, one run call per read, and the library runs on the capture itself.
"""
import numpy as np

import fm_any_chunk as fac
import fm_read as frd
from fm_any_chunk import M_FM, P, with_
from rx_tools_b200 import synth

READS = [2 * 1021, 2 * 333, 2 * 4093]     # the read lengths of every case, in int16, repeated until the capture ends


def mix_model(cs16, table, phase=0):
    """The mixer: int16[2n] CS16 -> int16[2n]; table int32[L][2] of (c, s); sample n uses entry (phase + n) mod L."""
    x = np.asarray(cs16, dtype=np.int16).reshape(-1, 2).astype(np.int64)
    idx = (phase + np.arange(x.shape[0], dtype=np.int64)) % table.shape[0]
    c, s = table[idx, 0].astype(np.int64), table[idx, 1].astype(np.int64)
    out = np.empty_like(x)
    out[:, 0] = (x[:, 0] * c - x[:, 1] * s + (1 << 14)) >> 15
    out[:, 1] = (x[:, 0] * s + x[:, 1] * c + (1 << 14)) >> 15
    return out.astype(np.int16).reshape(-1)                # int64 -> int16 wraps, like the reference's stores


def capture(n_complex, rate, offsets, seed, deviation=2500.0, amplitude=2500.0, quiet_half=False):
    """An FM channel at each offset (own tones, own phase), summed, with a little noise.  quiet_half: the second half
    of every channel 40 dB down (a squelch opens and closes)."""
    x = np.zeros(2 * n_complex, dtype=np.int64)
    for k, f in enumerate(offsets):
        tones = [(300.0 + 110.0 * k, 0.7), (1700.0 + 230.0 * k, 0.3)]
        ch = synth.fm_iq(n_complex, fs=float(rate), deviation_hz=deviation, tones=tones, amplitude=amplitude,
                         noise_lsb=0, seed=seed + k, center_hz=float(f)).astype(np.int64)
        if quiet_half:
            ch[n_complex:] //= 100
        x += ch
    x += np.random.default_rng(seed).integers(-3, 4, size=x.size)
    return np.clip(x, -32768, 32767).astype(np.int16)


def n_complex_for(lens16, extra=777):
    """A capture for three rounds of the read sequence and a short last read."""
    return 3 * sum(lens16) // 2 + extra


# name -> (parameters, capture rate, offsets in Hz, capture keyword arguments)
SHAPES = {
    # fm5a's channel: 2.4 Msps -> 24 kHz, boxcar D = 100, -A lut, on a 12.5 kHz raster
    "fm5a_lut_d100": (with_(fac.FM5A, offset_tuning=1), 2_400_000, [-25000, 0, 12500, 37500], {}),
    # fm2b: -M wbfm -s 300k -F 9 -r 48k, three broadcast channels of a 2.4 Msps capture
    "fm2b_f9": (with_(frd.FM2B, offset_tuning=1), 2_400_000, [-600000, 0, 450000], dict(deviation=75000.0)),
    "am_d42": (with_(fac.AM, offset_tuning=1), 1_008_000, [-30000, 10000], {}),
    "raw_d42": (with_(fac.RAW, offset_tuning=1), 1_008_000, [0, 24000, -48000], {}),
    # the fp64 discriminator, with rotate16_90 still on (any parameters are taken) and a period of 1000 samples
    "fm_std_d10_rotate": (P(mode=M_FM, downsample=10, custom_atan=0, rate_out=100000), 1_000_000, [0, 33000], {}),
    # squelch with -L on a capture whose channels fall quiet half way
    "fm_lut_d42_squelch": (with_(fac.FM24K_LUT, squelch_level=60, offset_tuning=1), 1_008_000, [-20000, 20000],
                           dict(quiet_half=True)),
}


def case_input(name, seed=0):
    """(params, rate, offsets, capture) of a shape."""
    p, rate, offs, kw = SHAPES[name]
    return p, rate, offs, capture(n_complex_for(READS), rate, offs, 700 + seed + len(name), **kw)
