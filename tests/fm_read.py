"""Cases of the per-read rx_fm tests (rxb200_fm_process_read): shapes with fifth_order passes, which a device read of any
even length reaches through the read entry point, the read lengths they run on, and a slot-level model of the
reference's in-place passes over one read.

The runs of the port and of the reference over a read sequence are fm_any_chunk's: one run call per read on one
configured state.  Parameters are the reference's derived numbers, spelled out so that the CPU tests need no GPU library.
"""
import numpy as np

from fm_any_chunk import M_AM, M_FM, M_LSB, M_RAW, M_USB, P, signal, with_  # noqa: F401
from rx_tools_b200 import synth

# -M wbfm -s 300k -F 9 -r 48k: the project's default workload (bench fm2b)
FM2B = P(mode=M_FM, downsample=8, downsample_passes=3, comp_fir_size=9, custom_atan=1, deemph=1, deemph_a=23,
         rate_out=300000, rate_out2=48000)


def passes(p_, fir=True, **kw):
    """A shape with p_ fifth_order passes (downsample 2^p_), the droop FIR with fir."""
    d = dict(mode=M_FM, downsample=1 << p_, downsample_passes=p_, comp_fir_size=9 if fir else 0, custom_atan=1,
             rate_out=max(24000, 2400000 >> p_))
    d.update(kw)
    return P(**d)


def shapes():
    """name -> parameters: P = 1..10 (for P <= 3 also without -F 9), every mode and discriminator, the squelch, the raw
    and audio DC blocks, offset tuning, de-emphasis with the resampler and -o 2."""
    s = {}
    for p_ in range(1, 11):
        s[f"fm_fast_p{p_}_fir"] = passes(p_)
        if p_ <= 3:
            s[f"fm_fast_p{p_}"] = passes(p_, fir=False)
    s["fm2b"] = FM2B
    s["fm_std_p2_fir"] = passes(2, custom_atan=0)
    s["fm_lut_p4_fir"] = passes(4, custom_atan=2)
    s["fm_ale_p5"] = passes(5, fir=False, custom_atan=3)
    s["am_p3_fir"] = passes(3, mode=M_AM, output_scale=6)
    s["usb_p6_fir"] = passes(6, mode=M_USB, output_scale=4)
    s["lsb_p7"] = passes(7, fir=False, mode=M_LSB, output_scale=4)
    s["raw_p3_fir"] = passes(3, mode=M_RAW)
    s["raw_p5"] = passes(5, fir=False, mode=M_RAW)
    s["fm_lut_p4_squelch"] = passes(4, custom_atan=2, squelch_level=60)
    s["usb_p2_squelch_adc"] = passes(2, fir=False, mode=M_USB, output_scale=4, squelch_level=30, dc_block_audio=1)
    s["fm_fast_p3_rdc"] = passes(3, dc_block_raw=1, rdc_block_const=9)
    s["am_p5_rdc_adc"] = passes(5, mode=M_AM, output_scale=6, dc_block_raw=1, rdc_block_const=30, dc_block_audio=1)
    s["raw_p2_rdc"] = passes(2, mode=M_RAW, dc_block_raw=1, rdc_block_const=9)
    s["fm_fast_p3_offset"] = with_(FM2B, offset_tuning=1)
    s["fm_lut_p6_deemph_even"] = passes(6, custom_atan=2, deemph=1, deemph_a=16, rate_out=37500, rate_out2=24000)
    s["fm_fast_p2_o2"] = passes(2, post_downsample=2)
    return s


def read_lens(p_, seed, n_extra=16, even_dec=False):
    """Read lengths in int16 for a shape with p_ passes: one of every residue mod 2^(p_+1) int16 (so every pattern of
    lone I samples at the passes' ends occurs), a read of exactly 2^p_ complex samples, and n_extra lengths drawn up to
    8192 complex, shuffled.  even_dec: only reads whose (n_int16 / 2) >> p_ is even (-o 2)."""
    rng = np.random.default_rng(seed)
    g = 2 << p_
    lens = [g * int(rng.integers(1, 4)) + r for r in range(0, g, 2)]
    lens += [2 * int(v) for v in rng.integers(1 << p_, 8193, size=n_extra)]
    rng.shuffle(lens)
    lens.insert(int(rng.integers(0, len(lens) + 1)), g)
    if even_dec:
        lens = [n + (2 << p_) if ((n // 2) >> p_) % 2 else n for n in lens]
    return lens


def stream_for(lens, seed, quiet_half=False):
    """The signal for one pass over the read sequence."""
    n = sum(lens) // 2
    if quiet_half:
        h = n // 2
        return np.concatenate([signal(h, seed), signal(n - h, seed + 1, quiet=True)])
    return signal(n, seed)


# ---- slot-level model of full_demod's passes over one read of n int16 (src/rtl_fm.c:411-440, :765-768): every slot
# of lowpassed carries the pass that last wrote it; a pass that reads a slot the previous pass did not write reads stale
# data from an earlier read.
def pass_model(n_int16, p_):
    """Per pass l: (I inputs, Q inputs, I outputs written, Q outputs written, stale slots read)."""
    gen = np.zeros(n_int16, dtype=np.int64)              # 0: written by rtlsdr_callback (this read's input)
    out = []
    for l in range(p_):
        length = n_int16 >> l
        row = []
        for comp, ln in ((0, length), (1, length - 1)):     # fifth_order(lowpassed + comp, ln)
            idx = np.arange(0, ln, 2) + comp                  # the component's samples: data[0], data[2], ...
            stale = int(np.count_nonzero(gen[idx] != l))
            # outputs at even sample indices i = 0, 2, 4, ... (data[i] for i = 0 and i % 4 == 0 < ln), written to data[i/2]
            src = np.arange(0, ln, 4)
            dst = src // 2 + comp
            row.append((idx.size, src.size, stale, dst))
        for _, _, _, dst in row:
            gen[dst] = l + 1
        out.append((row[0][0], row[1][0], row[0][1], row[1][1], row[0][2] + row[1][2]))
    return out, gen


def stream_counts(n_int16, p_, l):
    """The read kernel's counts at pass l (l = p_: after the passes): pairs n >> l, plus a lone I when (n >> (l-1)) is
    odd -- (I samples, Q samples) that pass runs over."""
    n = n_int16 // 2
    pairs = n >> l
    lone = 1 if l > 0 and (n >> (l - 1)) & 1 else 0
    return pairs + lone, pairs


def golden_cases():
    """name -> (params, input, lens16): the fm2b shape over reads of 2044 complex samples, of 1021:333:4093 and of
    131071, and one read sequence per pass count with a shuffled residue set."""
    out = {}
    x = synth.cfg2_iq(3 << 19)
    out["fm2b_r2044"] = (FM2B, x, [2 * 2044])
    out["fm2b_r1021_333_4093"] = (FM2B, x, [2 * 1021, 2 * 333, 2 * 4093])
    out["fm2b_r131071"] = (FM2B, x, [2 * 131071])
    for p_ in (1, 2, 4, 6, 8, 10):
        lens = read_lens(p_, 900 + p_, n_extra=6)
        out[f"p{p_}_residues"] = (passes(p_), stream_for(lens, 950 + p_), lens)
    out["raw_p5_residues"] = (passes(5, fir=False, mode=M_RAW), stream_for(read_lens(5, 905), 960), read_lens(5, 905))
    return out
