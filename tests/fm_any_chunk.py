"""Cases of the any-length rx_fm tests: shapes without fifth_order passes (downsample_passes == 0), which the library
demodulates for chunks of any whole number of complex samples, the inputs and chunk sequences they run on, and the
runs of the port and of the reference over a ragged chunk sequence (one run call per chunk on one configured state,
through the oracle libraries' own entry points).

Parameters are the reference's derived numbers, spelled out so that the CPU tests need no GPU library:
tests/golden/make_fm_any_chunk_golden.py checks the command-line ones against the reference's own main().
"""
import ctypes as C

import numpy as np

import oracle
from rx_tools_b200 import synth

P = oracle.FmParams
M_FM, M_AM, M_USB, M_LSB, M_RAW = range(5)

# rx_fm command lines (reference optimal_settings) -> parameters
FM1 = P(mode=M_FM, downsample=1, custom_atan=0, rate_out=1024000, rate_out2=24000)            # -M fm -s 1024000 -r 24000
FM2A = P(mode=M_FM, downsample=1, custom_atan=1, deemph=1, deemph_a=181, rate_out=2400000,
         rate_out2=48000)                                                                     # -M wbfm -s 2400000 -r 48000
WBFM = P(mode=M_FM, downsample=6, custom_atan=1, deemph=1, deemph_a=13, rate_out=170000, rate_out2=32000)   # -M wbfm
FM24K_LUT = P(mode=M_FM, downsample=42, custom_atan=2, rate_out=24000)                        # -M fm -s 24k -A lut
AM = P(mode=M_AM, downsample=42, output_scale=6, rate_out=24000)                              # -M am
USB = P(mode=M_USB, downsample=42, output_scale=6, rate_out=24000)                            # -M usb
LSB = P(mode=M_LSB, downsample=42, output_scale=6, rate_out=24000)                            # -M lsb
RAW = P(mode=M_RAW, downsample=42, output_scale=6, rate_out=24000)                            # -M raw
FM5A = P(mode=M_FM, downsample=100, custom_atan=2, rate_out=24000)                            # bench fm5a channel
CLI = {"fm1": (FM1, dict(rate_s=1024000, rate_r=24000)),
       "fm2a": (FM2A, dict(wbfm=1, rate_s=2400000, rate_r=48000)),
       "wbfm": (WBFM, dict(wbfm=1)),
       "fm24k_lut": (FM24K_LUT, dict(rate_s=24000, custom_atan=2)),
       "am": (AM, dict(mode=M_AM)), "usb": (USB, dict(mode=M_USB)), "lsb": (LSB, dict(mode=M_LSB)),
       "raw": (RAW, dict(mode=M_RAW))}


def with_(p, **kw):
    d = dict(vars(p))
    d.update(kw)
    return P(**d)


def shapes():
    """name -> parameters: every P = 0 mode and optional stage the any-length kernel takes (the integer discriminators
    with squelch, raw and audio DC blocks, offset tuning, de-emphasis with the resampler, D = 1 at a = 181, D = 100)."""
    s = {}
    for atan, an in ((0, "std"), (1, "fast"), (2, "lut"), (3, "ale")):
        s[f"fm_{an}_d10"] = P(mode=M_FM, downsample=10, custom_atan=atan, rate_out=100000)
    s["fm_lut_d100"] = FM5A
    s["fm_fast_d1_deemph181"] = FM2A
    s["fm_std_d1_resample"] = FM1
    s["wbfm"] = WBFM
    s["am"], s["usb"], s["lsb"], s["raw"] = AM, USB, LSB, RAW
    s["fm_fast_d6_offset"] = with_(WBFM, offset_tuning=1)
    s["fm_lut_d42_squelch"] = with_(FM24K_LUT, squelch_level=60)
    s["fm_fast_d42_rdc"] = P(mode=M_FM, downsample=42, custom_atan=1, rate_out=24000, dc_block_raw=1, rdc_block_const=9)
    s["fm_ale_d8_adc"] = P(mode=M_FM, downsample=8, custom_atan=3, rate_out=128000, rate_out2=32000, dc_block_audio=1)
    s["am_d42_rdc_adc"] = with_(AM, dc_block_raw=1, rdc_block_const=30, dc_block_audio=1)
    s["fm_lut_d3_deemph_even"] = P(mode=M_FM, downsample=3, custom_atan=2, deemph=1, deemph_a=16, rate_out=300000,
                                   rate_out2=48000)
    s["usb_d5_squelch_adc"] = P(mode=M_USB, downsample=5, output_scale=4, rate_out=200000, squelch_level=30,
                                dc_block_audio=1)
    return s


INTEGER = lambda p: not (p.mode == M_FM and p.custom_atan == 0)    # noqa: E731  every result through integer arithmetic


def signal(n_complex, seed, quiet=False):
    """An FM test signal with a silent stretch (squelch and de-emphasis dead zone) and some DC (the DC blocks)."""
    rng = np.random.default_rng(seed)
    amp = 60.0 if quiet else 9000.0
    x = synth.fm_iq(n_complex, fs=1.0e6, deviation_hz=40e3, tones=[(900.0, 0.7), (3100.0, 0.3)], amplitude=amp,
                    noise_lsb=3, seed=seed).astype(np.int32)
    a = int(rng.integers(0, max(1, n_complex // 2)))
    x[2 * a:2 * (a + n_complex // 6)] = 0
    x[0::2] += 300
    x[1::2] -= 200
    return np.clip(x, -32768, 32767).astype(np.int16)


def loud_quiet(n_complex, seed):
    """Loud first half, quiet second half: a squelch opens and closes."""
    h = n_complex // 2
    return np.concatenate([signal(h, seed), signal(n_complex - h, seed + 1, quiet=True)])


def ragged_lens(rng, n, lo, hi):
    """n chunk lengths in int16, uniform in [lo, hi] complex samples."""
    return [2 * int(v) for v in rng.integers(lo, hi + 1, size=n)]


# ---- ragged chunk sequences on the oracles: one configuration, then one run call per chunk.  Both libraries keep
# their state between run calls (only orx_fm_new / ref_fm_configure reset it), so a call per chunk is the reference's
# rtlsdr_callback + full_demod once per chunk of the given length.
def seq_bounds(n_int16, lens16):
    """(start, length) in int16 of each chunk: the lengths of `lens16` in turn, repeated until the stream ends (the last
    chunk is what is left), the way a device that reads in packets hands the stream on."""
    lens16 = [int(v) for v in lens16]
    assert lens16 and all(v > 0 and v % 2 == 0 for v in lens16), lens16
    out, pos, i = [], 0, 0
    while pos < n_int16:
        n = min(lens16[i % len(lens16)], n_int16 - pos)
        out.append((pos, n))
        pos += n
        i += 1
    return out


def _pi(a):
    return a.ctypes.data_as(C.POINTER(C.c_int))


def _p16(a):
    return a.ctypes.data_as(C.POINTER(C.c_int16))


def _run_seq(run_one, x, lens16, return_chunks):
    """run_one(chunk, out, result_len[1], squelch_hits[1]) -> int16 written, once per chunk of the sequence."""
    bounds = seq_bounds(x.size, lens16)
    out = np.empty(x.size + 64 * (len(bounds) + 1), dtype=np.int16)
    rl = np.zeros(len(bounds), dtype=np.int32)
    hits = np.zeros(len(bounds), dtype=np.int32)
    one_len, one_hit = np.zeros(1, dtype=np.int32), np.zeros(1, dtype=np.int32)
    w = 0
    for c, (pos, n) in enumerate(bounds):
        k = run_one(np.ascontiguousarray(x[pos:pos + n]), out[w:], one_len, one_hit)
        if k < 0:
            raise RuntimeError(f"run failed on chunk {c}: {k}")
        rl[c], hits[c] = one_len[0], one_hit[0]
        w += k
    res = out[:w].copy()
    return (res, rl, hits) if return_chunks else res


def _levels_seq(run_one, x, lens16):
    bounds = seq_bounds(x.size, lens16)
    lv = np.zeros(len(bounds), dtype=np.int32)
    one = np.zeros(1, dtype=np.int32)
    for c, (pos, n) in enumerate(bounds):
        if run_one(np.ascontiguousarray(x[pos:pos + n]), one) != 1:
            raise RuntimeError(f"levels run failed on chunk {c}")
        lv[c] = one[0]
    return lv


def port_run_seq(port, params, cs16, lens16, return_chunks=False):
    """The port (oracle.Port) over a ragged chunk sequence; same returns as Port.fm_run."""
    x = np.ascontiguousarray(cs16, dtype=np.int16)
    pc = params.to_c()
    h = port.L.orx_fm_new(C.byref(pc))
    try:
        return _run_seq(lambda part, out, rl, hits: port.L.orx_fm_run(h, _p16(part), part.size, part.size, _p16(out),
                                                                      out.size, _pi(rl), _pi(hits)),
                        x, lens16, return_chunks)
    finally:
        port.L.orx_fm_free(h)


def port_levels_seq(port, params, cs16, lens16):
    """Per-chunk rms() (-L) of the port over a ragged chunk sequence."""
    x = np.ascontiguousarray(cs16, dtype=np.int16)
    pc = params.to_c()
    h = port.L.orx_fm_new(C.byref(pc))
    try:
        return _levels_seq(lambda part, lv: port.L.orx_fm_run_levels(h, _p16(part), part.size, part.size, _pi(lv)),
                           x, lens16)
    finally:
        port.L.orx_fm_free(h)


def ref_run_seq(ref, params, cs16, lens16, return_chunks=False):
    """The unmodified reference (oracle.RefFm) over a ragged chunk sequence; same returns as RefFm.run."""
    x = np.ascontiguousarray(cs16, dtype=np.int16)
    pc = params.to_c()
    if ref.L.ref_fm_configure(C.byref(pc)) != 0:
        raise ValueError("bad params")
    return _run_seq(lambda part, out, rl, hits: ref.L.ref_fm_run(_p16(part), part.size, part.size, _p16(out), out.size,
                                                                 _pi(rl), _pi(hits)),
                    x, lens16, return_chunks)


def ref_levels_seq(ref, params, cs16, lens16):
    """Per-chunk rms() (-L) of the reference over a ragged chunk sequence."""
    x = np.ascontiguousarray(cs16, dtype=np.int16)
    pc = params.to_c()
    if ref.L.ref_fm_configure(C.byref(pc)) != 0:
        raise ValueError("bad params")
    return _levels_seq(lambda part, lv: ref.L.ref_fm_run_levels(_p16(part), part.size, part.size, _pi(lv)), x, lens16)


def seq_len(lens16):
    """A stream for a ragged sequence: the whole sequence, then its first chunk one sample short (every chunk, the
    last one included, at least two boxcars long when ragged_lens drew it so)."""
    return sum(lens16) // 2 + lens16[0] // 2 - 1


def golden_cases():
    """name -> (params, input, lens16): the benchmark shapes at chunks of 131071 / 131069 complex and one
    ragged sequence per mode.  lens16 repeats until the stream ends (seq_bounds)."""
    out = {}
    x1 = synth.cfg1_iq(1 << 20)
    for atan, an in ((0, "std"), (1, "fast"), (2, "lut")):
        out[f"fm1_{an}_c131071"] = (with_(FM1, custom_atan=atan), x1, [2 * 131071])
    out["fm2a_c131071"] = (FM2A, synth.cfg2_iq(3 << 20), [2 * 131071])
    for ch in range(3):
        out[f"fm5a_ch{ch}_c131069"] = (FM5A, synth.cfg5_iq(1_000_001, ch), [2 * 131069])
    rng = np.random.default_rng(77)
    for name, p in (("seq_fm_std", with_(FM24K_LUT, custom_atan=0)), ("seq_fm_fast", with_(FM24K_LUT, custom_atan=1)),
                    ("seq_fm_lut", FM24K_LUT), ("seq_fm_ale", with_(FM24K_LUT, custom_atan=3)), ("seq_wbfm", WBFM),
                    ("seq_am", AM), ("seq_usb", USB), ("seq_lsb", LSB), ("seq_raw", RAW)):
        lens = ragged_lens(rng, 12, 2 * p.downsample, 9000)
        out[name] = (p, signal(seq_len(lens), 400 + len(out)), lens)
    return out
