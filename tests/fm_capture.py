"""Cases of the tests of the rx_fm shell's capture mode (RXB200_CAPTURE_RATE): the capture plan restated in Python, the
shell's -f parsing and tuned frequencies, the block rule, the named command lines with their captures, each channel's
decimated stream (fm_ddc.ddc_model over the library's mixer table and rx_power's capture-mode filter) cut into the reads
the chain sees, and the squelch rule applied to the port's output.

Channel k of a capture-mode run is the reference's rtlsdr_callback() + full_demod() on the decimated stream of channel
k, one read per block: a block is M * 131072 complex capture samples, so each full block is one chain read of 131072
complex samples, and a last partial block is handed on when it decimates to at least min_chunk int16.
"""
import math

import numpy as np

import fm_any_chunk as fac
import fm_ddc as fdd
import oracle
from rx_tools_b200 import fm, power, synth

CHUNK = 131072                       # complex samples per chain read (src/rtl_fm.c:871)
MIX_MAX_PERIOD = 1 << 20


# ---- the plan, restated (include/rxb200.h, "rx_fm channels of one capture in the shell")
def plan_rule(tuned, c, cap):
    """(fc, M, R, T, offsets) or the refusal as a string: "rate" (R above the cap or 2^31 - 1, or M > 256) or
    "period" (a mixer table with a period above 2^20)."""
    tmin, tmax = min(tuned), max(tuned)
    g = 0
    for t in tuned:
        g = math.gcd(g, t - tmin)
    fc = tmin if g == 0 else tmin + g * ((tmax - tmin) // (2 * g))
    offs = [t - fc for t in tuned]
    A = max(abs(o) for o in offs)
    M = -(-(2 * A + c) // c)
    R = M * c
    if R > cap or R > 2**31 - 1 or M > 256:
        return "rate"
    if any(R // math.gcd(R, abs(o)) > MIX_MAX_PERIOD for o in offs):
        return "period"
    assert all(2 * abs(o) < R for o in offs)
    return fc, M, R, min(8191, 32 * M + 1), offs


# ---- the shell's -f values (parse_scaled, add_range) and tuned frequencies (capture_freq)
def parse_scaled(s):
    mult = {"k": 1e3, "K": 1e3, "m": 1e6, "M": 1e6, "g": 1e9, "G": 1e9}.get(s[-1:])
    return float(s[:-1]) * mult if mult else float(s)


def freqs_of(values):
    """-f values (a:b:step ranges expanded as the shell does, C int arithmetic) -> the frequencies in Hz."""
    out = []
    for v in values:
        if ":" in v:
            a, b, st = v.split(":")
            f = int(parse_scaled(a))
            while f <= int(parse_scaled(b)):
                out.append(f)
                f += int(parse_scaled(st))
        else:
            out.append(int(parse_scaled(v)) & 0xFFFFFFFF)
    return out


def tuned_of(freqs, der, wbfm=False, edge=False):
    """capture_freq(k) with offset_tuning on (capture_freq_offset 0): +16 kHz under wbfm, + rate_out * post / 2 with
    -E edge."""
    p = der.params
    return [f + (16000 if wbfm else 0) + der.capture_freq_offset + ((p.rate_out * p.post_downsample) // 2 if edge else 0)
            for f in freqs]


# ---- blocks
def min_chunk(p):
    """The plain shell's min_chunk without -o: 2^P complex with passes, one boxcar with a per-chunk stage, else one."""
    if p.downsample_passes:
        return 2 << p.downsample_passes
    return 2 * p.downsample if (p.squelch_level or p.dc_block_audio or p.dc_block_raw) else 2


def blocks(n_complex, decim, min_chunk16):
    """Capture complex samples of each block handed on: whole blocks of M * 131072, then the partial block if it
    decimates to at least min_chunk int16."""
    full, rest = divmod(n_complex, decim * CHUNK)
    out = [decim * CHUNK] * full
    if rest and 2 * (rest // decim) >= min_chunk16:
        out.append(rest)
    return out


def chain_reads(block_lens, decim):
    """The int16 of each chain read: a block of b capture samples starting at a multiple of M decimates to b // M."""
    return [2 * (b // decim) for b in block_lens]


# ---- named command lines
# name -> (-f values, other arguments, derive_params keywords, capture: (n_complex, stop sample per channel or None))
SHAPES = {
    # three NBFM channels 25 kHz apart: c = 1.008 Msps, M = 2; the last block is partial and handed on
    "nbfm_3ch": (["162.4M", "162.425M", "162.45M"], [], {}, (2 * 2 * CHUNK + 70001, None)),
    # AM with -E wav, centred between channels of a 10 kHz grid
    "am_wav": (["10M", "10.03M", "10.05M"], ["-M", "am", "-E", "wav"], dict(mode=fm.MODE_AM),
               (2 * CHUNK + 1001, None)),
    # squelch: channels that fall quiet at different blocks, -t 0
    "squelch_3ch": (["100M:100.2M:100k"], ["-l", "60", "-t", "0"], dict(squelch_level=60),
                    (3 * 2 * CHUNK + 5000, [int(1.3 * 2 * CHUNK), int(2.6 * 2 * CHUNK), None])),
    # fm2b's command line: fifth_order passes (P = 3), so the last block must decimate to 2^P samples
    "fm2b_f9": (["99.4M", "100M", "100.6M"], ["-M", "wbfm", "-s", "300k", "-F", "9", "-r", "48k"],
                dict(wbfm=1, rate_s=300000, rate_r=48000, use_F=1, comp_fir_size=9), (2 * CHUNK + 999, None)),
}
# DESIGN 4.4's FM-band plan: 19 wbfm channels, M = 21, R = 21.42 Msps, T = 673
WBFM19 = (["88.1M:107.9M:1.1M"], ["-M", "wbfm"], dict(wbfm=1), (21 * CHUNK + 40000, None))


def plan_of(fvals, args, kw, cap=10**10):
    """(chain parameters, frequencies, CapturePlan, offsets, taps) of a command line, as the shell derives them."""
    der = fm.derive_params(offset_tuning=1, **kw)
    freqs = freqs_of(fvals)
    tuned = tuned_of(freqs, der, wbfm=bool(kw.get("wbfm")), edge="edge" in args)
    pl, offs = fm.plan_capture(tuned, der.capture_rate, cap)
    return der.params, freqs, pl, offs, power.ddc_lowpass(pl.decim, pl.n_taps, 15)


def capture(n_complex, rate, offsets, seed, stops=None, deviation=2500.0, amplitude=2500.0):
    """An FM channel at each offset, channel k switched off from sample stops[k] (None: never), plus a little noise."""
    x = np.zeros(2 * n_complex, dtype=np.int64)
    for k, f in enumerate(offsets):
        tones = [(300.0 + 110.0 * k, 0.7), (1700.0 + 230.0 * k, 0.3)]
        ch = synth.fm_iq(n_complex, fs=float(rate), deviation_hz=deviation, tones=tones, amplitude=amplitude,
                         noise_lsb=0, seed=seed + k, center_hz=float(f)).astype(np.int64)
        if stops is not None and stops[k] is not None:
            ch[2 * stops[k]:] = 0
        x += ch
    x += np.random.default_rng(seed).integers(-3, 4, size=x.size)
    return np.clip(x, -32768, 32767).astype(np.int16)


def case(name, seed=0):
    """(arguments of the shell, parameters, frequencies, plan, offsets, taps, capture) of a named shape."""
    fvals, args, kw, (n, stops) = SHAPES[name] if name in SHAPES else WBFM19
    p, freqs, pl, offs, taps = plan_of(fvals, args, kw)
    dev = 75000.0 if kw.get("wbfm") else 2500.0
    x = capture(n, pl.capture_rate, offs, 1700 + seed + len(name), stops, deviation=dev)
    argv = [a for v in fvals for a in ("-f", v)] + args
    return argv, p, freqs, pl, offs, taps, x


def decimated(x, pl, offs, taps):
    """Each channel's decimated stream over the whole capture (fm_ddc.ddc_model)."""
    return [fdd.ddc_model(x, fm.mix_table(pl.capture_rate, o), taps, pl.decim, 15)[0] for o in offs]


def oracle_params(p):
    return oracle.FmParams(**fm.FmParams.from_any(p).reference_fields())


def port_channel(port, p, dec, lens):
    """The port on one channel's decimated stream, one run call per chain read: (pcm, result_len, squelch hits)."""
    y = dec[:sum(lens)]
    return fac.port_run_seq(port, oracle_params(p), y, lens, return_chunks=True)


def squelched(pcm, result_len, hits, conseq, squelch_level, zero):
    """What the shell writes for one channel: per read, nothing when the squelch is active (hits > -t) and -E zero is
    not given, zeros with -E zero, the PCM otherwise."""
    out, pos = [], 0
    for n, h in zip(result_len, hits):
        part = pcm[pos:pos + n]
        pos += n
        if squelch_level and h > conseq:
            if zero:
                out.append(np.zeros_like(part))
            continue
        out.append(part)
    return np.concatenate(out) if out else np.zeros(0, np.int16)


def wav_header(rate, raw):
    """generate_header() (src/rtl_fm.c:1174-1206) as the shell writes it."""
    brate = rate * 2 * (2 if raw else 1)
    return (b"RIFF\xff\xff\xff\xffWAVEfmt \x10\x00\x00\x00\x01\x00" + bytes([2 if raw else 1, 0])
            + rate.to_bytes(4, "little") + brate.to_bytes(4, "little") + bytes([4 if raw else 2, 0, 16, 0])
            + b"data\xff\xff\xff\xff")
