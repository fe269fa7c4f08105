"""Seeded draws for the specialised rx_fm paths: the split kernel with the row front end (kernel_kind 1), the stream
path (kernel_kind 3) and the fused kernel's compile-time specialisations (kernel_kind 0).

A draw is everything one parity check needs: the parameters, the chunk length, the call splits (always on chunk
boundaries: SURVEY F7 makes the chunk part of every result), the environment knobs read at create, the
``rxb200_fm_tune`` values, the channel inputs and the kernel_kind every call must report.  The expectation restates the
rules of ``rxb200_fm_create`` and ``fm_launch`` (csrc/fm_kernels.cu), so a change of those rules shows up as a failing
test instead of a silently different path.  No fixtures: the GPU tests, the CPU coverage test and the oracle pin import
the same families."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from oracle import ATAN_FAST, ATAN_LUT, MODE_FM, FmParams

ROW_LEN = 1024                      # complex samples per row of the row front end (fm_rows.cuh)
ROW_I16 = 2 * ROW_LEN

# ---- the host planner's figures (csrc/fm_kernels.cu, fm_rows.cuh) and the H100's shared memory (cudaDeviceProp)
SMEM_PER_SM, SMEM_RESERVED, SMEM_OPTIN = 233472, 1024, 232448
ROWS_FE_WARPS, ROWS_MINB, ROWS_STAGES, ROW_BYTES = 7, 2, 2, 4 * ROW_LEN
SPLIT_STATIC_SMEM = 1840            # static shared memory of every fm_split_kernel instantiation (ptxas; checked in
                                    # tests/test_fm_paths_cpu.py against the build's ptxas log)
FUSED_STATIC_SMEM = 3344            # ... of the fused kernels with a back end (SPEC 0, 1, 2; same check)
FUSED_T = {0: 256}                  # fm_cta_threads: 256 at P = 0, 128 with passes
PCM_PAD_SEG = 2

ROWS_A = (1, 2, 3, 13, 23, 46, 91, 181, 301, 541, 601)
ROWS_CHUNK_ROWS = (1, 2, 3, 5, 7, 32, 128)
RATE_OUT = {1: 1_200_000, 2: 600_000, 3: 300_000}
RATE_OUT2 = {"rate_out": lambda r: r, "rate_out-1": lambda r: r - 1, "rate_out/5": lambda r: r // 5,
             "rate_out/6": lambda r: r // 6, "48000": lambda r: 48_000, "44100": lambda r: 44_100,
             "32000": lambda r: 32_000, "8000": lambda r: 8_000}
SERIAL = ("deemph", "resample", "both")
INPUTS = ("loud", "quiet", "noise", "overshoot")


@dataclass
class Draw:
    family: str
    seed: int
    params: FmParams
    chunk: int                       # int16 per chunk
    cuts: list                       # int16 offsets of the call boundaries, 0 first, the stream length last
    x: np.ndarray                    # int16 [n_channels][n]
    kinds: list                      # kernel_kind expected after every call
    single_kind: int                 # ... after one call over the whole stream
    env: dict = field(default_factory=dict)
    tune: tuple = (0, 0)             # rxb200_fm_tune(segment_len, deemph_warmup)
    tags: dict = field(default_factory=dict)

    @property
    def n_channels(self) -> int:
        return self.x.shape[0]

    def calls(self):
        return list(zip(self.cuts[:-1], self.cuts[1:]))


# ------------------------------------------------------------------------------------------ the planner, restated
def replay(p: FmParams, warm: int, stream: bool = False) -> int:
    """fm_replay: the back end's de-emphasis replay in decimated samples."""
    if not p.deemph:
        return 0
    return warm if warm > 0 else (20 if stream else 16) * p.deemph_a + 64


def margin(p: FmParams, warm: int) -> int:
    """fm_margin: PCM a back end needs from before its stretch."""
    return replay(p, warm) + ((p.rate_out // p.rate_out2 + 2) if p.rate_out2 > 0 else 0) + 2


def _spec(p: FmParams) -> int:
    serial = bool(p.deemph) or p.rate_out2 > 0
    plain = not p.squelch_level and not p.dc_block_audio and not p.dc_block_raw and p.post_downsample <= 1
    if not plain:
        return 2
    if p.mode == MODE_FM and p.custom_atan == ATAN_FAST and not p.offset_tuning and serial:
        return 1
    if p.mode == MODE_FM and p.custom_atan == ATAN_LUT and not p.offset_tuning and not serial and p.downsample_passes == 0:
        return 3
    return 0


def rows_geometry(p: FmParams, warm: int):
    """fm_plan_rows: (rows an item's PCM buffer holds, margin rows).  The margin fits when the first is larger."""
    P = p.downsample_passes
    row_pcm = ROW_LEN >> P
    rows_margin = -(-margin(p, warm) // row_pcm)
    xs_words = 256 + 32 * (32 >> P)                      # RowSmem<P>::WORDS
    xs_bytes = ROWS_FE_WARPS * xs_words * 4 + 1008 + ROWS_FE_WARPS * ROWS_STAGES * ROW_BYTES
    dyn_max = min(SMEM_PER_SM // ROWS_MINB - SMEM_RESERVED, SMEM_OPTIN) - SPLIT_STATIC_SMEM

    def cap_for(r):
        e = r * row_pcm + 8 + 16
        return (e + 7) & ~7

    rows_item = ((dyn_max - xs_bytes) // 2 // 2) // (row_pcm + 1)
    while rows_item > rows_margin + 1 and 2 * cap_for(rows_item) * 2 + xs_bytes > dyn_max:
        rows_item -= 1
    return rows_item, rows_margin


def rows_fit(p: FmParams, warm: int) -> bool:
    rows_item, rows_margin = rows_geometry(p, warm)
    return rows_item - rows_margin >= 1


def fused_fit(p: FmParams, warm: int, seg: int = 0) -> bool:
    """fm_plan_segments: whether any segment length gives the fused kernel a PCM buffer and a replay that fit."""
    P = p.downsample_passes
    D = (1 << P) if P else p.downsample
    T = FUSED_T.get(P, 128)
    G = max(1 << P, 8)
    dec_exact = (16 if p.comp_fir_size == 9 else 8) if P else 3
    halo = -(-(dec_exact * D) // G) * G
    direct = not p.deemph and p.rate_out2 <= 0
    m = 0 if direct else margin(p, warm)

    def geometry(sf):
        n_extra = 0 if direct else (m * D + halo + sf - 1) // sf
        cap = 8 if direct else T * (sf // D + 2) + 64
        cap += PCM_PAD_SEG * (cap >> 7) + 8
        return 2 * cap <= SMEM_OPTIN - FUSED_STATIC_SMEM and n_extra <= T // 2

    sf = seg
    if sf <= 0:
        sf = min(128 * D, 2048)
        sf = max(sf, 4 * halo)
        gs = G
        if P == 0:
            l = D // np.gcd(D, 8) * 8
            if l <= 1024:
                gs = l
        if sf >= 2 * gs:
            sf = sf // gs * gs
    sf = -(-sf // G) * G
    if geometry(sf):
        return True
    s = -(-(sf * 8) // G) * G
    while s >= G:
        if geometry(s):
            return True
        if s == G:
            break
        s = -(-(s // 2) // G) * G
    return False


def replay_limits(p: FmParams):
    """The largest de-emphasis replay (rxb200_fm_tune's deemph_warmup) the split kernel holds for p, and the largest
    the fused kernel holds."""
    def largest(fits):
        lo, hi = 1, 1 << 20
        assert fits(lo) and not fits(hi)
        while hi - lo > 1:
            mid = (lo + hi) // 2
            lo, hi = (mid, hi) if fits(mid) else (lo, mid)
        return lo
    return largest(lambda w: rows_fit(p, w)), largest(lambda w: fused_fit(p, w))


def stream_min(p: FmParams, n_ch: int, env: dict, warm: int) -> int:
    if "RXB200_FM_STREAM_MIN" in env:
        return int(env["RXB200_FM_STREAM_MIN"])
    D = (1 << p.downsample_passes) if p.downsample_passes else p.downsample
    return 32 * replay(p, warm) * D // n_ch


def expected_kind(p: FmParams, n_ch: int, n16: int, chunk16: int, env: dict, warm: int) -> int:
    """kernel_kind of one call of n16 int16 per channel: 1 = row kernel, 3 = stream path, 0 = fused kernel.  A row shape
    whose margin does not fit the split kernel runs on the fused kernel; -1 when neither kernel fits it."""
    n = n16 // 2
    spec = _spec(p)
    P = p.downsample_passes
    if spec == 1 and 1 <= P <= 3 and (chunk16 // 2) % ROW_LEN == 0 and n % ROW_LEN == 0 and n >= 16 * ROW_LEN \
            and rows_fit(p, warm):
        return 1
    if spec == 1 and P == 0 and p.deemph and n >= stream_min(p, n_ch, env, warm):
        return 3
    return 0 if fused_fit(p, warm) else -1


# ------------------------------------------------------------------------------------------ inputs
def channel_input(rng, kind: str, n: int, silent_stretch: bool) -> np.ndarray:
    """int16[2 n]: an FM signal (loud or quiet), full-scale noise, or the droop FIR's Nyquist overshoot tone (a
    full-scale tone at -3/16 of the capture rate, the largest products the row discriminator sees) followed by
    signal; optionally a silent stretch (de-emphasis brackets that never close)."""
    t = np.arange(n)
    if kind == "noise":
        x = rng.integers(-32768, 32768, size=2 * n).astype(np.int16)
    elif kind == "overshoot":
        ph = 2.0 * np.pi * (-3.0 / 16.0) * t
        ph[n // 2:] = 2 * np.pi * 0.03 * t[n // 2:] + 2.0 * np.sin(2 * np.pi * 0.0011 * t[n // 2:])
        x = np.empty(2 * n, dtype=np.int16)
        x[0::2] = np.clip(np.round(32767 * np.cos(ph)), -32768, 32767)
        x[1::2] = np.clip(np.round(32767 * np.sin(ph)), -32768, 32767)
    else:
        amp = 300.0 if kind == "quiet" else float(rng.choice([8000.0, 20000.0, 32767.0]))
        f0 = float(rng.uniform(-0.2, 0.2))
        ph = 2 * np.pi * f0 * t + float(rng.uniform(0.5, 6.0)) * np.sin(2 * np.pi * float(rng.uniform(1e-4, 2e-3)) * t)
        nz = max(1, int(amp / 100))
        x = np.empty(2 * n, dtype=np.int32)
        x[0::2] = np.rint(amp * np.cos(ph)) + rng.integers(-nz, nz + 1, size=n)
        x[1::2] = np.rint(amp * np.sin(ph)) + rng.integers(-nz, nz + 1, size=n)
        x = np.clip(x, -32768, 32767).astype(np.int16)
    if silent_stretch:
        a, b = sorted(int(v) for v in rng.integers(0, n, size=2))
        x[2 * a:2 * b] = 0
    return x


def _inputs(rng, n_ch: int, n: int):
    kinds = [str(rng.choice(INPUTS)) for _ in range(n_ch)]
    xs = [channel_input(rng, k, n, bool(rng.random() < 0.3)) for k in kinds]
    if n_ch > 1:                                         # one channel silent
        s = int(rng.integers(0, n_ch))
        xs[s][:] = 0
        kinds[s] = "silent"
    return np.stack(xs), kinds


def _cuts(rng, n_chunks: int, chunk16: int, n16: int, max_calls: int = 4):
    inner = sorted(set(int(c) for c in rng.integers(1, n_chunks, size=int(rng.integers(0, max_calls)))) if n_chunks > 1 else [])
    return [0] + [c * chunk16 for c in inner] + [n16]


# ------------------------------------------------------------------------------------------ families
def rows_draw(seed: int) -> Draw:
    """The wbfm shape with 1..3 fifth_order passes on whole rows."""
    rng = np.random.default_rng(10_000 + seed)
    P = int(rng.integers(1, 4))
    fir = int(rng.choice([0, 9]))
    serial = SERIAL[seed % 3] if seed < 18 else str(rng.choice(SERIAL))
    if seed < 18:                                        # the first 18 draws walk P x FIR x serial stage
        P, fir = 1 + (seed // 6) % 3, (0, 9)[(seed // 3) % 2]
    a = int(rng.choice(ROWS_A))
    if seed % 20 == 19:                                  # a replay longer than the split kernel's P = 1 margin holds
        P, serial, a = 1, str(rng.choice(["deemph", "both"])), int(rng.choice([541, 601]))
    rate_out = RATE_OUT[P]
    p = FmParams(downsample=1 << P, downsample_passes=P, comp_fir_size=fir, custom_atan=ATAN_FAST, rate_out=rate_out)
    if serial in ("deemph", "both"):
        p.deemph, p.deemph_a = 1, a
    r2 = None
    if serial in ("resample", "both"):
        r2 = list(RATE_OUT2)[int(rng.integers(0, len(RATE_OUT2)))]
        p.rate_out2 = RATE_OUT2[r2](rate_out)
    chunk_rows = int(rng.choice(ROWS_CHUNK_ROWS))
    n_ch = int(rng.integers(1, 6))
    rows = int(rng.integers(16, max(17, min(400, 900 // n_ch))))
    if rows % chunk_rows == 0 and chunk_rows > 1:        # ragged last chunk
        rows += int(rng.integers(1, chunk_rows))
    seg = 0 if rng.random() < 0.3 else int(rng.integers(1, 21)) * ROW_LEN + int(rng.choice([0, 0, 1, 300, 777]))
    warm = int(rng.choice([0, 1, 7, a, 4 * a])) if p.deemph and seed % 20 != 19 else 0
    chunk16 = chunk_rows * ROW_I16
    n16 = rows * ROW_I16
    cuts = _cuts(rng, -(-rows // chunk_rows), chunk16, n16)
    x, kinds = _inputs(rng, n_ch, rows * ROW_LEN)
    env: dict = {}
    exp = [expected_kind(p, n_ch, b - a_, chunk16, env, warm) for a_, b in zip(cuts[:-1], cuts[1:])]
    rows_item, rows_margin = rows_geometry(p, warm)
    own = min(max(seg // ROW_LEN, 1), rows_item - rows_margin) if seg else 0
    tags = dict(P=P, fir=fir, serial=serial, a=a if p.deemph else None, rate_out2=r2, chunk_rows=chunk_rows,
                margin_fits=rows_item - rows_margin >= 1,
                rows=rows, n_ch=n_ch, seg_rows=seg // ROW_LEN if seg else 0, seg_ragged=bool(seg % ROW_LEN),
                warm=warm, warm_is=("0" if warm == 0 else "1" if warm == 1 else "7" if warm == 7 else
                                    "a" if warm == a else "4a"),
                inputs=kinds, margin_items=(-(-rows_margin // own) if own > 0 else 0),
                ratio=(p.rate_out // p.rate_out2 if p.rate_out2 > 0 else 0))
    return Draw("rows", seed, p, chunk16, cuts, x, exp, expected_kind(p, n_ch, n16, chunk16, env, warm),
                env, (seg, warm), tags)


def stream_draw(seed: int) -> Draw:
    """The undecimated wbfm shape with de-emphasis: front kernel + back kernel on calls of at least STREAM_MIN."""
    rng = np.random.default_rng(20_000 + seed)
    a = int(rng.integers(1, 401))
    if seed < 2:
        a = (2, 1)[seed]
    rate_out = int(rng.choice([2_400_000, 1_024_000, 240_000]))
    p = FmParams(downsample=1, custom_atan=ATAN_FAST, deemph=1, deemph_a=a, rate_out=rate_out)
    r = seed % 3
    if r == 1:
        p.rate_out2 = int(rng.choice([rate_out, rate_out - 1]))
    elif r == 2:
        p.rate_out2 = int(rng.choice([48_000, 44_100, rate_out // 5, rate_out // 50]))
    chunk16 = 16 * int(np.exp(rng.uniform(0.0, np.log(16384))))
    n_ch = int(rng.integers(1, 4))
    n16 = 16 * int(rng.integers(6_000, 6_000 + 24_000 // n_ch))
    n_chunks = -(-n16 // chunk16)
    cuts = _cuts(rng, n_chunks, chunk16, n16, max_calls=5)
    sizes = sorted({(b - a_) // 2 for a_, b in zip(cuts[:-1], cuts[1:])})
    # STREAM_MIN between two call sizes when there are several, so that the calls of one stream switch paths
    smin = int(rng.integers(sizes[0] + 1, sizes[-1] + 1)) if len(sizes) > 1 and rng.random() < 0.8 else \
        int(rng.choice([1, sizes[0] + 1]))
    env = {"RXB200_FM_STREAM_MIN": str(smin),
           "RXB200_FM_STREAM_PIECE": str(int(rng.choice([0, 64, int(rng.integers(64, 3001))]))),
           "RXB200_FM_STREAM_WIN": str(int(rng.choice([128, 256]))),
           "RXB200_FM_STREAM_T": str(int(rng.choice([32, 64, 128])))}
    x, kinds = _inputs(rng, n_ch, n16 // 2)
    exp = [expected_kind(p, n_ch, b - a_, chunk16, env, 0) for a_, b in zip(cuts[:-1], cuts[1:])]
    tags = dict(a=a, rate_out2=p.rate_out2, resample=("off", "ratio1", "ratio")[r], n_ch=n_ch, chunk16=chunk16,
                piece=int(env["RXB200_FM_STREAM_PIECE"]), win=int(env["RXB200_FM_STREAM_WIN"]),
                t=int(env["RXB200_FM_STREAM_T"]), inputs=kinds)
    return Draw("stream", seed, p, chunk16, cuts, x, exp, expected_kind(p, n_ch, n16, chunk16, env, 0), env, (0, 0), tags)


def fused_draw(seed: int) -> Draw:
    """The fused kernel's specialisations: SPEC 3 (FM through the LUT, no serial stage, boxcar), and the wbfm SPEC 1
    kernel at P = 0 with a boxcar D > 1 and at P = 4."""
    rng = np.random.default_rng(30_000 + seed)
    shape = ("spec3", "spec1_boxcar", "spec1_p4")[seed % 3]
    env: dict = {}
    if shape == "spec3":
        D = int(rng.integers(1, 301))
        p = FmParams(downsample=D, custom_atan=ATAN_LUT, rate_out=int(rng.choice([24_000, 48_000, 240_000])))
        n_ch = int(rng.integers(1, 9))
    else:
        P = 0 if shape == "spec1_boxcar" else 4
        D = int(rng.integers(2, 65)) if P == 0 else 16
        rate_out = int(rng.choice([170_000, 150_000, 75_000]))
        p = FmParams(downsample=D, downsample_passes=P, comp_fir_size=int(rng.choice([0, 9])) if P else 0,
                     custom_atan=ATAN_FAST, rate_out=rate_out)
        if rng.random() < 0.7:
            p.deemph, p.deemph_a = 1, int(rng.choice([1, 2, 13, 23, 90]))
        if not p.deemph or rng.random() < 0.6:
            p.rate_out2 = int(rng.choice([rate_out, 48_000, 32_000, 8_000]))
        if P == 0 and p.deemph:
            env["RXB200_FM_STREAM_MIN"] = str(1 << 40)   # keep the boxcar shape on the fused kernel
        n_ch = int(rng.integers(1, 5))
    G = max(16, 2 << p.downsample_passes)            # int16 granularity of a chunk
    n16 = G * int(rng.integers(40_000 // G, 40_000 // G + 200_000 // (n_ch * G)))
    chunk16 = G * int(rng.integers((16 * D) // G + 1, min(262144, n16) // G + 1))
    cuts = _cuts(rng, -(-n16 // chunk16), chunk16, n16)
    x, kinds = _inputs(rng, n_ch, n16 // 2)
    exp = [expected_kind(p, n_ch, b - a_, chunk16, env, 0) for a_, b in zip(cuts[:-1], cuts[1:])]
    tags = dict(shape=shape, D=D, P=p.downsample_passes, n_ch=n_ch, inputs=kinds)
    return Draw("fused", seed, p, chunk16, cuts, x, exp, expected_kind(p, n_ch, n16, chunk16, env, 0), env, (0, 0), tags)


N_DRAWS = {"rows": 200, "stream": 100, "fused": 60}
FAMILIES = {"rows": rows_draw, "stream": stream_draw, "fused": fused_draw}


def draw(family: str, seed: int) -> Draw:
    return FAMILIES[family](seed)


def all_ids():
    return [(f, s) for f, n in N_DRAWS.items() for s in range(n)]


# ------------------------------------------------------------------------------------------ named edge cases
def _cli(rate_s, rate_r, tc_us, use_F=1):
    """The parameters the reference's main() + optimal_settings() derive for `-M wbfm -s rate_s [-F 9] [-r rate_r]
    -c tc_us` (checked against the reference by tests/golden/make_fm_paths_golden.py)."""
    D = 1_000_000 // rate_s + 1
    P = int(np.log2(D)) + 1 if use_F else 0
    a = int(round(1.0 / (1.0 - np.exp(-1.0 / (rate_s * tc_us * 1e-6)))))
    return FmParams(downsample=(1 << P) if P else D, downsample_passes=P, comp_fir_size=9 if use_F else 0,
                    custom_atan=ATAN_FAST, deemph=1, deemph_a=a, rate_out=rate_s, rate_out2=rate_r)


def golden_cases():
    """name -> (params, chunk int16, input int16[n]): the edges the golden file pins to the reference's bytes."""
    def wb(seed, rows):
        return channel_input(np.random.default_rng(seed), "loud", rows * ROW_LEN, False)

    def p_rows(P, **kw):
        return FmParams(downsample=1 << P, downsample_passes=P, comp_fir_size=9, custom_atan=ATAN_FAST,
                        rate_out=RATE_OUT[P], **kw)

    cs = {
        "cli_s300k_F9_r48k_c2000": (_cli(300_000, 48_000, 2000), 64 * ROW_I16, wb(1, 160)),
        "cli_s1200k_F9_r48k_c450": (_cli(1_200_000, 48_000, 450), 64 * ROW_I16, wb(2, 160)),
        "cli_s1200k_F9_c500": (_cli(1_200_000, 32_000, 500), 128 * ROW_I16, wb(3, 200)),
        "one_row_chunks_P3": (p_rows(3, deemph=1, deemph_a=23, rate_out2=48_000), ROW_I16, wb(4, 40)),
        "deemph_only_P1": (p_rows(1, deemph=1, deemph_a=91), 7 * ROW_I16, wb(5, 50)),
        "deemph_only_P2": (p_rows(2, deemph=1, deemph_a=46), 5 * ROW_I16, wb(6, 50)),
        "deemph_only_P3": (p_rows(3, deemph=1, deemph_a=23), 3 * ROW_I16, wb(7, 50)),
        "ratio1_P2": (p_rows(2, deemph=1, deemph_a=46, rate_out2=600_000 - 1), 32 * ROW_I16, wb(8, 70)),
        "a1_P3": (p_rows(3, deemph=1, deemph_a=1, rate_out2=48_000), 2 * ROW_I16, wb(9, 33)),
        "a2_P1": (p_rows(1, deemph=1, deemph_a=2, rate_out2=44_100), 5 * ROW_I16, wb(10, 41)),
        "overshoot_P3_a601": (p_rows(3, deemph=1, deemph_a=601, rate_out2=48_000), 32 * ROW_I16,
                              channel_input(np.random.default_rng(11), "overshoot", 100 * ROW_LEN, False)),
        "stream_D1_a2_even": (FmParams(downsample=1, custom_atan=ATAN_FAST, deemph=1, deemph_a=2, rate_out=2_400_000,
                                       rate_out2=48_000), 4096, wb(12, 60)),
    }
    # full-scale noise whose decimated samples once make fast_atan2's 4096 (|x| - |y|) leave int32 (the channel of rows
    # draw 76 that showed it): the row front end must wrap as the reference does
    d = rows_draw(76)
    cs["fullscale_noise_atan_wrap_P3"] = (d.params, d.chunk, d.x[4].copy())
    return cs
