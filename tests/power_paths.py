"""Seeded draws for the rx_power accumulate paths: every kernel ``rxb200_power_accumulate_device``
(csrc/power_kernels.cu) chooses among, on both sides of each boundary of that choice.

A draw is everything one parity check needs: the plan, the window table and optionally a caller's sine table, the hop
buffers (``n_pass x hops x buf_len``), the call splits (pass and hop sub-ranges, run one after the other on one
handle), the environment knobs read at create, and the path every call must report through
``rxb200_power_last_path``.  ``expected_path`` restates the launch rule, so a change of that rule shows up as a failing
test instead of a silently different path.  No fixtures: the GPU sweep, the CPU coverage test and the reference pin
import the same families.

Families:
* ``cli``: seeded rx_power command lines (span, bin size, crop, boxcar / -F 0 / -F 9, -P, window, passes) planned by
  ``rxb200_power_plan_range``.  Draws the planner refuses, with more than 10 passes, or over a size cap are kept as
  dropped draws (``Draw.dropped``) so that the coverage test can count them.
* ``geometry``: explicit plans at the edges the planner only brushes: every FFT size at ``buf_len`` 16384 under each
  knob, every ``NB`` of the generic kernel with boxcar and -F decimation, both sides of the shared-memory limit and of
  the ``tables_in_smem`` flip, partial boxcar slots and partial last N-blocks.
* ``launch``: slice choice and atomics: many passes on one hop, many hops, the ``rxb200_power_shard`` ranges of 871
  hops run as hop sub-ranges, back-to-back device calls without a sync.
* ``tables``: caller sine tables that keep or break the fast path's trivial first-trip twiddles, random int16 sine
  tables, and int32 window tables beyond int16.

Only the ``cli`` draws are planner shapes, and only those are pinned to the unmodified reference (the reference has no
entry point for a plan, a sine table or a call split of its own); every other draw compares with the port alone.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Optional

import numpy as np

import oracle
from rx_tools_b200 import power

SMEM_LIMIT = 227 * 1024             # the shared memory every rx_power kernel may opt in to (power_kernels.cu)
N_SM = 132                          # H100 SXM; the GPU test passes the device's own count
WINDOWS = list(power.WINDOWS)
INPUTS = ("noise", "tones", "dc", "zeros", "rail")
SIZE_CAP = 1 << 22                  # int16 per cli draw (n_pass x hops x buf_len)
NB_LADDER = (1, 2, 4, 8, 16, 0)


@dataclass
class Draw:
    family: str
    seed: int
    plan: Optional[power.Plan]
    window: Optional[np.ndarray] = None      # int32[N]
    sine: Optional[np.ndarray] = None        # int16[3N/4], None: the library's own table
    x: Optional[np.ndarray] = None           # int16[n_pass][n_hops][buf_len]
    calls: list = field(default_factory=list)  # (pass_lo, pass_hi, hop_lo, hop_hi), run in order, cover x once
    env: dict = field(default_factory=dict)
    paths: list = field(default_factory=list)  # expected last_path() after every call
    device: bool = False                     # scanner_device(sync=False) calls from one device buffer
    tags: dict = field(default_factory=dict)
    dropped: Optional[str] = None
    cli: Optional[dict] = None               # the command line of a cli draw

    @property
    def n_pass(self) -> int:
        return self.x.shape[0]


# ------------------------------------------------------------------------------------------ the launch rule, restated
def fft8_threads(bin_e: int, env: dict) -> int:
    force = int(env.get("RXB200_POWER_THREADS", "0") or 0)
    if force in (512, 1024):
        return force if bin_e <= 12 else 1024
    return 512 if bin_e <= 12 else 1024


def generic_nb(bin_e: int) -> int:
    nb = (1 << bin_e) // 256
    return 1 if nb <= 1 else (nb if nb <= 16 else 0)


def smem_generic(buf_len: int, bin_e: int) -> int:
    n = 1 << bin_e
    return 16 + 256 + 2 * buf_len + 2 * ((n * 3 // 4 + 7) & ~7) + 2 * n


def is_big(plan) -> bool:
    return plan.bin_e > 0 and 16 + 256 + 2 * plan.buf_len > SMEM_LIMIT


def fast_slices(n_pass: int, nh: int, threads: int, n_sm: int) -> int:
    slots = n_sm * (1024 // threads)
    sl, best = 1, -1
    c = 1
    while c <= n_pass and c <= 2 * slots:
        rounds = (nh * c + slots - 1) // slots
        t = rounds * ((n_pass + c - 1) // c + 1) * 4096 + c
        if best < 0 or t < best:
            best, sl = t, c
        c += 1
    return sl


def expected_path(plan, env: dict, n_pass: int, nh: int, n_sm: int = N_SM) -> dict:
    """rxb200_power_last_path after one call of n_pass passes over nh hops."""
    e = plan.bin_e
    slices = max(1, min(n_pass, (n_sm * 4 + nh - 1) // nh))
    if e == 0:
        return dict(kernel="rms", bin_e=0, threads=256, nb=-1, tables_in_smem=0, slices=slices, launches=1)
    if is_big(plan):
        decim = not plan.boxcar and plan.downsample > 1 and plan.downsample_passes > 0
        return dict(kernel="big_decim" if decim else "big_load", bin_e=e, threads=256, nb=-1, tables_in_smem=0,
                    slices=0, launches=n_pass * nh * (3 + e))
    if plan.downsample == 1 and plan.buf_len == 16384 and 3 <= e <= 13 and "RXB200_POWER_V1" not in env:
        t = fft8_threads(e, env)
        return dict(kernel="fft8", bin_e=e, threads=t, nb=-1, tables_in_smem=1, slices=fast_slices(n_pass, nh, t, n_sm),
                    launches=1)
    return dict(kernel="generic", bin_e=e, threads=256, nb=generic_nb(e),
                tables_in_smem=int(smem_generic(plan.buf_len, e) <= SMEM_LIMIT), slices=slices, launches=1)


def valid(plan) -> Optional[str]:
    """power_validate: None when rxb200_power_create accepts the plan, else why not."""
    if plan.buf_len < 16 or plan.buf_len % 8:
        return "buf_len"
    if plan.bin_e == 0:
        return None
    ds, n2 = plan.downsample, 2 << plan.bin_e
    if n2 * ds > plan.buf_len:
        return "2N x downsample > buf_len"
    if is_big(plan) and ds > 1 and not plan.boxcar and (plan.downsample_passes < 1 or ds != 1 << plan.downsample_passes
                                                        or plan.buf_len % (n2 * ds)):
        return "big -F geometry"
    used = plan.buf_len // ds
    if -(-used // n2) * n2 > plan.buf_len:
        return "last block past the hop buffer"
    return None


def triv(sine: Optional[np.ndarray], bin_e: int) -> int:
    """PowArgs::triv: W^0 and W^(N/4) have a zero component, so the fast path's first trip uses two products."""
    n = 1 << bin_e
    s = power.sine_table(bin_e) if sine is None else sine
    return int(n >= 8 and s[0] == 0 and s[n // 2] in (0, 1))


def oracle_params(plan) -> oracle.PowerParams:
    return oracle.PowerParams(bin_e=plan.bin_e, buf_len=plan.buf_len, downsample=plan.downsample,
                              downsample_passes=plan.downsample_passes, comp_fir_size=plan.comp_fir_size,
                              boxcar=plan.boxcar, peak_hold=plan.peak_hold)


def mkplan(bin_e, buf_len, ds=1, passes=0, fir=0, boxcar=1, peak=0, n_hops=1) -> power.Plan:
    return power.Plan(n_hops=n_hops, bin_e=bin_e, buf_len=buf_len, downsample=ds, downsample_passes=passes,
                      comp_fir_size=fir, boxcar=boxcar, peak_hold=peak, rate=2_000_000, crop=0.0,
                      first_freq=100_000_000, freq_step=2_000_000, bin_size_hz=0.0)


# ------------------------------------------------------------------------------------------ inputs
def hop_input(rng, kind: str, shape, silent: bool) -> np.ndarray:
    """int16[shape]: full-scale noise (every int16 wrap of the window multiply, butterflies, boxcar sums and half-band
    passes), tones plus noise, a large DC offset (remove_dc's int16 mean), all zeros, or constant rails; optionally a
    silent stretch inside every hop buffer."""
    n_pass, n_hops, buf_len = shape
    if kind == "noise":
        x = rng.integers(-32768, 32768, size=shape, dtype=np.int32)
    elif kind == "tones":
        t = np.arange(buf_len // 2)
        f = rng.uniform(-0.5, 0.5, size=2)
        z = 9000 * np.exp(2j * np.pi * f[0] * t) + 300 * np.exp(2j * np.pi * f[1] * t)
        x = np.empty(shape, dtype=np.int32)
        x[..., 0::2] = np.rint(z.real)
        x[..., 1::2] = np.rint(z.imag)
        x += rng.integers(-200, 201, size=shape, dtype=np.int32)
    elif kind == "dc":
        off = rng.integers(-30000, 30001, size=2)
        x = rng.integers(-2000, 2001, size=shape, dtype=np.int32)
        x[..., 0::2] += off[0]
        x[..., 1::2] += off[1]
    elif kind == "zeros":
        x = np.zeros(shape, dtype=np.int32)
    else:                                                    # rails: runs of +32767 / -32768 / -32767
        x = np.empty(shape, dtype=np.int32)
        flat = x.reshape(-1)
        pos = 0
        while pos < flat.size:
            run = int(rng.integers(1, 4 * buf_len))
            flat[pos:pos + run] = int(rng.choice([32767, -32768, -32767]))
            pos += run
    x = np.clip(x, -32768, 32767).astype(np.int16)
    if silent:
        a, b = sorted(int(v) for v in rng.integers(0, buf_len, size=2))
        x[..., a:b] = 0
    return x


def _input(rng, shape, kind=None):
    kind = kind or str(rng.choice(INPUTS))
    silent = bool(rng.random() < 0.25)
    return hop_input(rng, kind, shape, silent), kind, silent


def _finish(d: Draw, rng, splits: str = "auto") -> Draw:
    """Fill in the calls (whole, or split by passes and hops) and the path every call must report."""
    n_pass, n_hops = d.x.shape[0], d.x.shape[1]
    if not d.calls:
        mode = splits if splits != "auto" else str(rng.choice(["whole", "whole", "passes", "hops", "both"]))
        pc = [0, n_pass] if mode in ("whole", "hops") or n_pass == 1 else \
            [0] + sorted(set(int(v) for v in rng.integers(1, n_pass, size=2))) + [n_pass]
        hc = [0, n_hops] if mode in ("whole", "passes") or n_hops == 1 else \
            [0] + sorted(set(int(v) for v in rng.integers(1, n_hops, size=2))) + [n_hops]
        d.calls = [(p0, p1, h0, h1) for p0, p1 in zip(pc[:-1], pc[1:]) for h0, h1 in zip(hc[:-1], hc[1:])]
        d.tags["split"] = mode
    d.paths = [expected_path(d.plan, d.env, p1 - p0, h1 - h0) for p0, p1, h0, h1 in d.calls]
    d.tags.update(kernel=d.paths[-1]["kernel"], bin_e=d.plan.bin_e, ds=d.plan.downsample,
                  boxcar=int(d.plan.boxcar and d.plan.downsample > 1),
                  F=int(not d.plan.boxcar and d.plan.downsample > 1 and d.plan.downsample_passes > 0),
                  fir=int(d.plan.comp_fir_size == 9 and d.plan.downsample_passes > 0),
                  peak=d.plan.peak_hold, triv=triv(d.sine, d.plan.bin_e) if d.plan.bin_e else None,
                  slices={p["slices"] for p in d.paths}, paths={_key(p) for p in d.paths})
    assert valid(d.plan) is None, (d.family, d.seed, valid(d.plan))
    return d


def _key(p: dict):
    """The path row a call reached: kernel, then E and T, NB and the table placement."""
    if p["kernel"] == "fft8":
        return ("fft8", p["bin_e"], p["threads"])
    if p["kernel"] == "generic":
        return ("generic", p["nb"], p["tables_in_smem"])
    return (p["kernel"],)


def _window(rng, n: int, name: Optional[str] = None) -> tuple:
    name = name or str(rng.choice(WINDOWS))
    if n == 1:                                               # rms_power uses no window
        return np.ones(1, dtype=np.int32), name
    return power.window_table(name, n), name


# ------------------------------------------------------------------------------------------ families
def cli_draw(seed: int) -> Draw:
    rng = np.random.default_rng(40_000 + seed)
    span = int(np.exp(rng.uniform(np.log(2e3), np.log(5e6))))
    bin_hz = int(np.exp(rng.uniform(0.0, np.log(1e5))))
    crop = float(rng.choice([0.0, 0.1, 0.285, 0.5]))
    mode = ("boxcar", "F0", "F9")[seed % 3]
    peak = int(rng.random() < 0.3)
    win = WINDOWS[seed % len(WINDOWS)]
    n_pass = int(rng.integers(1, 5))
    lo = int(rng.integers(24, 1700)) * 1_000_000
    cli = dict(freq=f"{lo}:{lo + span}:{bin_hz}", crop=crop, boxcar=int(mode == "boxcar"),
               fir=9 if mode == "F9" else 0, peak=peak, window=win, n_pass=n_pass)
    d = Draw("cli", seed, None, cli=cli, tags=dict(mode=mode, window=win, crop=crop))
    try:
        plan = power.plan_range(cli["freq"], crop, cli["boxcar"], cli["fir"], peak)
    except power._lib.Rxb200Error as e:
        d.dropped = f"planner: {e}"
        return d
    d.plan = plan
    if plan.downsample_passes > 10:
        d.dropped = "more than 10 passes"
    elif n_pass * plan.n_hops * plan.buf_len > SIZE_CAP:
        d.dropped = "size cap"
    elif valid(plan) is not None:
        d.dropped = "refused: " + valid(plan)
    if d.dropped:
        return d
    d.window, _ = _window(rng, 1 << plan.bin_e, win)
    d.x, kind, silent = _input(rng, (n_pass, plan.n_hops, plan.buf_len))
    d.tags.update(input=kind, silent=silent)
    return _finish(d, rng)


def _geometry_plans():
    """(plan, env, tags) of every geometry draw, in a fixed order."""
    out = []
    knobs = (("default", {}), ("T1024", {"RXB200_POWER_THREADS": "1024"}), ("V1", {"RXB200_POWER_V1": "1"}))
    for name, env in knobs:
        for e in range(1, 14):
            out.append((mkplan(e, 16384, n_hops=3), env, dict(knob=name, what="fft_size")))
    out.append((mkplan(13, 16384, n_hops=2), {"RXB200_POWER_THREADS": "512"}, dict(knob="T512", what="fft_size")))
    out.append((mkplan(0, 16384, n_hops=3), {}, dict(what="rms")))
    out.append((mkplan(0, 16, n_hops=1), {}, dict(what="rms")))
    # every NB with boxcar and with -F (P 1..6 as far as the buffer fits shared memory, FIR 0 and 9)
    for i, e in enumerate((3, 8, 9, 10, 11, 12, 13, 14)):
        n2 = 2 << e
        for j, ds in enumerate((3, 7) if e < 13 else (2,)):
            k = max(1, 16384 // (n2 * ds))
            out.append((mkplan(e, n2 * ds * k + 8 * j, ds=ds, n_hops=2), {}, dict(what="nb_boxcar")))
        pmax = max(p for p in range(1, 7) if n2 << p <= 116088) if n2 * 2 <= 116088 else 0
        for fir in (0, 9):
            if pmax:
                P = 1 + (i + fir) % pmax
                out.append((mkplan(e, n2 << P, ds=1 << P, passes=P, fir=fir, boxcar=0, n_hops=2), {},
                            dict(what="nb_F")))
    for P in range(1, 7):                                      # every P at one NB
        for fir in (0, 9):
            out.append((mkplan(5, 64 << P, ds=1 << P, passes=P, fir=fir, boxcar=0, n_hops=2), {}, dict(what="F_P")))
    # the shared-memory limit: the largest valid buf_len on the shared-memory path and the next valid one up
    for e, ds, P, box in ((3, 1, 0, 1), (8, 1, 0, 1), (12, 1, 0, 1), (13, 1, 0, 1), (10, 5, 0, 1), (10, 4, 2, 0),
                          (7, 16, 4, 0)):
        step = int(np.lcm(8, (2 << e) * ds)) if not box or ds == 1 else 8
        below = (116088 // step) * step
        while valid(mkplan(e, below, ds=ds, passes=P, boxcar=box)) is not None:
            below -= step
        above = below + step
        while valid(mkplan(e, above, ds=ds, passes=P, boxcar=box)) is not None:
            above += step
        for b, side in ((below, "below"), (above, "above")):
            out.append((mkplan(e, b, ds=ds, passes=P, fir=9 if P else 0, boxcar=box), {},
                        dict(what="smem_limit", side=side)))
    # the tables_in_smem flip at N 8192 and 16384
    for e in (13, 14):
        n2 = 2 << e
        below = max(b for b in range(n2, 116089, n2) if smem_generic(b, e) <= SMEM_LIMIT)
        for b, side in ((below, "in"), (below + n2, "out")):
            out.append((mkplan(e, b, n_hops=1), {}, dict(what="tables_flip", side=side)))
    # boxcar slots that do not divide buf_len/2 and a partial last N-block
    for e, ds, buf in ((4, 3, 16384), (6, 9, 16384), (9, 5, 12288), (2, 1400, 16384), (7, 311, 80000), (11, 3, 24576),
                       (1, 7, 40)):
        out.append((mkplan(e, buf, ds=ds, n_hops=2), {}, dict(what="partial")))
    return out


GEOMETRY = _geometry_plans()


def geometry_draw(seed: int) -> Draw:
    rng = np.random.default_rng(50_000 + seed)
    plan, env, tags = GEOMETRY[seed]
    plan = mkplan(plan.bin_e, plan.buf_len, plan.downsample, plan.downsample_passes, plan.comp_fir_size, plan.boxcar,
                  int(seed % 4 == 3 or plan.buf_len == 16), plan.n_hops)
    d = Draw("geometry", seed, plan, env=dict(env), tags=dict(tags))
    d.window, d.tags["window"] = _window(rng, 1 << plan.bin_e)
    n_pass = int(rng.integers(1, 4))
    d.x, d.tags["input"], d.tags["silent"] = _input(rng, (n_pass, plan.n_hops, plan.buf_len),
                                                    "noise" if seed % 2 == 0 else None)
    used = plan.buf_len // plan.downsample
    d.tags.update(partial_slot=int(plan.boxcar and plan.downsample > 1 and (plan.buf_len // 2) % plan.downsample != 0),
                  partial_block=int(used % (2 << plan.bin_e) != 0))
    return _finish(d, rng)


SHARD_RANKS = (2, 3, 4, 5, 6, 7, 8)


def launch_draw(seed: int) -> Draw:
    rng = np.random.default_rng(60_000 + seed)
    d = Draw("launch", seed, None)
    if seed < 2:                                              # one hop, 700 passes: slices and atomics
        plan = mkplan(10 if seed == 0 else 6, 16384 if seed == 0 else 4096, peak=seed)
        shape = (700, 1)
        d.tags["what"] = "700_passes"
    elif seed < 12:                                           # 2-3 hops x 1-9 passes
        e = int(rng.choice([4, 7, 9, 12, 13]))
        plan = mkplan(e, 16384 if seed % 2 else (2 << e) * 2, n_hops=int(rng.integers(2, 4)), peak=int(seed % 5 == 0))
        shape = (int(rng.integers(1, 10)), plan.n_hops)
        d.tags["what"] = "few_hops"
    elif seed < 18:                                           # many hops on the fast and the generic kernel
        nh = (131, 264, 600)[(seed - 12) % 3]
        plan = mkplan(10, 16384, n_hops=nh) if seed < 15 else mkplan(8, 1024, n_hops=nh, peak=int(seed == 17))
        shape = (int(rng.integers(1, 3)), nh)
        d.tags["what"] = "many_hops"
    elif seed < 25:                                           # power4's 871 hops, one rank's range per call
        ranks = SHARD_RANKS[seed - 18]
        plan = mkplan(12, 16384, n_hops=871)
        shape = (1, 871)
        d.calls = [(0, 1) + power.shard(871, ranks, r) for r in range(ranks)]
        d.calls = [c for c in d.calls if c[3] > c[2]]
        d.tags.update(what="shard", ranks=ranks, split="shard")
    else:                                                     # back-to-back device calls without a sync
        e = (10, 13, 9, 3, 0)[seed - 25]
        plan = mkplan(e, 16384 if e != 9 else 8192, n_hops=4, peak=int(seed == 27))
        shape = (3, 4)
        d.device = True
        d.tags["what"] = "device"
    d.plan = plan
    d.window, d.tags["window"] = _window(rng, 1 << plan.bin_e)
    d.x, d.tags["input"], d.tags["silent"] = _input(rng, shape + (plan.buf_len,), "noise" if seed < 2 else None)
    return _finish(d, rng, "both" if d.device else "auto")


def tables_draw(seed: int) -> Draw:
    rng = np.random.default_rng(70_000 + seed)
    kind = ("half1", "sine0", "half2", "random", "window")[seed % 5]
    e = (3, 5, 8, 10, 12, 13, 4, 11)[seed % 8] if seed < 16 else int(rng.integers(3, 14))
    generic = seed % 2 == 1 and kind != "window"
    plan = mkplan(e, 16384 if not generic else (2 << e) * 2 if e < 13 else 32768, n_hops=2, peak=int(seed % 7 == 3))
    d = Draw("tables", seed, plan, tags=dict(table=kind))
    n = 1 << e
    s = power.sine_table(e).copy()
    if kind == "half1":                                       # keeps triv: W^(N/4)'s real part 1 >> 1 == 0
        s[n // 2] = 1
    elif kind == "sine0":                                     # W^0 with an imaginary part
        s[0] = int(rng.choice([1, -1, 2, -32768, 32767]))
    elif kind == "half2":
        s[n // 2] = 2
    elif kind == "random":                                    # every twiddle arbitrary, -32768 included
        s = rng.integers(-32768, 32768, size=s.size, dtype=np.int32).astype(np.int16)
        s[rng.integers(0, s.size, size=3)] = -32768
        if seed % 3 == 0:
            s[0], s[n // 2] = 0, int(rng.integers(0, 2))
    d.sine = s if kind != "window" else None
    if kind == "window":                                      # int32 coefficients: only w mod 2^16 reaches the kernel
        w = rng.integers(-65535, 65537, size=n, dtype=np.int64)
        w[rng.integers(0, n, size=max(1, n // 8))] = rng.choice([65536, 65537, 1 << 20, (1 << 20) + 3, -(1 << 18) - 1])
        d.window = w.astype(np.int32)
        d.tags["window"] = "int32"
    else:
        d.window, d.tags["window"] = _window(rng, n)
    d.x, d.tags["input"], d.tags["silent"] = _input(rng, (int(rng.integers(1, 4)), 2, plan.buf_len),
                                                    "noise" if seed % 2 == 0 else None)
    return _finish(d, rng)


N_DRAWS = {"cli": 150, "geometry": len(GEOMETRY), "launch": 30, "tables": 20}
FAMILIES = {"cli": cli_draw, "geometry": geometry_draw, "launch": launch_draw, "tables": tables_draw}


def draw(family: str, seed: int) -> Draw:
    return FAMILIES[family](seed)


def all_ids():
    return [(f, s) for f, n in N_DRAWS.items() for s in range(n)]


def port_result(port, d: Draw):
    """The port's avg and samples over the whole draw (every call's passes and hops once)."""
    return port.power_scan(oracle_params(d.plan), d.window, d.x, d.n_pass, d.plan.n_hops, sine=d.sine)


# ------------------------------------------------------------------------------------------ named edge cases
# name -> the rx_power command line (the golden file holds the reference's avg sha256 and samples for each)
GOLDEN_CASES = {
    "box1400_bin_e1": dict(freq="100M:100.002M:1k", crop=0.0, boxcar=1, fir=0, peak=0, window="hamming", n_pass=3,
                           input="noise", seed=1),
    "box311_bin_e7": dict(freq="100M:100.009003M:71", crop=0.0, boxcar=1, fir=0, peak=0, window="blackman", n_pass=2,
                          input="tones", seed=2),
    "F9_P8_bin_e1": dict(freq="100M:100.008M:4k", crop=0.0, boxcar=0, fir=9, peak=0, window="rectangle", n_pass=3,
                         input="noise", seed=3),
    "F9_P10_bin_e1": dict(freq="100M:100.002M:1k", crop=0.0, boxcar=0, fir=9, peak=0, window="kaiser", n_pass=2,
                          input="dc", seed=4),
    "F0_P4_crop": dict(freq="100M:100.1M:100", crop=0.285, boxcar=0, fir=0, peak=1, window="youssef", n_pass=2,
                       input="noise", seed=5),
    "smem_limit_box7_bin_e13": dict(freq="100M:100.375M:46", crop=0.0, boxcar=1, fir=0, peak=0, window="hann-poisson",
                                    n_pass=2, input="noise", seed=6),
    "bin_e15_global_tables": dict(freq="100M:101M:31", crop=0.0, boxcar=1, fir=0, peak=0, window="blackman-harris",
                                  n_pass=1, input="tones", seed=7),
    "peak_fullscale_bin_e10": dict(freq="100M:101M:1k", crop=0.0, boxcar=1, fir=0, peak=1, window="rectangle",
                                   n_pass=4, input="noise", seed=8),
    "peak_fullscale_rails": dict(freq="100M:101M:1k", crop=0.0, boxcar=1, fir=0, peak=1, window="bartlett", n_pass=3,
                                 input="rails", seed=9),
    "dc_offset_bin_e12": dict(freq="100M:101M:300", crop=0.1, boxcar=1, fir=0, peak=0, window="hamming", n_pass=2,
                              input="dc", seed=10),
    "rms_bin_e0": dict(freq="100M:110M:1M", crop=0.0, boxcar=1, fir=0, peak=0, window="rectangle", n_pass=3,
                       input="dc", seed=11),
    "hops5_bin_e4": dict(freq="100M:106M:250k", crop=0.5, boxcar=1, fir=0, peak=0, window="blackman", n_pass=2,
                         input="noise", seed=12),
    "F9_P2_bin_e8": dict(freq="100M:100.5M:3k", crop=0.0, boxcar=0, fir=9, peak=0, window="hamming", n_pass=2,
                         input="tones", seed=13),
    "box3_bin_e14": dict(freq="100M:100.9M:60", crop=0.0, boxcar=1, fir=0, peak=0, window="rectangle", n_pass=1,
                         input="noise", seed=14),
    "zeros_bin_e9": dict(freq="100M:102M:4k", crop=0.0, boxcar=1, fir=0, peak=0, window="hamming", n_pass=2,
                         input="zeros", seed=15),
}


def golden_plan(c: dict) -> power.Plan:
    return power.plan_range(c["freq"], c["crop"], c["boxcar"], c["fir"], c["peak"])


def golden_input(c: dict, plan) -> np.ndarray:
    kind = "rail" if c["input"] == "rails" else c["input"]
    return hop_input(np.random.default_rng(c["seed"]), kind, (c["n_pass"], plan.n_hops, plan.buf_len), False)
