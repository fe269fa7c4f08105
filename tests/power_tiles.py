"""Cases of the tests of wide rx_power sweeps in tiles (rxb200_power_plan_tiles, rxb200_power_mix_accumulate_burst*):
the tiling rule restated in Python, the burst model, and the named shapes.

A burst is one self-contained capture after a retune: the lead of G = M ceil((T - 1) / M) complex samples, then whole
passes.  Hop i of the burst is power_mix.ddc over the whole burst from n = 0 with a zero history, less its first G / M
outputs (whose windows reach before the burst); every index the remaining outputs read lies inside the burst.  Each
tile's hop buffers are [P][he - hb][buf_len]; a sweep of one burst per tile gives every hop P passes, so the tiles
side by side along the hop axis are the hop buffers [P][n_hops][buf_len] the reference's scanner() sees.
"""
import numpy as np

import power_mix as pm
from rx_tools_b200 import power

MAX_INT = (1 << 31) - 1


def c(k, s):
    """A run of k hops is centred at its first hop plus c(k)."""
    return (k - 1) * s // 2


def mreq(k, s, r):
    ck = c(k, s)
    return -(-(2 * max(ck, (k - 1) * s - ck) + r) // r)


def tiling(plan, cap):
    """The planner's rule: None when refused, else (n_tiles, h, M, T, R, [(hb, he, centre)], offsets)."""
    r, s, f0, n = plan.rate, plan.freq_step, plan.first_freq, plan.n_hops
    mcap = min(4096, min(int(cap), MAX_INT) // r)
    if mcap < 1:
        return None
    hmax = max(k for k in range(1, n + 1) if mreq(k, s, r) <= mcap)
    n_tiles = -(-n // hmax)
    h = -(-n // n_tiles)
    M = mreq(h, s, r)
    tiles = []
    for t in range(n_tiles):
        hb, he = t * h, min((t + 1) * h, n)
        tiles.append((hb, he, f0 + t * h * s + c(he - hb, s)))
    offs = [plan.hop_freq(i) - tiles[i // h][2] for i in range(n)]
    return n_tiles, h, M, min(8191, 32 * M + 1), M * r, tiles, offs


def lead(decim, n_taps):
    return decim * (-(-(n_taps - 1) // decim))


def burst_buffers(burst, rate, offsets, dd, buf_len):
    """int16[P][len(offsets)][buf_len]: each hop of one burst (offsets: the tile's hops)."""
    decim, taps, _ = dd
    G = lead(decim, taps.size)
    x = np.asarray(burst, dtype=np.int16).reshape(-1)
    assert (x.size - 2 * G) % (decim * buf_len) == 0 and x.size > 2 * G
    P = (x.size - 2 * G) // (decim * buf_len)
    out = np.empty((P, len(offsets), buf_len), dtype=np.int16)
    for k, f in enumerate(offsets):
        y, _ = pm.ddc(x, rate, f, dd, 0)
        out[:, k, :] = y[2 * (G // decim):].reshape(P, buf_len)
    return out


# name -> the command line, the cap on the capture rate (Hz), passes per burst, the window, and an optional filter in
# place of the shell's (M from the tiling, taps from rxb200_ddc_lowpass(M, T, S) with the given T and S)
SHAPES = {
    "fm_band_6M": dict(pm.SHAPES["fm_band"], cap=6_000_000, n_pass=2),
    "hf_crop285_10M": dict(pm.SHAPES["hf_crop285"], cap=10_000_000, n_pass=1),
    "uhf_crop25_8M": dict(pm.SHAPES["uhf_crop25"], cap=8_000_000, n_pass=1),
    # -F 9 in place of the boxcar, two hops per tile (fifth_order passes need a span below 1 MHz: one hop, one tile)
    "F9": dict(freq="100M:110M:10k", crop=0.0, boxcar=0, fir=9, peak=0, window="kaiser", cap=5_000_000, n_pass=1),
    # -P peak hold
    "peak_hold": dict(pm.SHAPES["peak_hold"], cap=6_000_000, n_pass=2),
    # bin size >= 1 MHz: rms_power, bin_e = 0
    "rms": dict(pm.SHAPES["rms"], cap=6_000_000, n_pass=2),
    # a cap equal to the hop rate: tiles of one hop, M = 1
    "one_hop": dict(freq="100M:105M:10k", crop=0.0, boxcar=1, fir=0, peak=0, window="hamming", cap=2_500_000,
                    n_pass=2),
    # tiles of 300 hops (two grid rows of the kernel), the second starting at hop 300
    "hops300": dict(freq="100M:116.8M:10k", crop=0.99, boxcar=1, fir=0, peak=0, window="bartlett", cap=12_000_000,
                    n_pass=1, taps=(17, 15)),
    # taps summing to 2^17 at S = 17: the 64-bit accumulator
    "wide_acc": dict(pm.SHAPES["wide_acc"], cap=2_500_000, n_pass=1, taps=(65, 17)),
}


def shape(name):
    """(plan, window, Tiling, tiles, offsets, (M, taps, S)) of a named shape."""
    s = SHAPES[name]
    plan = power.plan_range(s["freq"], s["crop"], s["boxcar"], s["fir"], s["peak"])
    tl, tiles, offs = power.plan_tiles(plan, s["cap"])
    T, S = s.get("taps", (tl.n_taps, 15))
    dd = (tl.decim, power.ddc_lowpass(tl.decim, T, S), S)
    return plan, power.window_table(s["window"], 1 << plan.bin_e), tl, tiles, offs, dd


def bursts(name, seed=0, n_pass=None):
    """One burst per tile, n_pass passes each (the shape's by default)."""
    plan, win, tl, tiles, offs, dd = shape(name)
    P = SHAPES[name]["n_pass"] if n_pass is None else n_pass
    n_complex = lead(dd[0], dd[1].size) + P * dd[0] * plan.buf_len // 2
    return [pm.capture(n_complex, tl.capture_rate, offs[hb:he], 2600 + 17 * t + seed + len(name))
            for t, (hb, he, _) in enumerate(tiles)]


def case_input(name, seed=0):
    """(plan, window, Tiling, tiles, offsets, ddc, bursts) of a named shape."""
    return shape(name) + (bursts(name, seed),)


def tile_buffers(name, seed=0):
    """Each tile's hop buffers, and all of them side by side: int16[P][n_hops][buf_len]."""
    plan, win, tl, tiles, offs, dd, bs = case_input(name, seed)
    per = [burst_buffers(b, tl.capture_rate, offs[hb:he], dd, plan.buf_len) for b, (hb, he, _) in zip(bs, tiles)]
    return per, np.concatenate(per, axis=1)
