"""rx_power's capture and tile planners at a device rate (include/rxb200.h, "rx_power plans at a device rate") restated
in Python, and the shell's old inline capture-mode rule they replace.

A plan's hop rate is r = plan.rate, its step s, its first hop F0 and its n hops.  The capture planner centres the
capture at F0 + floor((n - 1) s / 2) and takes M = ceil((span + r + G) / r), span = 2 max |f_i|; the tiler shrinks its
tiles until each fits min(cap, R_dev).  G = ceil(R_dev / 32), or 0 without a device rate.
"""
import resample as rsm

MAX_RATE = (1 << 31) - 1


def inline_rule(plan, cap):
    """What rx_power_b200's capture mode computed inline before rxb200_power_plan_capture: (fc, offsets, M, R, T), or
    "rate" where it refused."""
    n = plan.n_hops
    fc = plan.first_freq + ((n - 1) * plan.freq_step) // 2
    offs = [plan.hop_freq(i) - fc for i in range(n)]
    span = 0
    for f in offs:
        span = max(span, 2 * abs(f))
    M = (span + plan.rate + plan.rate - 1) // plan.rate
    R = M * plan.rate
    if R > cap or R > MAX_RATE or M > 4096:
        return "rate"
    return fc, offs, M, R, min(8191, 32 * M + 1)


def capture_at_rule(plan, cap, R_dev):
    """rxb200_power_plan_capture_at restated: (fc, offsets, M, R, T, span), or the refusal "device_rate" (R_dev out of
    range), "rate" (the cap, 2^31 - 1 or M > 4096) or "device" (R > R_dev)."""
    if R_dev < 1 or R_dev > MAX_RATE:
        return "device_rate"
    n = plan.n_hops
    fc = plan.first_freq + ((n - 1) * plan.freq_step) // 2
    offs = [plan.hop_freq(i) - fc for i in range(n)]
    span = max(2 * abs(f) for f in offs)
    M = rsm.ceil_div(span + plan.rate + rsm.ceil_div(R_dev, 32), plan.rate)
    R = M * plan.rate
    if R > cap or R > MAX_RATE or M > 4096:
        return "rate"
    if R > R_dev:
        return "device"
    return fc, offs, M, R, min(8191, 32 * M + 1), span + plan.rate


def _c(k, s):
    return (k - 1) * s // 2


def _mreq(k, s, r, G):
    c = _c(k, s)
    return rsm.ceil_div(2 * max(c, (k - 1) * s - c) + r + G, r)


def tiles_at_rule(plan, cap, R_dev):
    """rxb200_power_plan_tiles_at restated: (n_tiles, h, M, R, T, offsets, [(hb, he, centre, span)]), or the refusal
    "device_rate", "mcap" (Mcap < 1) or "one" (a tile of one hop does not fit)."""
    if R_dev < 1 or R_dev > MAX_RATE:
        return "device_rate"
    n, r, s = plan.n_hops, plan.rate, plan.freq_step
    G = rsm.ceil_div(R_dev, 32)
    mcap = min(4096, min(cap, R_dev, MAX_RATE) // r)
    if mcap < 1:
        return "mcap"
    if _mreq(1, s, r, G) > mcap:
        return "one"
    hmax = 1
    while hmax < n and _mreq(hmax + 1, s, r, G) <= mcap:
        hmax += 1
    n_tiles = rsm.ceil_div(n, hmax)
    h = rsm.ceil_div(n, n_tiles)
    M = _mreq(h, s, r, G)
    offs, tiles = [], []
    for t in range(n_tiles):
        b, e = t * h, min((t + 1) * h, n)
        c = _c(e - b, s)
        tiles.append((b, e, plan.first_freq + b * s + c, 2 * max(c, (e - b - 1) * s - c) + r))
        offs += [(i - b) * s - c for i in range(b, e)]
    return n_tiles, h, M, M * r, min(8191, 32 * M + 1), offs, tiles
