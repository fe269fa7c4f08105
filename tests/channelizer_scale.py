"""The launch rules of fm_raster.cu and fm_two_stage.cu restated, so that a test can say which regime of the raster
kernels and of the two-stage plan it reaches and assert it, an exact model of both channelizers that scales to long
captures and many bins, and the captures that drive the raster sum to its exactness bound.

raster_plan is RasterPlan::plan's shape (Kp, Np, frames per scratch group); branch_regime is raster_front's choice of
frames per raster_branch_kernel CTA; two_stage_plan is TwoStage::plan's slots, grid rows and G.  The fine stage's
launch is ddc_launch, restated by mix_scale.ddc_regime with its rows argument.

raster_sparse evaluates the raster rule of include/rxb200.h straight from its definition,
    A = sum_{j<T} h[j] x[e - j] tw[(k (e - j)) mod K],
at the requested emission points only, in int64 torch on whatever device holds the capture: it never regroups the sum
by residue, so it shares nothing with the kernels' polyphase algorithm.  two_stage_sparse takes the coarse rows of the
distinct bins from it and runs the NCO mixer and the DDC in int64 over a chosen subset of the channels.
"""
import numpy as np

import fm_raster as frs
import fm_two_stage as fts
import mix_scale as ms
import power_mix as pmx

RAS_SPAN = 8192                  # capture samples a branch CTA stages at most
RAS_BM = 64                      # DFT tile: frames
RAS_BN = 64                      # DFT tile: output columns (32 channels)
RAS_BK = 16                      # DFT tile: input columns per stage
SCRATCH_BYTES = 64 << 20         # RXB200_RASTER_SCRATCH_BYTES
H100_SMS = (132, 114)            # SXM and PCIe


def raster_plan(K, C):
    """RasterPlan::plan's shape for K bins and C channels: (Kp, Np, frames per scratch group)."""
    Kp = -(-2 * K // RAS_BK) * RAS_BK
    Np = -(-2 * C // RAS_BN) * RAS_BN
    return Kp, Np, SCRATCH_BYTES // (Kp * 8) // RAS_BM * RAS_BM


def branch_regime(F, M, T, n_sm):
    """raster_front's frames per raster_branch_kernel CTA for a group of F frames: (U, which, dynamic shared memory
    bytes), which is "span" (the staging room) or "n_out" (the even share of the frames over 2 n_sm CTAs)."""
    ws = M if T >= M else T
    span = (RAS_SPAN - T) // ws + 1
    share = -(-F // (2 * n_sm))
    U = max(1, min(span, share))
    return U, "n_out" if share < span else "span", (T + (U - 1) * ws + T + U) * 4


def branch_span(M, T):
    """The most frames one branch CTA's staging room holds."""
    return (RAS_SPAN - T) // (M if T >= M else T) + 1


def two_stage_plan(K, bins, T2):
    """TwoStage::plan for the channels' bins: (the distinct bins in slot order, the grid rows as (slot, c0, nc) over the
    channels in bin order, G coarse frames per group)."""
    order = sorted(range(len(bins)), key=lambda c: bins[c])               # stable, as std::stable_sort
    slots, rows = [], []
    for k, c in enumerate(order):
        new_bin = not slots or slots[-1] != bins[c]
        if new_bin:
            slots.append(bins[c])
        if new_bin or rows[-1][2] == ms.MIX_GROUP:
            rows.append([len(slots) - 1, k, 0])
        rows[-1][2] += 1
    Kp, _, _ = raster_plan(K, len(slots))
    fixed = len(slots) * (T2 - 1) * 4
    per = Kp * 8 + len(slots) * 4
    G = max(64, int((SCRATCH_BYTES - fixed) / per) // 64 * 64)            # C++ division: toward zero
    return slots, [tuple(r) for r in rows], G


def _torch():
    import torch
    return torch


def _as_pairs(x):
    torch = _torch()
    return (x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x, dtype=np.int16))).reshape(-1, 2)


def _finish(acc, shift):
    y = acc if shift == 0 else (acc + (1 << (shift - 1))) >> shift
    return y.clamp(-32768, 32767).to(_torch().int16)


def raster_sparse(x, K, bins, taps, M, S, phase, pos=0, hist=None, frames=None, block=1 << 22):
    """The raster rule over one call at the emission points of `frames` (indices into the call's outputs; None: all):
    x is the call's capture as int16[2c] (numpy or a torch tensor on any device), phase the residue mod K of its first
    sample's index, pos the capture samples before the call (emission points are global samples m M + M - 1), hist the
    T - 1 samples before it as int16[2(T - 1)] (None: zeros).  Returns int16[len(bins)][2 len(frames)] numpy."""
    torch = _torch()
    xt = _as_pairs(x)
    dev = xt.device
    taps = np.asarray(taps, dtype=np.int64).reshape(-1)
    T, H, K, M = taps.size, taps.size - 1, int(K), int(M)
    assert frs.sum_abs(taps) < (1 << 22)
    h = (torch.zeros((H, 2), dtype=torch.int16, device=dev) if hist is None
         else _as_pairs(hist).to(dev))
    assert h.shape[0] == H
    c = xt.shape[0]
    m0, m1 = pos // M, (pos + c) // M
    fr = (torch.arange(m1 - m0, dtype=torch.int64) if frames is None
          else torch.as_tensor(np.asarray(frames, dtype=np.int64))).to(dev)
    assert fr.numel() == 0 or (int(fr.min()) >= 0 and int(fr.max()) < m1 - m0)
    e = (m0 + fr) * M + (M - 1 - pos)                                    # local emission points
    hr = torch.as_tensor(taps[::-1].copy()).to(dev)
    span = torch.arange(T, dtype=torch.int64, device=dev) - H
    tw = torch.as_tensor(frs.table(K).astype(np.int64)).to(dev)
    kb = torch.as_tensor(np.asarray(bins, dtype=np.int64)).to(dev)
    acc = torch.empty((kb.numel(), fr.numel(), 2), dtype=torch.int64, device=dev)
    per = max(1, block // T)
    for a in range(0, fr.numel(), per):
        j = e[a:a + per, None] + span                                     # local index of each window sample
        raw = xt[j.clamp(min=0)].to(torch.int64)
        if H:
            raw = torch.where((j >= 0)[..., None], raw, h[(j + H).clamp(min=0, max=H - 1)].to(torch.int64))
        res = torch.remainder(int(phase) % K + j, K)                     # each sample's index mod K
        nb = max(1, block // j.numel())
        for b in range(0, kb.numel(), nb):
            t = tw[(kb[b:b + nb, None, None] * res) % K]                   # (bins, frames, T, 2)
            zr = raw[..., 0] * t[..., 0] - raw[..., 1] * t[..., 1]       # |z| <= 2^31: exact
            zi = raw[..., 0] * t[..., 1] + raw[..., 1] * t[..., 0]
            acc[b:b + nb, a:a + per, 0] = (zr * hr).sum(-1)
            acc[b:b + nb, a:a + per, 1] = (zi * hr).sum(-1)
    return _finish(acc, S).reshape(kb.numel(), -1).cpu().numpy()


def two_stage_sparse(x, rate, K, offsets, coarse, fine, n0=0, channels=None):
    """The two-stage rule (fm_two_stage.two_stage_model) over a whole stream for the channels in `channels` (indices
    into offsets; None: all): int16[len(channels)][2 floor(c / (M1 M2))] numpy.  The coarse rows come from
    raster_sparse for the distinct bins of those channels, on the device that holds x; the fine stage is the NCO
    mixer by word and the sparse DDC."""
    torch = _torch()
    xt = _as_pairs(x)
    M1, h1, S1 = coarse
    M2, h2, S2 = fine
    M1, M2 = int(M1), int(M2)
    chans = list(range(len(offsets))) if channels is None else [int(c) for c in channels]
    n_out = xt.shape[0] // (M1 * M2)
    out = np.empty((len(chans), 2 * n_out), np.int16)
    if n_out == 0:
        return out
    n1 = n_out * M2
    bw = [fts.bin_word(rate, K, M1, offsets[c]) for c in chans]
    slots = sorted({b for b, _ in bw})
    y = raster_sparse(xt[:n1 * M1], K, slots, h1, M1, S1, int(n0) % K)
    for i, (b, w) in enumerate(bw):
        z = torch.as_tensor(fts.nco_mix_word(y[slots.index(b)], w, int(n0) // M1)).to(xt.device)
        out[i], _ = ms.ddc_sparse(z, pmx.IDENTITY, h2, M2, S2, block=(1 << 24) if z.is_cuda else (1 << 21))
    return out


def split_reads(y, lens16, M, pos=0):
    """A channel's whole decimated stream from create split by a read sequence: each read's part (possibly empty)."""
    out, at = [], 0
    for n16 in lens16:
        d = ((pos + n16 // 2) // M - pos // M) * 2
        out.append(y[at:at + d])
        at += d
        pos += n16 // 2
    assert at == y.size
    return out


# ---- the GPU cases' sizes, derived from the SM count -------------------------------------------------------------
# a. DFT column tiles: (K, bins) of rxb200_raster_device calls with F frames (above 64, not a multiple of 64)
def column_tile_cases():
    rng = np.random.default_rng(768)
    return {
        "k768_all": (768, [int(b) for b in rng.permutation(768)]),
        "k100_c33": (100, [int(b) for b in rng.choice(100, size=33, replace=False)]),
        "k4096_c1000": (4096, [int(b) for b in rng.integers(0, 4096, size=1000)]),
        "k12_twice": (12, [b for b in range(12) for _ in range(2)]),
    }


COLUMN_TILE_FRAMES = 131         # three row tiles, the last of 3 frames


def tile_channels(C, seed, extra=16):
    """The first and last channel of every 32-channel DFT column tile, and `extra` seeded others."""
    picked = {c for t in range(0, C, 32) for c in (t, min(C, t + 32) - 1)}
    picked |= {int(c) for c in np.random.default_rng(seed).choice(C, size=min(C, extra), replace=False)}
    return sorted(picked)


# b. fine grid-row split: one bin with 600 channels, one with 257, one with 1
SPLIT_RATE, SPLIT_K = 2_048_000, 16
SPLIT_BINS = ((3, 600), (12, 257), (7, 1))


def split_offsets():
    """The channels of the grid-row split case in a seeded order: distinct offsets inside each bin of SPLIT_BINS."""
    rng = np.random.default_rng(600)
    width = SPLIT_RATE // SPLIT_K
    offs = []
    for b, n in SPLIT_BINS:
        centre = (b if 2 * b <= SPLIT_K else b - SPLIT_K) * width
        offs += [int(centre + d) for d in rng.choice(np.arange(-width // 2 + 1, width // 2), size=n, replace=False)]
    return [offs[i] for i in rng.permutation(len(offs))]


def many_rows_offsets(n_sm):
    """More than 2 n_sm distinct bins of K = 4096 at 4.096 Msps, one channel each plus a second in every 7th bin: the
    fine stage gets one CTA per grid row."""
    n = 2 * n_sm + 7
    offs = [1000 * k - 2_000_000 + 311 for k in range(n)]
    return offs + [f + 13 for f in offs[::7]]


# c. coarse groups shorter than the fine history
GROUP_RATE, GROUP_K = 4_096_000, 4096
GROUP_OFFSETS = [-1_999_001, -777_777, -1000, 0, 1_500_250, 123_457, 1_000_500, 2_047_499]   # eight distinct bins
GROUP_READS = [2 * 1931] * 7 + [2 * 5, 2 * 967, 2 * 2 * 960]     # 1931 = 6 mod 7: each read starts at a new residue


def group_reads_phases(reads, G, M2):
    """(the fine decimation phase ph2 at the start of each read, whether it holds more than one coarse group) for a
    handle at M1 = 1 from create."""
    out, pos = [], 0
    for n16 in reads:
        out.append((pos % M2, n16 // 2 > G))
        pos += n16 // 2
    return out


# d. branch kernel with U set by the staging room: K = 8, one scratch group
SPAN_K = 8
SPAN_SHAPES = [(8, 8), (64, 13), (1, 6500)]


def span_frames(M, T, n_sm):
    """Frames of a call whose every branch CTA but the last holds the staging room's U frames: 2 n_sm + 1 CTAs, the last
    with 37 frames."""
    return 2 * n_sm * branch_span(M, T) + 37


# e. raster handle over scratch groups with T > M > 1
GROUPS_K, GROUPS_M, GROUPS_T = 4096, 7, 129
GROUPS_BINS = [0, 1, 2048, 4095, 1365]


def groups_frames():
    return 5 * raster_plan(GROUPS_K, len(GROUPS_BINS))[2] + 300


# f. sums at the exactness bound
BOUND_KS = (3, 48, 4096)
BOUND_H = (1 << 21) - 1          # two taps of H and one of 1: sum |h| = 2^22 - 1


def bound_case(K):
    """(cancelling bin, taps, M = T): taps H at 0 and +-H at d, 1 at d + 1.  The samples at e and e - d fall in residue
    classes whose twiddles at the cancelling bin are equal (K = 3, bin 0, taps H and -H) or opposite (even K, an odd
    bin, d = K / 2, taps H and H), so equal samples there cancel exactly; windows do not overlap (M = T)."""
    if K == 3:
        k, d, sign = 0, 1, -1
    else:
        k, d, sign = {48: 5, 4096: 1365}[K], K // 2, 1
    T = d + 2
    taps = np.zeros(T, np.int32)
    taps[0], taps[d], taps[T - 1] = BOUND_H, sign * BOUND_H, 1
    return k, taps, T


def bound_capture(K, n_frames, phase, seed, aligned):
    """A full-scale capture of n_frames windows for bound_case(K), sample i of index residue (phase + i) mod K.
    aligned=False: in every window the two big taps see one full-scale sample (-32768 in every fourth), so the
    cancelling bin's sum is t x with x in {0, +-1, +-i} at the unit tap, |A| < 2^15.  aligned=True: the big taps' samples
    are signed so that every term of bin 1's I sum has the frame's sign, at full scale in even frames and at a random
    scale in [1/2, 1] in odd ones, so |A| reaches 2^52 and the output crosses the saturation edge near S = 37."""
    k, taps, M = bound_case(K)
    T = taps.size
    tw = frs.table(K).astype(np.int64)
    rng = np.random.default_rng(seed)
    x = rng.integers(-32768, 32768, size=(n_frames * M, 2)).astype(np.int64)
    big = [j for j in range(T) if abs(int(taps[j])) > 1]
    for m in range(n_frames):
        e = m * M + M - 1
        if not aligned:
            v = rng.integers(24000, 32768, size=2) * rng.choice([-1, 1], size=2)
            if m % 4 == 0:
                v[m % 8 // 4] = -32768
            for j in big:
                x[e - j] = v
            t3 = tw[(k * ((phase + e - (T - 1)) % K)) % K]
            units = [u for u in ((0, 0), (1, 0), (0, 1), (-1, 0), (0, -1))
                     if max(abs(t3[0] * u[0] - t3[1] * u[1]), abs(t3[1] * u[0] + t3[0] * u[1])) < 32768]
            x[e - (T - 1)] = units[rng.integers(len(units))]
            continue
        sigma = 1 if m % 2 else -1
        scale = 1.0 if m % 4 < 2 else rng.uniform(0.5, 1.0)
        for j in big:
            t = tw[(1 * ((phase + e - j) % K)) % K]
            want_a = sigma * np.sign(int(taps[j]) * t[0])                # sign of a making h c a of sign sigma
            want_b = -sigma * np.sign(int(taps[j]) * t[1])               # sign of b making -h s b of sign sigma
            x[e - j] = [int(round((32767 if w > 0 else -32768) * scale)) if w else rng.integers(-32768, 32768)
                        for w in (want_a, want_b)]
    return x.reshape(-1).astype(np.int16)
