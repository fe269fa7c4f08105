"""The rational resampler and the capture handles that carry one, on the GPU, in the regimes the short tests never reach.
Every case first asserts the regime it claims (tests/device_rate_scale.py restates the launch rule and the groups),
then compares bytes.

a. resample_kernel at the edges of its accepted range: J L = 2^22 with v up to 512 (L - 1) just below 2^31, U set by
   the staging span (82 and 1), both sides of the shared-memory taps flip (L J = 12288 / 12289), and both sides of the
   int32 / int64 accumulator flip with the input that drives every sum to its bound; at device counts 0, around the
   count where the output index passes 2^32, and near 2^64; against the numpy model or the sparse model, with guard
   words, through the stateless entry and a ragged handle sequence.
b. The six named plans with their real taps over 2^23 device samples, stateless and through the handle.
c. Capture handles at the named plans with the fronts the _at planners make, over about a second of device samples,
   cut four ways through the host and device entries (and rx_fm in one chunked call of the whole stream, since a read
   holds fewer capture samples than most groups), against the composition on the GPU (the resampler, then the same
   handle without one), with the raster, two-stage and rx_sdr host groups each case crosses asserted; and a host call
   whose device memory, counted per process, stays within the rx_sdr scratch bytes.
d. rx_power calls that resample to more passes than one scratch group holds, and an L > N resampler whose whole-pass
   cuts are found by search, a cut one sample short refused without changing the handle.
e. An rx_sdr and an rx_power handle fed past 2^32 device and capture samples, their last call compared with the
   stateless entries at those counts.
"""
import numpy as np
import pytest

import channelizer_scale as cs
import device_rate as dr
import device_rate_scale as drs
import fm_handles as fh
import fm_two_stage as fts
import mix_scale as ms
import power_mix as pm
import resample as rsm
from rx_tools_b200 import _lib, fm, power, sdr
from rx_tools_b200 import resample as rs

pytestmark = pytest.mark.gpu

GUARD = 0x7A7A
P = fm.derive_params(rate_s=170_000).params


def _sms():
    return ms.device_sms()


def _stream(n, seed):
    return np.random.default_rng(seed).integers(-32768, 32768, size=2 * n).astype(np.int16)


def _device_entry(L, N, h, S, n0, d_x, c, extra=16):
    """rxb200_resample_device over c samples of the CUDA tensor d_x: (outputs int16 [2 n], guard tail)."""
    torch = fh.torch()
    n = rsm.out_count(n0, c, L, N)
    dst = torch.full((2 * (n + extra),), GUARD, dtype=torch.int16, device="cuda")
    rs.resample_device(L, N, h, S, n0, d_x.data_ptr(), c, dst.data_ptr())
    torch.cuda.synchronize()
    d = dst.cpu().numpy()
    return d[:2 * n], d[2 * n:]


def _handle_device_calls(r, d_x, cuts, total):
    """A resampler handle's device entry over the cuts (complex samples) of d_x, into one buffer with guard words."""
    torch = fh.torch()
    dst = torch.full((2 * total + 32,), GUARD, dtype=torch.int16, device="cuda")
    at, done = 0, 0
    for c in cuts:
        done += r.process_device(d_x.data_ptr() + 4 * at, 2 * c, dst.data_ptr() + 4 * done, total - done, sync=0)
        at += c
    torch.cuda.synchronize()
    d = dst.cpu().numpy()
    assert done == total and np.all(d[2 * total:] == GUARD)
    return d[:2 * total]


def _ragged(n, seed, lo=1, hi=200_000):
    rng = np.random.default_rng(seed)
    out, at = [], 0
    for c in [1, 3, 2]:
        out.append(c)
        at += c
    while at < n:
        c = min(int(rng.integers(lo, hi)), n - at)
        out.append(c)
        at += c
    return out


def _check(got, x_ext, H, L, N, h, S, n0, a, lead, edges=(), seed=0):
    """got equals the rule over the call at n0: the numpy model where affordable, else the sparse model at
    check_indices.  a: the plan of the launch that made got, lead outputs ahead of the call's first."""
    J = h.size // L
    n = a["n_out"] - lead
    assert got.size == 2 * n
    if n * J <= (1 << 25):
        want, _ = rsm.resample_model(x_ext[2 * H:], L, N, h, S, n0, x_ext[2 * (H - (J - 1)):2 * H] if J > 1 else None)
        assert np.array_equal(got, want)
        return
    idx = drs.check_indices(n, a["U"], J, edges, seed, lead=lead)
    want = drs.sparse_outputs(x_ext, H, L, N, h, S, n0, idx)
    assert np.array_equal(got.reshape(-1, 2)[idx], want)


def _launched(L, N, J, n0, H, c, n_sm):
    """The plan of the launch _call_with_context makes for the call of c samples at n0, and its outputs ahead of the
    call's first."""
    if n0 == 0:
        return drs.launch(L, N, J, 0, c, n_sm), 0
    return drs.launch(L, N, J, n0 - H, H + c, n_sm), rsm.out_count(n0 - H, H, L, N)


def _call_with_context(L, N, h, S, n0, d_x, x, xz, H, c):
    """The stateless entry over the call of c samples at n0 whose stream is x[H:] (int16 pairs), its context the H
    samples before: zeros for a call from 0, else the stream's own, the entry starting H samples earlier and the
    outputs whose q falls in the context dropped.  (the call's outputs, the stream with its context)"""
    if n0 == 0:
        got, tail = _device_entry(L, N, h, S, 0, d_x[2 * H:], c)
        assert np.all(tail == GUARD)
        return got, xz
    got_all, tail = _device_entry(L, N, h, S, n0 - H, d_x, H + c)
    assert np.all(tail == GUARD)
    return got_all[2 * rsm.out_count(n0 - H, H, L, N):], x


# ---- a. the kernel at the edges of its range
def _edge_taps(kind, L, J, rng):
    """(taps, S, wide) of an edge case.  acc_S_sum: every phase's taps non-negative and summing to sum, so that an input
    of -32768 drives every output's sum, and each lane's partial sum, to -32768 sum."""
    if kind.startswith("acc"):
        _, S, total = kind.split("_")
        S, total = int(S), int(total)
        h = np.zeros(L * J, np.int64)
        for p in range(L):
            w = rng.integers(1, 1000, size=J).astype(np.float64)
            col = np.floor(w / w.sum() * total).astype(np.int64)
            col[int(rng.integers(0, J))] += total - col.sum()
            h[p::L] = col
        return h.astype(np.int32), S
    if kind == "wide":
        return rng.integers(-(1 << 20), (1 << 20) + 1, size=L * J).astype(np.int32), 24
    lim = max(1, 65535 // J - 1)
    return rng.integers(-lim, lim + 1, size=L * J).astype(np.int32), 15


# name: (L, N, J, taps kind, the regime: (U, which), smem_taps, wide)
EDGES = {
    "top_J1_N=L-1": (4194301, 4194300, 1, "narrow", (512, "max_u"), False, False),
    "top_J1_N=2L-1": (4194301, 8388601, 1, "wide", (512, "max_u"), False, True),
    "top_J1024": (4096, 8191, 1024, "narrow", (512, "max_u"), False, False),
    "span_U82": (1, 100, 8, "narrow", (82, "span"), True, False),
    "span_U1_J8": (3, 40_000, 8, "wide", (1, "span"), True, True),
    "span_U1_J1024": (3, 40_000, 1024, "narrow", (1, "span"), True, False),
    "smem_12288": (12288, 24575, 1, "narrow", (512, "max_u"), True, False),
    "gmem_12289": (12289, 24577, 1, "narrow", (512, "max_u"), False, False),
    "smem_1536x8": (1536, 3071, 8, "wide", (512, "max_u"), True, True),
    "gmem_1537x8": (1537, 3073, 8, "wide", (512, "max_u"), False, True),
    # g = 65535 * 2^15 + 2^14 = 2^31 - 2^14, the largest g at S = 15 below 2^31: int32
    "acc_15_65535": (5, 7, 24, "acc_15_65535", (512, "max_u"), True, False),
    # g = 65537 * 2^15 + 2^14 > 2^31: int64, and the sums reach -2^31 - 2^15
    "acc_15_65537": (5, 7, 24, "acc_15_65537", (512, "max_u"), True, True),
    # g = 65534 * 2^15 + 2^15 = 2^31 - 2^15: int32, outputs unsaturated (-32767)
    "acc_16_65534": (5, 7, 24, "acc_16_65534", (512, "max_u"), True, False),
    # g = 2^31 exactly: int64
    "acc_16_65535": (5, 7, 24, "acc_16_65535", (512, "max_u"), True, True),
}


def _edge_len(L, N, U, n_sm):
    """Device samples for at least two waves (4 n_sm CTAs) at U outputs per CTA."""
    return rsm.ceil_div(4 * n_sm * U * N, L) + 7


def _edge_n0s(L, N, c):
    x = (1 << 32) * N // L                     # the device count where the output index reaches 2^32
    return [0, x - 3, x + 3, min((1 << 64) - (1 << 20), (1 << 64) - c - 1)]


@pytest.mark.parametrize("name", list(EDGES))
def test_kernel_at_the_edges(name):
    torch = fh.torch()
    L, N, J, kind, (U, which), smem_taps, wide = EDGES[name]
    rng = np.random.default_rng(len(name) * 7919 + L)
    h, S = _edge_taps(kind, L, J, rng)
    assert rsm.wide(h, L, S) == wide
    if kind.startswith("acc"):
        g = max(int(h[p::L].astype(np.int64).sum()) for p in range(L)) * 32768 + (1 << (S - 1))
        assert (g >= 1 << 31) == wide and (g < 1 << 31 or g - (1 << 31) <= 2 * 32768)
    n_sm = _sms()
    c = _edge_len(L, N, U, n_sm)
    H = J + 8
    x = _stream(H + c, 11)
    if kind.startswith("acc"):
        x.reshape(-1, 2)[H + c // 3:H + 2 * c // 3] = -32768          # the adversarial third: every sum at its bound
    d_x = torch.from_numpy(x).cuda()
    xz = x.copy()
    xz[:2 * H] = 0                                                      # the context of a call from 0
    for k, n0 in enumerate(_edge_n0s(L, N, c)):
        a, lead = _launched(L, N, J, n0, H, c, n_sm)                   # the launch that runs, context included
        assert (a["U"], a["which"]) == (U, which) and a["smem_taps"] == smem_taps, (name, n0, a)
        assert a["ctas"] >= 4 * n_sm
        assert a["worst_v"] < 1 << 31 and a["worst_staged"] <= a["room"] <= drs.RS_SPAN
        if name.startswith("top_J1_"):
            assert a["worst_v"] > (1 << 31) - (1 << 23)
        got, ext = _call_with_context(L, N, h, S, n0, d_x, x, xz, H, c)
        _check(got, ext, H, L, N, h, S, n0, a, lead, seed=k)
        if kind.startswith("acc") and not kind.endswith("65537"):
            # the adversarial outputs: clipped to -32768 at S = 15, and exact and unsaturated (-32767) at S = 16
            mid = got.reshape(-1, 2)[(a["n_out"] - lead) // 2]
            total = int(kind.split("_")[2])
            assert mid[0] == max(-32768, (-32768 * total + (1 << (S - 1))) >> S)
    # a ragged handle sequence from 0 equals the stateless entry from 0 (zero context)
    r = rs.Resampler(L, N, h, S)
    d_c = d_x[2 * H:]
    want, _ = _device_entry(L, N, h, S, 0, d_c, c)
    cuts = _ragged(c, L + N, hi=max(2, 3 * c // 7))
    assert np.array_equal(_handle_device_calls(r, d_c, cuts, rsm.out_count(0, c, L, N)), want)
    r.close()


# ---- b. the named plans with their real taps
NAMED_LEN = (1 << 23) + 4321


@pytest.mark.parametrize("name", [p[0] for p in rsm.NAMED])
def test_named_plan_over_2_23_samples(name):
    torch = fh.torch()
    _, R_dev, R, span, (L, N), J = next(p for p in rsm.NAMED if p[0] == name)
    assert tuple(rs.plan_resample(R_dev, R, span)) == (L, N, J, 15)
    h = rs.lowpass(L, N, J)
    n_sm = _sms()
    c = NAMED_LEN
    H = J + 8
    x = _stream(H + c, L)
    d_x = torch.from_numpy(x).cuda()
    xz = x.copy()
    xz[:2 * H] = 0
    for n0 in (0, (1 << 32) * N // L - 1000):
        a, lead = _launched(L, N, J, n0, H, c, n_sm)
        assert a["U"] == 512 and a["which"] == "max_u" and a["smem_taps"] == (L * J <= drs.RS_SMEM_TAPS)
        assert a["worst_v"] < 1 << 31 and a["worst_staged"] <= a["room"] <= drs.RS_SPAN
        got, ext = _call_with_context(L, N, h, 15, n0, d_x, x, xz, H, c)
        idx = drs.check_indices(a["n_out"] - lead, a["U"], J, seed=n0 & 0xff, lead=lead)
        assert np.array_equal(got.reshape(-1, 2)[idx], drs.sparse_outputs(ext, H, L, N, h, 15, n0, idx))
        # in_len is exact at every count for L < N
        for k in (1, 1000, 123_457):
            m = rs.in_len(L, N, n0, k)
            assert rsm.out_count(n0, m, L, N) == k and rsm.out_count(n0, m - 1, L, N) == k - 1
    d_c = d_x[2 * H:]
    want, _ = _device_entry(L, N, h, 15, 0, d_c, c)
    r = rs.Resampler(L, N, h, 15)
    assert np.array_equal(_handle_device_calls(r, d_c, _ragged(c, J, hi=400_000), want.size // 2), want)
    r.reset()
    assert np.array_equal(r.process(x[2 * H:]), want)
    r.close()


# ---- c. capture handles at the named plans, with the fronts the _at planners make
def _named(name):
    _, R_dev, R, span, (L, N), J = next(p for p in rsm.NAMED if p[0] == name)
    return R_dev, R, span, L, N, J


def _subset(v, k=8):
    """k entries spread over v (all of them when there are at most k)."""
    if len(v) <= k:
        return list(v)
    return [v[i * (len(v) - 1) // (k - 1)] for i in range(k)]


# name: (handle family, front kind, device rate, tuned frequencies, chain rate, seconds of device samples, the named
# plan the front's resampler is, or None: the two-stage fronts' rate M' c, M' a multiple of 4, is a plan of its own)
HANDLES = {
    "fm_single_noaa_2.4M": ("fm", "single", 2_400_000, dr.NOAA7, 1_008_000, 1.0, "noaa7_nbfm_2.4M"),
    "fm_single_noaa_2.5M": ("fm", "single", 2_500_000, dr.NOAA7, 1_008_000, 1.0, "noaa7_nbfm_2.5M"),
    "fm_two_stage_fm100_30.72M": ("fm", "two_stage", 30_720_000, dr.FM100, 1_020_000, 1.0, None),
    "fm_raster_fm100_30.72M": ("fm", "raster", 30_720_000, dr.FM100, 1_020_000, 1.0, "fm100_wbfm_30.72M"),
    "fm_two_stage_fm100_61.44M": ("fm", "two_stage", 61_440_000, dr.FM100, 1_020_000, 0.5, None),
    "fm_raster_fm100_61.44M": ("fm", "raster", 61_440_000, dr.FM100, 1_020_000, 0.5, "fm100_wbfm_61.44M"),
    "sdr_two_stage_fm100_30.72M": ("sdr", "two_stage", 30_720_000, dr.FM100, 1_020_000, 1.0, None),
    "sdr_raster_fm100_61.44M": ("sdr", "raster", 61_440_000, dr.FM100, 1_020_000, 0.5, "fm100_wbfm_61.44M"),
    "sdr_single_sdr4_2.4M": ("sdr", "single", 2_400_000, dr.SDR4, 250_000, 7.5, "sdr4_250k_2.4M"),
    "sdr_raster_fm100_2125_3072": ("sdr", "raster", 30_720_000, dr.FM100, 250_000, 1.0, "fm100_sdr_raster_30.72M"),
}
CAP = 10 ** 10


def _front(fam, kind, tuned, chain, R_dev):
    """(constructor of the handle without a resampler, decimation, front description, capture rate, span) from the
    _at planner."""
    rule = dr.plan_at({"single": dr.FM if fam == "fm" else dr.SDR, "raster": dr.RASTER,
                       "two_stage": dr.TWO_STAGE}[kind], tuned, chain, CAP, R_dev)
    R, span = rule["R"], rule["span"]
    return _make(fam, kind, tuned, chain, R_dev, R) + (R, span)


def _make(fam, kind, tuned, chain, R_dev, R):
    if kind == "single":
        planner = fm.plan_capture if fam == "fm" else sdr.plan_sdr_capture
        pl, offs = planner(tuned, chain, CAP, device_rate=R_dev)
        assert pl.capture_rate == R
        dd = (pl.decim, power.ddc_lowpass(pl.decim, pl.n_taps, 15), 15)
        if fam == "fm":
            return (lambda: fm.FmMix(P, R, offs, ddc=dd)), pl.decim, dict(kind=kind)
        return (lambda: sdr.SdrMix(R, offs, ddc=dd)), pl.decim, dict(kind=kind)
    if kind == "raster":
        pl, bins = fm.plan_capture_raster(tuned, chain, CAP, device_rate=R_dev)
        assert pl.capture_rate == R
        bins = _subset(bins)
        dd = (pl.decim, power.ddc_lowpass(pl.decim, pl.n_taps, 15), pl.shift)
        _, _, group = cs.raster_plan(pl.n_bins, len(bins))
        info = dict(kind=kind, group=group)
        if fam == "fm":
            return (lambda: fm.FmMix(P, ddc=dd, raster=(pl.n_bins, bins))), pl.decim, info
        return (lambda: sdr.SdrMix(ddc=dd, raster=(pl.n_bins, bins))), pl.decim, info
    pl, offs = fm.plan_capture_two_stage(tuned, chain, CAP, device_rate=R_dev)
    assert pl.capture_rate == R
    offs = _subset(offs)
    coarse = (pl.coarse_decim, power.ddc_lowpass(pl.coarse_decim, pl.coarse_taps, 15), pl.coarse_shift)
    fine = (pl.fine_decim, power.ddc_lowpass(pl.fine_decim, pl.fine_taps, 15), pl.fine_shift)
    bins = [fts.bin_word(R, pl.n_bins, pl.coarse_decim, o)[0] for o in offs]
    info = dict(kind=kind, M1=pl.coarse_decim, G=cs.two_stage_plan(pl.n_bins, bins, pl.fine_taps)[2])
    ts = (pl.n_bins, coarse, fine)
    if fam == "fm":
        return (lambda: fm.FmMix(P, R, offs, two_stage=ts)), pl.coarse_decim * pl.fine_decim, info
    return (lambda: sdr.SdrMix(R, offs, two_stage=ts)), pl.coarse_decim * pl.fine_decim, info


def _groups_crossed(info, cap_cuts, M):
    """The most scratch groups of the front any one call crosses (1 for a single stage)."""
    if info["kind"] == "single":
        return 1
    if info["kind"] == "raster":
        G, D = info["group"], M
    else:
        G, D = info["G"], info["M1"]
    best, pos = 1, 0
    for c in cap_cuts:
        frames = (pos + c) // D - pos // D
        best = max(best, rsm.ceil_div(frames, G))
        pos += c
    return best


FM_READ = 131072                                # capture samples an rx_fm read holds at most


def _cut_patterns(n, L, N, big, fam):
    """Device-call lengths covering n samples, by pattern.  "whole": one call (rx_fm: reads of the most device samples
    whose capture fits one read)."""
    whole = n if fam == "sdr" else FM_READ * N // L
    big = min(big, whole)
    out = {"whole": [whole], "16384": [16384], "131072": [131072], "ragged": "rand"}
    if (L, N) == (187, 256):
        out["1"] = [1]
        out["3"] = [3]
    pats = {}
    for k, p in out.items():
        if p == "rand":
            pats[k] = _ragged(n, 99, lo=1000, hi=big)
            continue
        limit = 3000 if p[0] < 16 else n                               # 1- and 3-sample cuts over the first 3000
        cuts, at = [], 0
        while at < limit:
            cuts.append(min(p[0], limit - at))
            at += cuts[-1]
        while at < n:                                                   # the rest in reads of the "whole" length
            cuts.append(min(whole, n - at))
            at += cuts[-1]
        pats[k] = cuts
    return pats


def _fm_run(mx, d_x, cuts, device):
    torch = fh.torch()
    outs, at = [], 0
    for c in cuts:
        if device:
            cap = mx.max_output(2 * c, max(mx._capture_int16(2 * c), 1)) + 8
            d_out = torch.zeros((mx.n_channels, cap), dtype=torch.int16, device="cuda")
            n = mx.process_read_device(d_x.data_ptr() + 4 * at, 2 * c, d_out.data_ptr(), cap, sync=True)
            outs.append(d_out[:, :n].cpu().numpy())
        else:
            outs.append(mx.process_read(d_x[2 * at:2 * (at + c)].cpu().numpy()))
        at += c
    return np.concatenate(outs, axis=1)


def _sdr_run(mx, d_x, cuts, device):
    torch = fh.torch()
    outs, at = [], 0
    for c in cuts:
        if device:
            n = mx.decimated_len(2 * c)
            stride = max(n, 1)
            d_out = torch.zeros(mx.n_channels * stride * 2, dtype=torch.int16, device="cuda")
            got = mx.process_device(d_x.data_ptr() + 4 * at, 2 * c, sdr.OUT_CS16, d_out.data_ptr(),
                                    mx.n_channels * stride, stride, sync=1)
            assert got == n
            outs.append(d_out.reshape(mx.n_channels, -1)[:, :2 * n].cpu().numpy())
        else:
            outs.append(mx.process(d_x[2 * at:2 * (at + c)].cpu().numpy()))
        at += c
    return np.concatenate(outs, axis=1)


@pytest.mark.parametrize("name", list(HANDLES))
def test_handle_at_named_plan(name):
    torch = fh.torch()
    fam, kind, R_dev, tuned, chain, secs, plan = HANDLES[name]
    make, M, info, R, span = _front(fam, kind, tuned, chain, R_dev)
    L, N, J, S = rs.plan_resample(R_dev, R, span)
    assert S == 15 and L < N
    if plan is not None:
        assert (R_dev, R, span, L, N, J) == _named(plan)
    taps = rs.lowpass(L, N, J)
    n = int(R_dev * secs) + 777
    x = _stream(n, len(name))
    d_x = torch.from_numpy(x).cuda()
    # the reference's resampler stage: the stateless entry over the whole stream, spot-checked at the cut edges below
    y_all, tail = _device_entry(L, N, taps, 15, 0, d_x, n)
    assert np.all(tail == GUARD)
    d_y = torch.from_numpy(y_all).cuda()
    run = _fm_run if fam == "fm" else _sdr_run
    crossed = {}
    for pname, cuts in _cut_patterns(n, L, N, max(2000, R_dev // 3), fam).items():
        cap_cuts, n0 = [], 0
        for c in cuts:
            cap_cuts.append(rsm.out_count(n0, c, L, N))
            n0 += c
        crossed[pname] = _groups_crossed(info, cap_cuts, M)
        ref = make()
        if fam == "fm":
            want = run(ref, d_y, [v for v in cap_cuts if v], False)
        else:
            want = ref.process(y_all)
        ref.close()
        for device in (False, True):
            if pname in ("1", "3") and not device:
                continue                                                # the device entry covers the short cuts
            mx = make()
            mx.set_device_rate(L, N, taps, 15)
            got = run(mx, d_x, cuts, device)
            mx.close()
            assert np.array_equal(got, want), (name, pname, device)
    if fam == "fm":
        # one chunked call of the whole stream: its capture goes through the front at once, across the scratch groups
        # that no single read reaches (chunk_int16 counts capture int16)
        chunk = 2 * M * 2048
        crossed["chunked"] = _groups_crossed(info, [y_all.size // 2], M)
        ref = make()
        want = ref.full_demod(y_all, chunk)
        ref.close()
        mx = make()
        mx.set_device_rate(L, N, taps, 15)
        got = mx.full_demod(x, chunk)
        mx.close()
        assert np.array_equal(got, want), (name, "chunked")
    # the rx_sdr host entry's one call of the whole stream runs in host groups of its own
    if fam == "sdr":
        g, _ = drs.sdr_host_group(L, N, M, len(_subset(tuned)) if kind != "single" else len(tuned), 4)
        assert drs.host_groups_crossed(n, g) >= 2, (name, g)
    if kind != "single":
        # an rx_fm read of at most 131072 capture samples holds fewer frames than a group, but at 61.44 M's raster
        rows = info["group"] * M if kind == "raster" else info["G"] * info["M1"]
        assert crossed["whole"] >= 2 if fam == "sdr" or rows < FM_READ else crossed["whole"] == 1, (name, crossed)
        assert fam == "sdr" or crossed["chunked"] >= 2, (name, crossed)
    # spot-check the reference's resampler stage with the sparse model at the edges of the ragged cuts
    cuts = _cut_patterns(n, L, N, max(2000, R_dev // 3), fam)["ragged"]
    edges, n0 = [], 0
    for c in cuts:
        n0 += c
        edges.append(rsm.out_count(0, n0, L, N))
    a = drs.launch(L, N, J, 0, n, _sms(), ctas=False)
    idx = drs.check_indices(a["n_out"], a["U"], J, edges, every=4096)
    H = J
    ext = np.concatenate([np.zeros(2 * H, np.int16), x])
    assert np.array_equal(y_all.reshape(-1, 2)[idx], drs.sparse_outputs(ext, H, L, N, taps, 15, 0, idx))


# ---- d. rx_power
def _power_ref(pl, Rp, offs, dd, win, y):
    ref = power.PowerMix(pl, Rp, offs, dd, win)
    ref.accumulate(y)
    out = ref.read()
    ref.close()
    return out


@pytest.mark.parametrize("plan", ["fm100_wbfm_30.72M", "fm100_wbfm_61.44M"])
def test_power_call_over_several_pass_groups(plan):
    torch = fh.torch()
    _, _, _, L, N, J = _named(plan)
    taps = rs.lowpass(L, N, J)
    pl, win, Rp, offs, dd = pm.shape("fm_band")
    dd = (dd[0], power.ddc_lowpass(dd[0], 33, 15), 15)                  # a short filter: the groups are the point
    pas = dd[0] * pl.buf_len // 2
    per_group = drs.POWER_SCRATCH_BYTES // (pl.n_hops * pl.buf_len * 2)
    n_pass = per_group + 3
    assert drs.power_groups(n_pass, pl.n_hops, pl.buf_len)[1] == 2
    c = rs.in_len(L, N, 0, n_pass * pas)
    assert rsm.out_count(0, c, L, N) == n_pass * pas
    x = _stream(c, 41)
    d_x = torch.from_numpy(x).cuda()
    y, _ = _device_entry(L, N, taps, 15, 0, d_x, c)
    want = _power_ref(pl, Rp, offs, dd, win, y)
    for device in (False, True):
        mx = power.PowerMix(pl, Rp, offs, dd, win)
        mx.set_device_rate(L, N, taps, 15)
        if device:
            mx.accumulate_device(d_x.data_ptr(), x.size, sync=True)
        else:
            mx.accumulate(x)
        got = mx.read()
        mx.close()
        assert all(np.array_equal(u, v) for u, v in zip(got, want)), (plan, device)


def test_power_upsampling_whole_pass_cuts_by_search():
    """L > N: a device sample can emit two capture samples, so in_len is the least call and may overshoot a whole
    pass; the cuts are found by search, and a cut one sample short is refused and changes nothing."""
    torch = fh.torch()
    L, N, J = 25, 21, 24
    taps = rs.lowpass(L, N, J)
    pl, win, Rp, offs, dd = pm.shape("fm_band")
    dd = (dd[0], power.ddc_lowpass(dd[0], 33, 15), 15)
    pas = dd[0] * pl.buf_len // 2
    cuts, n0, k = [], 0, 1
    while len(cuts) < 4:
        c = rs.in_len(L, N, n0, k * pas)
        while rsm.out_count(n0, c, L, N) % pas:                        # the least whole-pass cut at or past in_len
            c += 1
        assert rsm.out_count(n0, c - 1, L, N) % pas != 0
        cuts.append(c)
        n0 += c
        k = k % 3 + 1
    assert any(rsm.out_count(a, rs.in_len(L, N, a, k), L, N) > k for a in range(50) for k in range(1, 30))
    x = _stream(n0, 43)
    d_x = torch.from_numpy(x).cuda()
    y, _ = _device_entry(L, N, taps, 15, 0, d_x, n0)
    want = _power_ref(pl, Rp, offs, dd, win, y)
    for device in (False, True):
        mx = power.PowerMix(pl, Rp, offs, dd, win)
        mx.set_device_rate(L, N, taps, 15)
        at = 0
        for i, c in enumerate(cuts):
            if i == 2:
                with pytest.raises(_lib.Rxb200Error) as e:
                    if device:
                        mx.accumulate_device(d_x.data_ptr() + 4 * at, 2 * (c - 1), sync=True)
                    else:
                        mx.accumulate(x[2 * at:2 * (at + c - 1)])
                assert e.value.code == _lib.EUNSUPPORTED
            if device:
                mx.accumulate_device(d_x.data_ptr() + 4 * at, 2 * c, sync=True)
            else:
                mx.accumulate(x[2 * at:2 * (at + c)])
            at += c
        got = mx.read()
        mx.close()
        assert all(np.array_equal(u, v) for u, v in zip(got, want)), device


# ---- e. past 2^32 device samples
E_PLAN = (21, 25, 24)
E_BASE = (1 << 26) + 12345                      # device samples per call: 9 mod 25, so each call starts at a new phase
E_DEVICE = rsm.ceil_div((1 << 32) * 25, 21) + 2 * E_BASE   # both counts past 2^32 before the last call


def _capture_context(L, N, taps, base_dev, n_end, s):
    """Capture samples [s, ceil(n_end L / N)) of the device stream that repeats base_dev (a CUDA tensor holding two
    periods), through the stateless resampler from a device count early enough that every one of them is exact."""
    torch = fh.torch()
    J = taps.size // L
    B = base_dev.numel() // 4
    D = s * N // L - (J - 1) - 1
    n = n_end - D
    idx = torch.arange(D % B, D % B + n, device="cuda", dtype=torch.int64) % B
    src = base_dev.view(-1, 2)[idx].reshape(-1).contiguous()
    y, tail = _device_entry(L, N, taps, 15, D, src, n)
    assert np.all(tail == GUARD)
    m0 = rsm.ceil_div(D * L, N)
    assert m0 <= s
    return y[2 * (s - m0):]


def test_sdr_handle_past_2_32_samples():
    torch = fh.torch()
    L, N, J = E_PLAN
    taps = rs.lowpass(L, N, J)
    R, M = 2_016_000, 8
    off = 252_001
    dd = (M, power.ddc_lowpass(M, 65, 15), 15)
    base = _stream(E_BASE, 51)
    d_base = torch.from_numpy(np.concatenate([base, base])).cuda()
    mx = sdr.SdrMix(R, [off], ddc=dd)
    mx.set_device_rate(L, N, taps, 15)
    cap = rsm.out_count(0, E_BASE, L, N) // M + 2
    d_out = torch.zeros(2 * cap, dtype=torch.int16, device="cuda")
    n0, calls = 0, 0
    while n0 + E_BASE <= E_DEVICE:
        got = mx.process_device(d_base.data_ptr(), 2 * E_BASE, sdr.OUT_CS16, d_out.data_ptr(), cap, cap, sync=0)
        n0 += E_BASE
        calls += 1
    # the last call: device samples [n0, n0 + E_BASE), capture samples [P, P_end)
    P = rsm.ceil_div(n0 * L, N)
    got = mx.process_device(d_base.data_ptr(), 2 * E_BASE, sdr.OUT_CS16, d_out.data_ptr(), cap, cap, sync=1)
    n_end = n0 + E_BASE
    P_end = rsm.ceil_div(n_end * L, N)
    assert n0 > 1 << 32 and P > 1 << 32 and calls == E_DEVICE // E_BASE
    assert got == P_end // M - P // M
    last = d_out[:2 * got].cpu().numpy()
    mx.close()
    # the stateless rule at those counts: the resampler, then the NCO DDC at capture phase s with T - 1 of context
    T = dd[1].size
    s = (P - (T - 1)) // M * M
    ycap = _capture_context(L, N, taps, d_base, n_end, s)
    d_y = torch.from_numpy(ycap).cuda()
    k = (ycap.size // 2) // M
    d_d = torch.zeros(2 * k + 2, dtype=torch.int16, device="cuda")
    power.power_ddc_device(R, off, s, dd, d_y.data_ptr(), ycap.size // 2, d_d.data_ptr())
    torch.cuda.synchronize()
    want = d_d.cpu().numpy()[:2 * k]
    assert P_end // M - s // M == k
    assert np.array_equal(last, want[2 * (k - got):])


def test_power_handle_past_2_32_samples():
    torch = fh.torch()
    L, N, J = E_PLAN
    taps = rs.lowpass(L, N, J)
    pl, win, Rp, offs, dd = pm.shape("fm_band")
    M = dd[0]
    dd = (M, power.ddc_lowpass(M, 33, 15), 15)
    pas = M * pl.buf_len // 2
    base = _stream(E_BASE, 53)
    d_base = torch.from_numpy(np.concatenate([base, base])).cuda()
    kp = rsm.out_count(0, E_BASE, L, N) // pas - 1                    # passes per call
    mx = power.PowerMix(pl, Rp, offs, dd, win)
    mx.set_device_rate(L, N, taps, 15)
    n0, calls = 0, 0
    while True:
        c = rs.in_len(L, N, n0, kp * pas)
        assert c <= E_BASE
        last = n0 > E_DEVICE - E_BASE
        if last:
            torch.cuda.synchronize()
            mx.reset_accumulators()
        mx.accumulate_device(d_base.data_ptr() + 4 * (n0 % E_BASE), 2 * c, sync=last)
        if last:
            break
        n0 += c
        calls += 1
    P = rsm.ceil_div(n0 * L, N)
    n_end = n0 + c
    assert n0 > 1 << 32 and P > 1 << 32 and P % pas == 0 and P // pas == calls * kp
    got = mx.read()
    mx.close()
    T = dd[1].size
    s = (P - (T - 1)) // M * M
    ycap = _capture_context(L, N, taps, d_base, n_end, s)
    assert ycap.size // 2 == rsm.ceil_div(n_end * L, N) - s == P - s + kp * pas
    d_y = torch.from_numpy(ycap).cuda()
    k = (ycap.size // 2) // M
    bl = pl.buf_len
    bufs = torch.zeros((kp, pl.n_hops, bl), dtype=torch.int16, device="cuda")
    d_d = torch.zeros(2 * k + 2, dtype=torch.int16, device="cuda")
    for i, f in enumerate(offs):
        power.power_ddc_device(Rp, f, s, dd, d_y.data_ptr(), ycap.size // 2, d_d.data_ptr())
        torch.cuda.synchronize()
        tail = d_d[2 * k - kp * bl:2 * k]
        bufs[:, i, :] = tail.reshape(kp, bl)
    torch.cuda.synchronize()
    sc = power.PowerScanner(pl, win)
    sc.scanner_device(bufs.data_ptr(), kp, sync=True)
    want = sc.read()
    sc.close()
    assert all(np.array_equal(u, v) for u, v in zip(got, want))


def _nvml_used():
    """{pid: device memory} of the compute processes NVML lists on device 0."""
    import pynvml
    torch = fh.torch()
    torch.cuda.synchronize()
    pynvml.nvmlInit()
    try:
        dev = pynvml.nvmlDeviceGetHandleByUUID("GPU-" + str(torch.cuda.get_device_properties(0).uuid))
        return {p.pid: p.usedGpuMemory for p in pynvml.nvmlDeviceGetComputeRunningProcesses(dev)}
    finally:
        pynvml.nvmlShutdown()


def _own_nvml_pid():
    """This process's entry in NVML's per-process list.  In a PID namespace NVML's pid need not be os.getpid(), so the
    entry is the one that grows by a 64 MiB probe allocation (this process's pid first, when it is among them)."""
    import os
    torch = fh.torch()
    torch.cuda.empty_cache()                                            # the probe is a fresh cudaMalloc
    before = _nvml_used()
    probe = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    after = _nvml_used()
    del probe
    torch.cuda.empty_cache()
    grew = [p for p, v in after.items()
            if v is not None and (64 << 20) <= v - (before.get(p) or 0) <= (72 << 20)]
    if os.getpid() in grew:
        return os.getpid()
    assert len(grew) == 1, ("NVML shows no single entry for this process", before, after)
    return grew[0]


def _process_device_bytes(pid):
    """The device memory this process holds on device 0, as NVML counts it per process: unlike the device's free
    memory, other processes on the same GPU do not move it."""
    v = _nvml_used().get(pid)
    assert v is not None, "NVML does not list this process's device memory"
    return int(v)


def test_sdr_host_groups_fit_the_scratch_bytes():
    """A host call of three groups grows the handle's device memory by what one group stages, within
    RXB200_SDR_MIX_SCRATCH_BYTES: host_group counts the device-rate upload and the resampled capture, not only the
    rows (one channel, CS16, 21/25 at M = 8: groups of 8 625 817 device samples).  Without the resampler term a group
    would stage about 111 MiB."""
    torch = fh.torch()
    L, N, J = E_PLAN
    taps = rs.lowpass(L, N, J)
    M = 8
    g, _ = drs.sdr_host_group(L, N, M, 1, 4)
    x = _stream(3 * g + 1001, 61)
    mx = sdr.SdrMix(2_016_000, [252_000], ddc=(M, power.ddc_lowpass(M, 65, 15), 15))
    mx.set_device_rate(L, N, taps, 15)
    mx.process(x[:2000])
    pid = _own_nvml_pid()
    used0 = _process_device_bytes(pid)
    got = mx.process(x[2000:])
    used1 = _process_device_bytes(pid)
    mx.close()
    assert got.shape[1] > 0 and drs.host_groups_crossed(x.size // 2 - 1000, g) >= 3
    assert 0 < used1 - used0 <= drs.SDR_SCRATCH_BYTES + (6 << 20), (used1 - used0)
