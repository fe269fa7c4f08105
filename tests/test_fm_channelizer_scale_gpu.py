"""The raster and two-stage channelizers at the bin counts, channel counts and lengths of real captures, where their
launch rules leave the corner every short call lands in (tests/channelizer_scale.py restates the rules; each case
asserts the regime it claims):

  a. rxb200_raster_device with 24 to 32 DFT column tiles, partial column tiles and repeated bins, over several row
     tiles; and a raster handle at the DESIGN operating point with all 768 channels;
  b. rxb200_two_stage_device with a bin of 600 channels (three fine grid rows), one of 257 and one of 1, and with more
     than 2 n_sm grid rows (one CTA per row); the 600-channel layout through a handle;
  c. coarse groups shorter than the fine history (G = 960 < T2 - 1): the stateless entry over six groups and more, a
     handle whose reads cross group boundaries at every fine decimation phase, and the 4000-bin G = 64 shape;
  d. raster_branch_kernel with U set by the staging room: T = M, T < M and T > M with about 64 KiB of shared memory;
  e. a raster handle over five scratch groups with T > M > 1, in one read and in reads at every phase of M;
  f. sums at the exactness bound: terms near 2^52 that cancel to |A| < 2^15 at S = 0, and |A| >= 2^52 at the shifts
     where the output crosses the saturation edge, through the raster entry and the two-stage coarse stage.

The kernels alone are compared bit for bit with the sparse models, with a guard past every output buffer that must stay
zero; the handles with the port on the models' decimated streams."""
import numpy as np
import pytest

import channelizer_scale as cs
import fm_any_chunk as fac
import fm_ddc as fdd
import fm_handles as fh
import fm_two_stage as fts
import mix_scale as ms
from rx_tools_b200 import fm

pytestmark = pytest.mark.gpu

GUARD = 64              # int16 past the last output that must stay zero
RAW = fac.with_(fac.RAW, downsample=1, offset_tuning=1)


def _capture(n_complex, seed):
    """A random full-range capture of n_complex samples, generated on the device."""
    torch = fh.torch()
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(-32768, 32768, (2 * n_complex,), dtype=torch.int16, device="cuda", generator=g)


def _taps(T, seed, bound=1 << 22):
    """Random taps with sum |h| below bound, and the shift that brings a raster sum's typical output near 2^13."""
    rng = np.random.default_rng(seed)
    h = rng.integers(-(bound // T) + 1, bound // T, size=T)            # sum |h| < bound
    h[0] = h[0] or 1
    shift = 17 + int(np.ceil(np.log2(np.sqrt(T) * (np.abs(h).mean() + 1))))
    return h.astype(np.int32), shift


def _check(dst, want, what):
    """dst holds want (int16[C][2 F]) then a zero guard."""
    got = dst[:want.size].cpu().numpy().reshape(want.shape)
    bad = np.argwhere(got != want)
    assert bad.size == 0, (what, bad.shape[0], bad[:4])
    assert not dst[want.size:].any().item(), what


def _port_compare(port, p, got, y, lens16, M, what):
    """A handle's PCM of one channel against the port on the model's whole decimated stream y split by the reads."""
    dec, lens = fdd.nonempty(cs.split_reads(y, lens16, M))
    fh.compare(p, got, fac.port_run_seq(port, p, dec, lens), what)


def _run_ops(mx, x, ops):
    """("read", n16) through process_read, ("chunk", n16, chunk16) through full_demod: (PCM, the chain's read lengths
    per op as capture int16 lengths for split_reads)."""
    out, lens, at = [], [], 0
    for op in ops:
        part = x[at:at + op[1]]
        if op[0] == "read":
            out.append(mx.process_read(part))
            lens.append(op[1])
        else:
            out.append(mx.full_demod(part, op[2]))
            lens += [min(op[2], op[1] - a) for a in range(0, op[1], op[2])]
        at += op[1]
    return np.concatenate(out, axis=1), lens


# ---- a. DFT column tiles ----------------------------------------------------------------------------------------
TILE_SHAPES = {"k768_all": (8, 65), "k100_c33": (3, 201), "k4096_c1000": (8, 33), "k12_twice": (5, 29)}   # (M, T)


@pytest.mark.parametrize("name", sorted(TILE_SHAPES))
def test_raster_device_column_tiles(name):
    torch = fh.torch()
    K, bins = cs.column_tile_cases()[name]
    M, T = TILE_SHAPES[name]
    F = cs.COLUMN_TILE_FRAMES
    Kp, Np, group = cs.raster_plan(K, len(bins))
    assert F > 64 and F % 64 and F <= group and Np // cs.RAS_BN >= (24 if len(bins) >= 768 else 1)
    taps, S = _taps(T, K + T)
    n = F * M + M - 1
    x = _capture(n, K * 3 + len(bins))
    dst = torch.zeros(len(bins) * 2 * F + GUARD, dtype=torch.int16, device="cuda")
    for n0 in ((1 << 64) - K + 1, (1 << 40) + 3):
        dst.zero_()
        fm.raster_device(K, bins, n0, (M, taps, S), x.data_ptr(), n, dst.data_ptr())
        torch.cuda.synchronize()
        _check(dst, cs.raster_sparse(x, K, bins, taps, M, S, n0 % K), (name, n0))


def test_raster_handle_design_point(port):
    """19.2 Msps, K = 768, M = 64, T = 257 into a D = 12 lut chain, all 768 bins as channels, over a read of two
    scratch groups and ragged reads; the first and last channel of every column tile and seeded others against the
    port."""
    torch = fh.torch()
    K, M = 768, 64
    taps, S = fdd.lowpass(257, 12500 / 19.2e6), 30
    bins = cs.column_tile_cases()["k768_all"][1]
    group = cs.raster_plan(K, K)[2]
    reads = [2 * (group * M + 7001)] + fdd.READS_LONG
    assert reads[0] // 2 // M > group
    x = np.random.default_rng(768).integers(-32768, 32768, size=sum(reads)).astype(np.int16)
    mx = fm.FmMix(fdd.NBFM12, ddc=(M, taps, S), raster=(K, bins))
    got, _ = fh.reads(mx, x, reads)
    mx.close()
    check = cs.tile_channels(K, 768)
    y = cs.raster_sparse(torch.from_numpy(x).cuda(), K, [bins[c] for c in check], taps, M, S, 0)
    for i, c in enumerate(check):
        _port_compare(port, fdd.NBFM12, got[c], y[i], reads, M, ("design", c))


# ---- b. fine grid-row split --------------------------------------------------------------------------------------
SPLIT_COARSE = (4,) + _taps(33, 33)
SPLIT_FINE = (4, _taps(129, 129, 1 << 20)[0], 19)


def _order(offs, M1, rate, K):
    bins = [fts.bin_word(rate, K, M1, f)[0] for f in offs]
    return sorted(range(len(offs)), key=lambda c: bins[c]), bins


def test_two_stage_device_grid_row_split():
    torch = fh.torch()
    rate, K, offs = cs.SPLIT_RATE, cs.SPLIT_K, cs.split_offsets()
    order, bins = _order(offs, SPLIT_COARSE[0], rate, K)
    _, rows, _ = cs.two_stage_plan(K, bins, SPLIT_FINE[1].size)
    assert [nc for _, _, nc in rows] == [256, 256, 88, 1, 256, 1]
    M = SPLIT_COARSE[0] * SPLIT_FINE[0]
    n_out = 1500
    n = n_out * M + M - 1
    x = _capture(n, 600)
    dst = torch.zeros(len(offs) * 2 * n_out + GUARD, dtype=torch.int16, device="cuda")
    n0 = (1 << 40) + 3
    fm.two_stage_device(rate, K, offs, n0, SPLIT_COARSE, SPLIT_FINE, x.data_ptr(), n, dst.data_ptr())
    torch.cuda.synchronize()
    _check(dst, cs.two_stage_sparse(x, rate, K, offs, SPLIT_COARSE, SPLIT_FINE, n0), "split")


def test_two_stage_handle_grid_row_split(port):
    rate, K, offs = cs.SPLIT_RATE, cs.SPLIT_K, cs.split_offsets()
    order, bins = _order(offs, SPLIT_COARSE[0], rate, K)
    _, rows, _ = cs.two_stage_plan(K, bins, SPLIT_FINE[1].size)
    M = SPLIT_COARSE[0] * SPLIT_FINE[0]
    ops = [("read", 2 * 5003), ("chunk", 2 * M * 300, 2 * M * 100), ("read", 2 * 37), ("read", 2 * (M * 211 + 3)),
           ("chunk", 2 * M * 64, 2 * M * 64)]
    x = np.random.default_rng(601).integers(-32768, 32768, size=sum(op[1] for op in ops)).astype(np.int16)
    mx = fm.FmMix(RAW, rate, offs, two_stage=(K, SPLIT_COARSE, SPLIT_FINE))
    got, lens = _run_ops(mx, x, ops)
    mx.close()
    check = sorted({order[c] for _, c0, nc in rows for c in (c0, c0 + nc - 1)})
    y = cs.two_stage_sparse(fh.torch().from_numpy(x).cuda(), rate, K, offs, SPLIT_COARSE, SPLIT_FINE, channels=check)
    for i, c in enumerate(check):
        _port_compare(port, RAW, got[c], y[i], lens, M, ("split handle", c))


def test_two_stage_device_one_cta_per_row():
    torch = fh.torch()
    n_sm = ms.device_sms()
    rate, K = 4_096_000, 4096
    offs = cs.many_rows_offsets(n_sm)
    coarse, fine = (1,) + _taps(5, 5), (2, _taps(33, 34, 1 << 20)[0], 19)
    bins = [fts.bin_word(rate, K, 1, f)[0] for f in offs]
    _, rows, _ = cs.two_stage_plan(K, bins, 33)
    assert len(rows) > 2 * n_sm and ms.ddc_ctas(len(offs), n_sm, rows=len(rows)) == 1
    n_out = 2000
    n = 2 * n_out + 1
    x = _capture(n, 271)
    dst = torch.zeros(len(offs) * 2 * n_out + GUARD, dtype=torch.int16, device="cuda")
    fm.two_stage_device(rate, K, offs, 77, coarse, fine, x.data_ptr(), n, dst.data_ptr())
    torch.cuda.synchronize()
    check = sorted({0, len(offs) - 1} | {int(c) for c in np.random.default_rng(n_sm).choice(len(offs), 48, False)})
    want = cs.two_stage_sparse(x, rate, K, offs, coarse, fine, 77, channels=check)
    got = dst[:len(offs) * 2 * n_out].cpu().numpy().reshape(len(offs), -1)
    for i, c in enumerate(check):
        assert np.array_equal(got[c], want[i]), c
    assert not dst[len(offs) * 2 * n_out:].any().item()


# ---- c. coarse groups shorter than the fine history ---------------------------------------------------------------
GROUP_COARSE = (1,) + _taps(5, 4096)
GROUP_FINE = (7, _taps(8192, 7, 1 << 20)[0], 19)


def _group_plan():
    bins = [fts.bin_word(cs.GROUP_RATE, cs.GROUP_K, 1, f)[0] for f in cs.GROUP_OFFSETS]
    G = cs.two_stage_plan(cs.GROUP_K, bins, GROUP_FINE[1].size)[2]
    assert G == 960 < GROUP_FINE[1].size - 1
    return G


def test_two_stage_device_groups_shorter_than_history():
    torch = fh.torch()
    G = _group_plan()
    n = 6 * G + 517
    assert (n // 7) * 7 > 6 * G
    x = _capture(n, 960)
    offs = cs.GROUP_OFFSETS
    dst = torch.zeros(len(offs) * 2 * (n // 7) + GUARD, dtype=torch.int16, device="cuda")
    for n0 in (0, (1 << 64) - 3):
        dst.zero_()
        fm.two_stage_device(cs.GROUP_RATE, cs.GROUP_K, offs, n0, GROUP_COARSE, GROUP_FINE, x.data_ptr(), n,
                            dst.data_ptr())
        torch.cuda.synchronize()
        _check(dst, cs.two_stage_sparse(x, cs.GROUP_RATE, cs.GROUP_K, offs, GROUP_COARSE, GROUP_FINE, n0), n0)


def test_two_stage_handle_groups_shorter_than_history(port):
    G = _group_plan()
    reads = cs.GROUP_READS
    assert {ph for ph, crosses in cs.group_reads_phases(reads, G, 7) if crosses} == set(range(7))
    x = np.random.default_rng(961).integers(-32768, 32768, size=sum(reads)).astype(np.int16)
    offs = cs.GROUP_OFFSETS
    mx = fm.FmMix(RAW, cs.GROUP_RATE, offs, two_stage=(cs.GROUP_K, GROUP_COARSE, GROUP_FINE))
    got, _ = fh.reads(mx, x, reads)
    mx.close()
    y = cs.two_stage_sparse(fh.torch().from_numpy(x).cuda(), cs.GROUP_RATE, cs.GROUP_K, offs, GROUP_COARSE, GROUP_FINE)
    for c in range(len(offs)):
        _port_compare(port, RAW, got[c], y[c], reads, 7, ("groups handle", c))


def test_two_stage_device_4000_bins():
    """The 4000-bin shape of test_long_call_equals_short_calls (G = 64, each bin its own grid row) through the
    stateless entry: the first and last channel of every 32-bin column tile and 64 seeded channels."""
    torch = fh.torch()
    rate, K = 4_096_000, 4096
    offs = [1000 * k - 2_000_000 + 7 for k in range(4000)]
    rng = np.random.default_rng(3)
    fine_taps = rng.integers(-(1 << 18) // 8192, (1 << 18) // 8192, size=8192, endpoint=False)
    fine_taps[0] = fine_taps[0] or 1
    coarse, fine = (1, np.array([7, -3, 11, 2, -9], np.int32), 19), (2, fine_taps.astype(np.int32), 15)
    bins = [fts.bin_word(rate, K, 1, f)[0] for f in offs]
    _, rows, G = cs.two_stage_plan(K, bins, 8192)
    assert G == 64 and len(rows) == 4000
    n = 6000
    x = torch.from_numpy(fh.every_int16(9)[:2 * n]).cuda()
    dst = torch.zeros(len(offs) * n + GUARD, dtype=torch.int16, device="cuda")
    fm.two_stage_device(rate, K, offs, 12345, coarse, fine, x.data_ptr(), n, dst.data_ptr())
    torch.cuda.synchronize()
    check = cs.tile_channels(4000, 4000, extra=64)
    want = cs.two_stage_sparse(x, rate, K, offs, coarse, fine, 12345, channels=check)
    got = dst[:len(offs) * n].cpu().numpy().reshape(len(offs), -1)
    for i, c in enumerate(check):
        assert np.array_equal(got[c], want[i]), c
    assert not dst[len(offs) * n:].any().item()


# ---- d. branch kernel with U set by the staging room ---------------------------------------------------------------
@pytest.mark.parametrize("M,T", cs.SPAN_SHAPES)
def test_raster_device_span_bound(M, T):
    torch = fh.torch()
    n_sm = ms.device_sms()
    K = cs.SPAN_K
    bins = [5, 0, 7, 3, 1, 6, 2, 4]
    F = cs.span_frames(M, T, n_sm)
    U, which, smem = cs.branch_regime(F, M, T, n_sm)
    assert which == "span" and F <= cs.raster_plan(K, len(bins))[2]
    taps, S = _taps(T, M * 7 + T)
    n = F * M
    x = _capture(n, T)
    dst = torch.zeros(len(bins) * 2 * F + GUARD, dtype=torch.int16, device="cuda")
    n0 = (1 << 40) + 3
    fm.raster_device(K, bins, n0, (M, taps, S), x.data_ptr(), n, dst.data_ptr())
    torch.cuda.synchronize()
    if T <= 64:
        _check(dst, cs.raster_sparse(x, K, bins, taps, M, S, n0 % K), (M, T))
        return
    frames = {f for b in range(-(-F // U)) for f in (b * U, min(F, (b + 1) * U) - 1)}
    frames |= {int(f) for f in np.random.default_rng(T).choice(F, 4096, replace=False)}
    frames = sorted(frames)
    want = cs.raster_sparse(x, K, bins, taps, M, S, n0 % K, frames=frames)
    got = dst[:len(bins) * 2 * F].view(len(bins), F, 2)[:, frames].cpu().numpy().reshape(len(bins), -1)
    bad = np.argwhere(got != want)
    assert bad.size == 0, (M, T, U, bad[:4])
    assert not dst[len(bins) * 2 * F:].any().item()


# ---- e. raster handle over scratch groups with T > M > 1 ----------------------------------------------------------
def test_raster_handle_groups(port):
    K, M, T, bins = cs.GROUPS_K, cs.GROUPS_M, cs.GROUPS_T, cs.GROUPS_BINS
    taps, S = _taps(T, 129)
    n = cs.groups_frames() * M + 3
    x = np.random.default_rng(1024).integers(-32768, 32768, size=2 * n).astype(np.int16)
    one = fm.FmMix(RAW, ddc=(M, taps, S), raster=(K, bins))
    a = one.process_read(x)
    one.close()
    reads = [2 * 1031] * (n // 1031) + [2 * (n % 1031)]                   # 1031 = 2 mod 7: every phase of M
    assert {sum(reads[:i]) // 2 % M for i in range(len(reads))} == set(range(M))
    many = fm.FmMix(RAW, ddc=(M, taps, S), raster=(K, bins))
    b, _ = fh.reads(many, x, reads)
    many.close()
    assert a.tobytes() == b.tobytes()
    y = cs.raster_sparse(fh.torch().from_numpy(x).cuda(), K, bins, taps, M, S, 0)
    for c in range(len(bins)):
        _port_compare(port, RAW, a[c], y[c], [2 * n], M, ("one read", c))
        _port_compare(port, RAW, b[c], y[c], reads, M, ("reads", c))


# ---- f. sums at the exactness bound -----------------------------------------------------------------------------
@pytest.mark.parametrize("aligned", [False, True])
@pytest.mark.parametrize("K", cs.BOUND_KS)
def test_exactness_bound(K, aligned):
    """Through rxb200_raster_device and through rxb200_two_stage_device with a unit fine stage at bin centres, whose
    outputs are the coarse outputs: the cancelling capture at S = 0, the aligned one across the saturation edge."""
    torch = fh.torch()
    k, taps, M = cs.bound_case(K)
    F = cs.COLUMN_TILE_FRAMES
    n0 = (1 << 64) - 5
    xn = cs.bound_capture(K, F, n0 % K, K + aligned, aligned)
    x = torch.from_numpy(xn).cuda()
    n = F * M
    bins = sorted({k, 1, 0, K - 1, K // 2})
    rate = K * 6000
    ts_bins = [b for b in bins if 2 * b != K]
    offs = [(b if 2 * b < K else b - K) * 6000 for b in ts_bins]
    assert [fts.bin_word(rate, K, M, f) for f in offs] == [(b, 0) for b in ts_bins]
    unit = (1, np.ones(1, np.int32), 0)
    ra = torch.zeros(len(bins) * 2 * F + GUARD, dtype=torch.int16, device="cuda")
    tw = torch.zeros(len(offs) * 2 * F + GUARD, dtype=torch.int16, device="cuda")
    for S in ((36, 37, 38) if aligned else (0,)):
        ra.zero_()
        tw.zero_()
        fm.raster_device(K, bins, n0, (M, taps, S), x.data_ptr(), n, ra.data_ptr())
        fm.two_stage_device(rate, K, offs, n0, (M, taps, S), unit, x.data_ptr(), n, tw.data_ptr())
        torch.cuda.synchronize()
        want = cs.raster_sparse(x, K, bins, taps, M, S, n0 % K)
        _check(ra, want, (K, aligned, S, "raster"))
        _check(tw, cs.two_stage_sparse(x, rate, K, offs, (M, taps, S), unit, n0), (K, aligned, S, "two-stage"))
        _check(tw, want[[bins.index(b) for b in ts_bins]], (K, aligned, S, "two-stage = raster"))
        y = want[bins.index(1 if aligned else k)]
        if aligned and S == 37:
            sat = (y == 32767) | (y == -32768)
            assert sat.any() and not sat.all(), (K, S)
