"""The restated launch rules of the raster and two-stage channelizers (tests/channelizer_scale.py) at the numbers the
repository states and at every case of tests/test_fm_channelizer_scale_gpu.py for both H100 SM counts, the sparse
models against fm_raster.raster_model and fm_two_stage.two_stage_model, and the bounds the exactness captures reach,
on the CPU."""
import numpy as np
import pytest

import channelizer_scale as cs
import fm_raster as frs
import fm_two_stage as fts
import mix_scale as ms


# ---- the sparse models against the models the goldens pin -------------------------------------------------------
RASTER_CASES = [  # (K, bins, M, T, S)
    (3, [0, 1, 2, 2], 3, 17, 33),
    (4, [3, 0], 7, 5, 19),
    (12, [11, 5, 0, 5], 5, 29, 30),
    (48, [47, 1, 24], 64, 13, 28),
    (100, [0, 99, 33], 1, 201, 31),
    (768, [408, 767, 0], 16, 1, 14),
]


def _taps(T, seed):
    rng = np.random.default_rng(seed)
    h = rng.integers(-(1 << 22) // T, (1 << 22) // T, size=T)
    h[0] = h[0] or 1
    return h.astype(np.int32)


@pytest.mark.parametrize("K,bins,M,T,S", RASTER_CASES)
def test_raster_sparse_equals_the_model(K, bins, M, T, S):
    rng = np.random.default_rng(K + M + T)
    taps = _taps(T, K * T)
    x = rng.integers(-32768, 32768, size=2 * (40 * M + 11)).astype(np.int16)
    hist = rng.integers(-32768, 32768, size=2 * (T - 1)).astype(np.int16)
    for pos, h, phase in ((0, None, 0), (5, hist, None), (M - 1, hist, ((1 << 64) - 5) % K), (123456789, None, 7)):
        want, _ = frs.raster_model(x, K, bins, taps, M, S, pos, h, phase)
        p0 = pos % K if phase is None else phase
        got = cs.raster_sparse(x, K, bins, taps, M, S, p0, pos, h)
        assert got.shape == want.shape and np.array_equal(got, want), (pos, phase)
        n = want.shape[1] // 2
        frames = sorted({0, n - 1, n // 2, 3, n - 4})
        sub = cs.raster_sparse(x, K, bins, taps, M, S, p0, pos, h, frames=frames, block=97)
        cols = np.array([[2 * f, 2 * f + 1] for f in frames]).reshape(-1)
        assert np.array_equal(sub, want[:, cols]), (pos, phase)


@pytest.mark.parametrize("name", ["raw_sat_k3", "raw_sat_k4096", "am_m100", "raw_centres_edges"])
def test_two_stage_sparse_equals_the_model(name):
    _, rate, K, offs, coarse, fine, x, _ = fts.case_input(name, seed=3)
    M = coarse[0] * fine[0]
    x = x[:2 * (40 * M + 7)]
    for n0 in (0, (1 << 64) - K + 1, (1 << 40) + 3):
        want = fts.two_stage_model(x, rate, K, offs, coarse, fine, n0)
        assert np.array_equal(cs.two_stage_sparse(x, rate, K, offs, coarse, fine, n0), want), (name, n0)
        sub = [len(offs) - 1, 0]
        assert np.array_equal(cs.two_stage_sparse(x, rate, K, offs, coarse, fine, n0, channels=sub), want[sub])


def test_split_reads():
    y = np.arange(2 * 10, dtype=np.int16)
    parts = cs.split_reads(y, [2 * 3, 2 * 1, 2 * 20, 2 * 7], 3)
    assert [p.size for p in parts] == [2, 0, 14, 4]
    assert np.array_equal(np.concatenate(parts), y)


# ---- the rules at the numbers the repository states ------------------------------------------------------------
def test_raster_plan():
    assert cs.raster_plan(4096, 5)[2] == 1024                              # DESIGN 4.4: 1 024 frames at K = 4096
    assert cs.raster_plan(768, 5)[2] == 5440                               # and 5 440 at K = 768
    assert cs.raster_plan(8, 8)[2] == 524288
    assert cs.raster_plan(3, 1)[:2] == (16, 64) and cs.raster_plan(100, 33)[:2] == (208, 128)


def test_two_stage_plan():
    offs = [1000 * k - 2_000_000 + 7 for k in range(4000)]                 # test_long_call_equals_short_calls
    bins = [fts.bin_word(4_096_000, 4096, 1, f)[0] for f in offs]
    slots, rows, G = cs.two_stage_plan(4096, bins, 8192)
    assert len(slots) == 4000 and len(rows) == 4000 and G == 64
    slots, rows, G = cs.two_stage_plan(4096, list(range(8)), 8192)
    assert G == 960
    slots, rows, G = cs.two_stage_plan(32, [5, 1, 5, 1, 9], 129)
    assert slots == [1, 5, 9] and rows == [(0, 0, 2), (1, 2, 2), (2, 4, 1)]


def test_branch_regime():
    # T = 8192: one frame per CTA; the short tests share at most a few hundred frames out
    assert cs.branch_regime(65536, 1, 8192, 132)[:2] == (1, "span")
    assert cs.branch_regime(65536, 1, 5, 132)[:2] == (249, "n_out")
    assert cs.branch_regime(10, 7, 129, 132) == (1, "n_out", (129 + 129 + 1) * 4)


def test_fine_rows_rule():
    assert ms.ddc_ctas(8, 132) == 264 and ms.ddc_ctas(8, 132, rows=6) == 44
    assert ms.ddc_ctas(300, 132, rows=264) == 1 and ms.ddc_ctas(300, 132, rows=263) == 2
    assert ms.ddc_regime(1000, 4, 129, 300, 132, rows=265) == (1000, "n_out")


# ---- every GPU case lands in the regime it claims, for both SM counts --------------------------------------------
def test_column_tile_cases():
    F = cs.COLUMN_TILE_FRAMES
    assert F > 64 and F % 64
    cases = cs.column_tile_cases()
    tiles = {name: cs.raster_plan(K, len(bins))[1] // cs.RAS_BN for name, (K, bins) in cases.items()}
    assert tiles == {"k768_all": 24, "k100_c33": 2, "k4096_c1000": 32, "k12_twice": 1}
    K, bins = cases["k768_all"]
    assert sorted(bins) == list(range(768))
    K, bins = cases["k100_c33"]
    assert len(set(bins)) == 33 and (2 * 33) % 64
    K, bins = cases["k4096_c1000"]
    assert len(bins) == 1000 and len(set(bins)) < 1000 and (2 * 1000) % 64
    assert sorted(cases["k12_twice"][1]) == sorted(list(range(12)) * 2)
    for K, bins in cases.values():
        assert F <= cs.raster_plan(K, len(bins))[2]
    assert cs.tile_channels(768, 1, extra=0) == sorted({t for t in range(0, 768, 32)} | {t + 31 for t in range(0, 768, 32)})


@pytest.mark.parametrize("n_sm", cs.H100_SMS)
def test_grid_row_split_cases(n_sm):
    offs = cs.split_offsets()
    bins = [fts.bin_word(cs.SPLIT_RATE, cs.SPLIT_K, 4, f)[0] for f in offs]
    assert sorted(bins.count(b) for b in set(bins)) == [1, 257, 600]
    assert len(set(offs)) == len(offs)
    slots, rows, _ = cs.two_stage_plan(cs.SPLIT_K, bins, 129)
    assert slots == [3, 7, 12]
    assert rows == [(0, 0, 256), (0, 256, 256), (0, 512, 88), (1, 600, 1), (2, 601, 256), (2, 857, 1)]
    offs = cs.many_rows_offsets(n_sm)
    bins = [fts.bin_word(4_096_000, 4096, 1, f)[0] for f in offs]
    slots, rows, _ = cs.two_stage_plan(4096, bins, 33)
    assert len(rows) == len(slots) > 2 * n_sm and len(offs) > len(slots)
    assert ms.ddc_ctas(len(offs), n_sm, rows=len(rows)) == 1


def test_group_shorter_than_history_cases():
    bins = [fts.bin_word(cs.GROUP_RATE, cs.GROUP_K, 1, f)[0] for f in cs.GROUP_OFFSETS]
    slots, _, G = cs.two_stage_plan(cs.GROUP_K, bins, 8192)
    assert len(slots) == 8 and G == 960 < 8191
    phases = cs.group_reads_phases(cs.GROUP_READS, G, 7)
    assert {ph for ph, crosses in phases if crosses} == set(range(7))
    assert sum(cs.GROUP_READS) // 2 > 6 * G


@pytest.mark.parametrize("n_sm", cs.H100_SMS)
@pytest.mark.parametrize("M,T", cs.SPAN_SHAPES)
def test_span_bound_cases(M, T, n_sm):
    F = cs.span_frames(M, T, n_sm)
    U, which, smem = cs.branch_regime(F, M, T, n_sm)
    assert which == "span" and U == cs.branch_span(M, T) and F > 2 * n_sm * (U - 1)
    assert -(-F // U) == 2 * n_sm + 1 and F % U == 37                    # the last CTA holds 37 frames
    assert F <= cs.raster_plan(cs.SPAN_K, cs.SPAN_K)[2]                   # one scratch group
    if T > M:
        assert U > 1600 and 64 * 1024 <= smem <= 65 * 1024                 # about 64 KiB of staging
    elif T < M:
        assert U >= 100
    else:
        assert T == M


def test_groups_case():
    F = cs.groups_frames()
    group = cs.raster_plan(cs.GROUPS_K, len(cs.GROUPS_BINS))[2]
    assert group == 1024 and F > 5 * group
    assert cs.GROUPS_T > cs.GROUPS_M > 1


# ---- the exactness captures ------------------------------------------------------------------------------------
def _sums(x, K, taps, M, phase, n_frames):
    T = taps.size
    ext = np.concatenate([np.zeros(2 * (T - 1), np.int16), x[:2 * n_frames * M]])
    return frs.branch_sums(ext, taps, M, K, (phase - (T - 1)) % K, n_frames)


@pytest.mark.parametrize("K", cs.BOUND_KS)
def test_bound_captures(K):
    k, taps, M = cs.bound_case(K)
    assert frs.sum_abs(taps) == (1 << 22) - 1
    tw = frs.table(K).astype(np.int64)
    if K > 3:
        assert all(np.array_equal(tw[(r + K // 2) % K], -tw[r]) for r in range(K))   # what the cancellation needs
    n = 12
    phase = ((1 << 64) - 5) % K
    x = cs.bound_capture(K, n, phase, K, aligned=False)
    assert (x == -32768).any()
    v = _sums(x, K, taps, M, phase, n)
    mag = np.hypot(v[..., 0].astype(np.float64), v[..., 1].astype(np.float64))
    assert (mag.max(axis=1) >= 2.0 ** 36).all()
    twm = np.hypot(*tw[(k * np.arange(K)) % K].T.astype(np.float64))
    assert ((mag * twm).sum(axis=1) >= 2.0 ** 52).all()
    A = frs.dft(v, K, [k])[0]
    assert np.abs(A).max() < (1 << 15)
    want, _ = frs.raster_model(x[:2 * n * M], K, [k, 1], taps, M, 0, phase=phase)
    assert np.array_equal(want[0].reshape(-1, 2), A)                         # S = 0 shows every bit of A
    assert np.array_equal(cs.raster_sparse(x[:2 * n * M], K, [k, 1], taps, M, 0, phase), want)
    x = cs.bound_capture(K, n, phase, K + 1, aligned=True)
    A = frs.dft(_sums(x, K, taps, M, phase, n), K, [1])[0]
    assert np.abs(A[:, 0]).max() >= 1 << 52
    y = (A[:, 0] + (1 << 36)) >> 37
    assert (np.abs(y) > 32767).any() and (np.abs(y) <= 32767).any()        # S = 37 crosses the saturation edge
    for S in (36, 37, 38):
        want, _ = frs.raster_model(x[:2 * n * M], K, [1, k], taps, M, S, phase=phase)
        assert np.array_equal(cs.raster_sparse(x[:2 * n * M], K, [1, k], taps, M, S, phase), want), S
