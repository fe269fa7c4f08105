"""The resampler's launch rule restated (tests/device_rate_scale.py), without a GPU: over a seeded sweep of every
accepted (L, N, J), with the tops of the range L = 2^22 / J, the largest v the kernel's multiply-high sees stays below
2^31, no CTA stages more than RS_SPAN samples or more than the room it is given, and the shared memory fits the H100;
the multiply-high needs at most one correction for every v up to each L's worst; the sparse model equals the full one;
and rxb200_resample_in_len is the least call for L > N too, where it need not be exact."""
import numpy as np
import pytest

import device_rate_scale as drs
import resample as rsm
from rx_tools_b200 import resample as rs

N_SM = 132
TOPS = [(1 << 22) // J for J in (1, 2, 8, 1024)]


def _sweep():
    rng = np.random.default_rng(2026)
    out = []
    for J in (1, 2, 8, 1024):
        L = (1 << 22) // J
        for N in (L - 1, L + 1, 2 * L - 1, 8191 * L + 1):
            if N >= 1:
                out.append((L, N, J))
    out += [(4194301, 4194300, 1), (4194301, 8388601, 1), (1, 100, 8), (3, 40_000, 8), (3, 40_000, 1024),
            (12288, 24575, 1), (12289, 24577, 1), (1536, 3071, 8), (1537, 3073, 8)]
    for _ in range(200):
        J = int(rng.integers(1, 1025))
        L = int(rng.integers(1, (1 << 22) // J + 1))
        N = int(rng.choice([rng.integers(1, 64), rng.integers(1, 4 * L + 2), rng.integers(1, 1 << 31)]))
        out.append((L, N, J))
    return out


@pytest.mark.parametrize("n0", [0, (1 << 32) + 5, (1 << 64) - (1 << 20)])
def test_launch_invariants_over_the_accepted_range(n0):
    rng = np.random.default_rng(n0 & 0xffff)
    for L, N, J in _sweep():
        for c in (1, N // max(1, L) + 1, int(rng.integers(1, 1 << 20)), (1 << 20) - 1):
            a = drs.launch(L, N, J, n0, c, N_SM)
            if a is None:
                continue
            assert a["worst_v"] <= a["v_bound"] < (1 << 31), (L, N, J, c)
            assert a["worst_staged"] <= a["room"] <= drs.RS_SPAN, (L, N, J, c)
            assert a["smem"] <= drs.H100_SMEM_OPTIN, (L, N, J)
            assert 1 <= a["U"] <= drs.RS_MAX_U and a["ctas"] * a["U"] >= a["n_out"]
            assert 0 <= a["p0"] < L and a["q0"] >= 0


def test_the_named_regimes_are_what_the_gpu_cases_claim():
    # the top of the range at U = 512: v can reach 512 (L - 1), just below 2^31, and some CTA comes within L of it
    a = drs.launch(4194301, 4194300, 1, 0, 600_000, N_SM)
    assert a["which"] == "max_u" and a["U"] == 512 and a["v_bound"] == 512 * (4194301 - 1)
    assert (1 << 31) - (1 << 22) - 2048 < a["worst_v"] < 1 << 31
    # span-limited U
    assert drs.launch(1, 100, 8, 0, 10_000_000, N_SM)["which"] == "span"
    assert drs.launch(1, 100, 8, 0, 10_000_000, N_SM)["U"] == 82
    for J in (8, 64, 1024):
        b = drs.launch(3, 40_000, J, 0, 10_000_000, N_SM)
        assert b["which"] == "span" and b["U"] == 1
    # the shared-memory taps flip
    assert drs.launch(12288, 24575, 1, 0, 1000, N_SM)["smem_taps"]
    assert not drs.launch(12289, 24577, 1, 0, 1000, N_SM)["smem_taps"]


def test_umulhi_needs_at_most_one_correction():
    """Every v up to each L's worst, for L where that is affordable; for the rest, the two ends of every quotient's
    block of v, which bound the whole block: the estimate is non-decreasing in v and floor(v / L) is constant on it."""
    for L in [1, 2, 3, 7, 25, 256, 625, 1024, 3072, 4095, 4097]:
        worst = 512 * (L - 1) + L
        v = np.arange(worst + 1, dtype=np.uint64)
        k = drs.umulhi_corrections(v, L)
        assert k.min() >= 0 and k.max() <= 1, L
    for L in [12289, 65537, 1 << 21, (1 << 21) + 1, 4194301, 4194303, 1 << 22]:
        worst = 512 * (L - 1) + L
        q = np.arange(worst // L + 1, dtype=np.uint64)
        ends = np.concatenate([q * np.uint64(L), q * np.uint64(L) + np.uint64(L - 1)])
        k = drs.umulhi_corrections(ends[ends <= worst], L)
        assert k.min() >= 0 and k.max() <= 1, L


@pytest.mark.parametrize("L,N,J,n0", [(21, 25, 24, 0), (25, 21, 8, 12345), (5, 8, 48, (1 << 40) + 7),
                                      (187, 256, 136, (1 << 64) - 5000), (1, 7, 3, 0), (7, 1, 5, 99)])
def test_sparse_model_equals_full_model(L, N, J, n0):
    rng = np.random.default_rng(L + N + J)
    h = rng.integers(-4000, 4001, size=L * J).astype(np.int32)
    x = rng.integers(-32768, 32768, size=2 * 3000).astype(np.int16)
    hist = rng.integers(-32768, 32768, size=2 * (J - 1)).astype(np.int16)
    for hh in (None, hist):
        want, _ = rsm.resample_model(x, L, N, h, 15, n0, hh)
        n = want.size // 2
        H = J + 3
        pre = np.zeros(2 * H, np.int16)
        if hh is not None:
            pre[2 * (H - (J - 1)):] = hh
        idx = list(range(n))
        got = drs.sparse_outputs(np.concatenate([pre, x]), H, L, N, h, 15, n0, idx)
        assert np.array_equal(got.reshape(-1), want)


def test_in_len_for_upsampling_is_the_least_call():
    """For L > N one device sample may emit several outputs, so in_len is the least call with at least n_out outputs;
    its count can pass n_out."""
    inexact = 0
    for L, N in [(25, 21), (7, 3), (1024, 391), (3, 2), (8, 5)]:
        for n0 in (0, 1, 17, (1 << 32) + 3):
            for n_out in (0, 1, 2, 5, 64, 1000, 4097):
                c = rs.in_len(L, N, n0, n_out)
                if n0 < 1000:                                           # the search is affordable
                    assert c == drs.in_len_brute(L, N, n0, n_out)
                assert rsm.out_count(n0, c, L, N) >= n_out
                assert c == 0 or rsm.out_count(n0, c - 1, L, N) < n_out
                inexact += rsm.out_count(n0, c, L, N) > n_out
    assert inexact > 0


def test_group_rules():
    # rx_sdr host groups at 21/25, M = 8, one CS16 channel: 8 625 817 device samples, whose upload (4 bytes each), 21/25
    # as many capture samples (4 bytes each) and an eighth of those as rows (4 bytes each) fit the scratch bytes
    g, gn = drs.sdr_host_group(21, 25, 8, 1, 4)
    assert g == 8_625_817 and gn == rsm.ceil_div(g * 21, 25) // 8 + 1
    assert 4 * g + 4 * g * 21 / 25 + 4 * g * 21 / 25 / 8 <= drs.SDR_SCRATCH_BYTES
    # the unattached rule (a multiple of M capture samples) holds 14.9 M: a group without the resampler term is larger
    assert 8 * (drs.SDR_SCRATCH_BYTES // (4 * 8 + 4)) > 1.5 * g
    group, n = drs.power_groups(100, 8, 1 << 14)
    assert group * 8 * (1 << 14) * 2 <= drs.POWER_SCRATCH_BYTES and n == rsm.ceil_div(100, group)


def test_check_indices_cover_ctas_and_edges():
    idx = set(drs.check_indices(100_000, 512, 24, edges=[40_000], seed=3))
    assert all(b in idx and min(100_000, b + 512) - 1 in idx for b in range(0, 100_000, 512))
    assert set(range(40_000 - 24, 40_000 + 24)) <= idx and set(range(24)) <= idx
    assert set(range(100_000 - 24, 100_000)) <= idx and len(idx) < 100_000 // 8
    # a launch that starts 100 outputs ahead of the call: its CTAs start at k 512 - 100 in the call's indices
    idx = set(drs.check_indices(10_000, 512, 24, seed=3, lead=100))
    assert all(b in idx and b - 1 in idx for b in range(412, 10_000, 512))


def test_umulhi_margin_past_rs_max_u():
    """RS_MAX_U = 512 keeps v below 2^31 with room to spare: even 1024 outputs per CTA at L = 2^22 keep v below 2^32,
    where the unsigned multiply-high still needs at most one correction, so the bound is a margin rather than an edge."""
    for L in [4194301, 1 << 22]:
        worst = 1024 * (L - 1)                          # pa + u (N mod L) at pa, N mod L = L - 1, u = 1023
        assert worst < 1 << 32
        q = np.arange(worst // L + 1, dtype=np.uint64)
        ends = np.concatenate([q * np.uint64(L), q * np.uint64(L) + np.uint64(L - 1)])
        k = drs.umulhi_corrections(ends[ends <= worst], L)
        assert k.min() >= 0 and k.max() <= 1, L
