"""Capture plans at a device rate and the resampler's input count, without a GPU: every _at planner against its
restatement (tests/device_rate.py) over seeded tuned sets, the header's worked examples, the R > R_dev refusal, the
guard edge and the cap; rxb200_resample_in_len against brute force and its closed form up to n0 = 2^63."""
import random

import pytest

import device_rate as dr
import resample as rsm
from rx_tools_b200 import _lib, fm, sdr
from rx_tools_b200 import resample as rs

PLANNERS = {
    dr.FM: fm.plan_capture,
    dr.SDR: sdr.plan_sdr_capture,
    dr.TWO_STAGE: fm.plan_capture_two_stage,
    dr.RASTER: fm.plan_capture_raster,
}


def library(kind, tuned, c, cap, R_dev):
    """The library's _at planner as the restatement's dict, or the refusal's code."""
    try:
        p, v = PLANNERS[kind](tuned, c, cap, device_rate=R_dev)
    except _lib.Rxb200Error as e:
        return e.code
    if kind == dr.TWO_STAGE:
        return dict(fc=p.centre_hz, R=p.capture_rate, K=p.n_bins, M1=p.coarse_decim, T1=p.coarse_taps, offsets=v)
    if kind == dr.RASTER:
        return dict(fc=p.centre_hz, M=p.decim, R=p.capture_rate, T=p.n_taps, K=p.n_bins, bins=v)
    return dict(fc=p.centre_hz, M=p.decim, R=p.capture_rate, T=p.n_taps, offsets=v)


CODES = {"rate": _lib.EINVAL, "m8": _lib.EINVAL, "bins": _lib.EINVAL, "device": _lib.EUNSUPPORTED,
         "period": _lib.EUNSUPPORTED}


def agree(kind, tuned, c, cap, R_dev):
    want = dr.plan_at(kind, tuned, c, cap, R_dev)
    got = library(kind, tuned, c, cap, R_dev)
    if isinstance(want, str):
        assert got == CODES[want], (kind, tuned, c, cap, R_dev, want, got)
    else:
        assert got == {k: v for k, v in want.items() if k != "span"}, (kind, tuned, c, cap, R_dev)
    return want


@pytest.mark.parametrize("kind", list(PLANNERS))
def test_planners_match_restatement_over_seeded_sets(kind):
    rng = random.Random(list(PLANNERS).index(kind))
    seen = {"plan": 0, "device": 0}
    for _ in range(300):
        grid = rng.choice([1, 1000, 12_500, 25_000, 200_000])
        n = rng.randint(1, 12)
        base = rng.randrange(24_000_000, 1_700_000_000)
        tuned = [base + grid * rng.randrange(0, rng.choice([4, 40, 400])) for _ in range(n)]
        c = rng.choice([25_000, 170_000, 250_000, 1_008_000, 1_020_000, rng.randrange(8_000, 3_000_000)])
        want = dr.plan_at(kind, tuned, c, 10**10, 10**9)
        R = want["R"] if isinstance(want, dict) else c * 8
        R_dev = rng.choice([R, R + 1, R - 1, rng.randrange(max(1, R // 2), 2 * R), 2_400_000, 30_720_000])
        cap = rng.choice([10**10, R, R - 1, R_dev])
        w = agree(kind, tuned, c, cap, R_dev)
        if isinstance(w, dict) or w == "device":
            seen["plan" if isinstance(w, dict) else w] += 1
    assert seen["plan"] > 20 and seen["device"] > 10


@pytest.mark.parametrize("case", dr.WORKED, ids=["noaa7_2.4M", "sdr4_2.4M", "fm100_30.72M"])
def test_worked_examples(case):
    kind, tuned, c, R_dev, M, R, LN = case
    w = agree(kind, tuned, c, 10**10, R_dev)
    assert (w["M"], w["R"]) == (M, R)
    p = rs.plan_resample(R_dev, R, w["span"])
    assert (p.up, p.down) == LN


def test_worked_examples_in_every_kind():
    for kind in PLANNERS:
        for _, tuned, c, R_dev, _M, _R, _LN in dr.WORKED:
            w = agree(kind, tuned, c, 10**10, R_dev)
            if isinstance(w, dict):
                # the floor leaves the guard band, so the resampler fits whenever R <= R_dev
                rs.plan_resample(R_dev, w["R"], w["span"])


def test_device_rate_refusal_and_guard_edge():
    tuned, c = dr.NOAA7, 1_008_000
    # R = 2.016 M: a device at R exactly plans with L = N = 1; one hertz below is refused as R > R_dev
    assert library(dr.FM, tuned, c, 10**10, 2_016_000)["R"] == 2_016_000
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.plan_capture(tuned, c, 10**10, device_rate=2_015_999)
    assert e.value.code == _lib.EUNSUPPORTED and "2016000" in str(e.value) and "2015999" in str(e.value)
    # the guard edge: with 2A = 150 kHz, M = ceil((2A + c + G) / c) is 2 at c = 2A + G and above, 3 one hertz below
    for R_dev in (31_999_999, 32_000_000, 32_000_001):
        G = dr.guard(R_dev)
        for dc, M in ((-1, 3), (0, 2), (1, 2)):
            assert agree(dr.SDR, tuned, 150_000 + G + dc, 10**10, R_dev)["M"] == M


def test_cap_stays_first():
    tuned, c = dr.FM100, 1_020_000
    # R = 22.44 M above both the cap and the device rate: the cap's refusal (EINVAL) comes first
    assert library(dr.FM, tuned, c, 22_439_999, 20_000_000) == _lib.EINVAL
    assert library(dr.FM, tuned, c, 22_440_000, 20_000_000) == _lib.EUNSUPPORTED
    assert library(dr.FM, tuned, c, 22_440_000, 30_720_000)["R"] == 22_440_000


def test_bad_device_rate():
    for R_dev in (0, -1, 1 << 31):
        for kind in PLANNERS:
            assert library(kind, dr.NOAA7, 1_008_000, 10**10, R_dev) == _lib.EINVAL


def test_existing_planners_unchanged_by_guard():
    """Without a device rate the planners are today's (the internal G = 0 path)."""
    rng = random.Random(5)
    for _ in range(100):
        tuned = [rng.randrange(100_000_000, 101_000_000, 25_000) for _ in range(rng.randint(1, 6))]
        c = rng.choice([250_000, 1_008_000])
        p, offs = fm.plan_capture(tuned, c, 10**10)
        A = max(abs(o) for o in offs)
        assert p.decim == -(-(2 * A + c) // c)


def test_in_len_brute_force():
    rng = random.Random(11)
    for _ in range(400):
        L, N = rng.randint(1, 40), rng.randint(1, 40)
        n0, n_out = rng.randrange(0, 5000), rng.randrange(0, 300)
        c = 0
        while rsm.out_count(n0, c, L, N) < n_out:
            c += 1
        assert rs.in_len(L, N, n0, n_out) == c == dr.in_len_rule(L, N, n0, n_out)
        if L <= N:
            assert rsm.out_count(n0, c, L, N) == n_out


def test_in_len_large_counts():
    rng = random.Random(12)
    for _ in range(400):
        L, N = rng.randint(1, (1 << 31) - 1), rng.randint(1, (1 << 31) - 1)
        if rng.random() < 0.5:
            L = rng.randint(1, N)                 # L <= N: the count is exact
        n0 = rng.randrange(0, 1 << 63)
        n_out = rng.choice([0, 1, 2, 131072, rng.randrange(0, 1 << 40)])
        c = rs.in_len(L, N, n0, n_out)
        assert c == dr.in_len_rule(L, N, n0, n_out)
        assert rsm.out_count(n0, c, L, N) >= n_out
        if n_out:
            assert rsm.out_count(n0, c - 1, L, N) < n_out
        if L <= N:
            assert rsm.out_count(n0, c, L, N) == n_out
    for args in ((0, 1, 0, 1), (1, 0, 0, 1)):
        with pytest.raises(_lib.Rxb200Error):
            rs.in_len(*args)
