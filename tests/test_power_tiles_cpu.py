"""Wide rx_power sweeps in tiles on the CPU: the planner (rxb200_power_plan_tiles, rxb200_power_tile) against its
restatement over seeded command lines and caps, its invariants, one tile being exactly the capture mode's plan, and its
refusals; the burst model against the stateless-DDC identity; and the port against the unmodified reference on every
named shape's burst hop buffers, with the golden hashes tests/golden/power_tiles_golden.json records."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

import power_mix as pm
import power_tiles as ptl
from rx_tools_b200 import _lib, power

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "power_tiles_golden.json")
TSTR = "2026-01-01, 00:00:00"


def _plans(seed, n):
    """n sweep plans from seeded rx_power command lines: lower edge, span, bin size, crop, boxcar or -F 9, -P (lines the
    planner refuses, such as a bin wider than the span, are drawn again)."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        lo = int(rng.integers(24, 1700)) * 1_000_000 + int(rng.integers(0, 1000)) * 1000
        span = int(rng.choice([300_000, 2_000_000, 9_000_000, 40_000_000, 250_000_000, 1_700_000_000]))
        span = int(span * rng.uniform(0.5, 1.5))
        bin_hz = int(rng.choice([1000, 10_000, 100_000, 1_000_000]))
        crop = float(rng.choice([0.0, 0.1, 0.25, 0.285, 0.5, 0.9]))
        fir = int(rng.choice([0, 0, 9]))
        try:
            out.append(power.plan_range(f"{lo}:{lo + span}:{bin_hz}", crop, 0 if fir else 1, fir,
                                        int(rng.integers(0, 2))))
        except _lib.Rxb200Error:
            pass
    return out


CAPS = [1_000_000, 2_800_000, 5_000_000, 6_000_000, 10_000_000, 20_000_000, 30_720_000, 61_440_000, 200_000_000,
        (1 << 31) - 1, 1 << 40]


@pytest.mark.parametrize("seed", range(4))
def test_planner_equals_restatement(seed):
    checked = 0
    for plan in _plans(seed, 12):
        for cap in CAPS:
            want = ptl.tiling(plan, cap)
            if want is None:
                with pytest.raises(_lib.Rxb200Error) as e:
                    power.plan_tiles(plan, cap)
                assert e.value.code == _lib.EINVAL
                continue
            tl, tiles, offs = power.plan_tiles(plan, cap)
            n_tiles, h, M, T, R, wtiles, woffs = want
            assert (tl.n_tiles, tl.hops_per_tile, tl.decim, tl.n_taps, tl.capture_rate) == (n_tiles, h, M, T, R)
            assert tiles == wtiles and offs == woffs, (plan, cap)
            checked += 1
    assert checked > 60


@pytest.mark.parametrize("seed", range(4))
def test_planner_invariants(seed):
    for plan in _plans(100 + seed, 12):
        for cap in CAPS:
            if cap < plan.rate:
                continue
            tl, tiles, offs = power.plan_tiles(plan, cap)
            assert len(tiles) == tl.n_tiles
            assert tiles[0][0] == 0 and tiles[-1][1] == plan.n_hops
            for (b0, e0, _), (b1, _, _) in zip(tiles, tiles[1:]):
                assert e0 == b1
            for hb, he, centre in tiles:
                assert 0 < he - hb <= tl.hops_per_tile
                assert ptl.mreq(he - hb, plan.freq_step, plan.rate) <= tl.decim <= 4096
                for i in range(hb, he):
                    assert offs[i] == plan.hop_freq(i) - centre
            assert tl.capture_rate == tl.decim * plan.rate <= min(cap, (1 << 31) - 1)
            assert all(2 * abs(f) < tl.capture_rate for f in offs)
            assert tl.n_taps == min(8191, 32 * tl.decim + 1)


@pytest.mark.parametrize("name", sorted(pm.SHAPES))
def test_one_tile_is_the_capture_plan(name):
    plan = pm.shape(name)[0]
    fc, offs, M, R, dd = pm.capture_plan(plan)
    for cap in (R, R + 1, 1 << 40):
        tl, tiles, toffs = power.plan_tiles(plan, cap)
        assert (tl.n_tiles, tl.hops_per_tile, tl.decim, tl.capture_rate, tl.n_taps) == (1, plan.n_hops, M, R, dd[1].size)
        assert tiles == [(0, plan.n_hops, fc)] and toffs == offs
    if M > 1:
        assert power.plan_tiles(plan, R - 1)[0].n_tiles > 1


def test_refusals():
    plan = power.plan_range("88M:108M:10k")
    for cap in (plan.rate - 1, 0, -5):
        with pytest.raises(_lib.Rxb200Error) as e:
            power.plan_tiles(plan, cap)
        assert e.value.code == _lib.EINVAL
    assert power.plan_tiles(plan, plan.rate)[0].decim == 1
    L = _lib.lib()
    pc = _lib.PowerPlanC(plan.to_c(), plan.rate, plan.crop, plan.first_freq, plan.freq_step, plan.bin_size_hz)
    tl = _lib.PowerTilingC()
    assert L.rxb200_power_plan_tiles(None, 10**8, C.byref(tl), None) == _lib.EINVAL
    assert L.rxb200_power_plan_tiles(C.byref(pc), 10**8, None, None) == _lib.EINVAL
    assert L.rxb200_power_plan_tiles(C.byref(pc), 6_000_000, C.byref(tl), None) == _lib.OK
    b, e, c = C.c_int(0), C.c_int(0), C.c_int64(0)
    for t in (-1, tl.n_tiles):
        assert L.rxb200_power_tile(C.byref(pc), C.byref(tl), t, C.byref(b), C.byref(e), C.byref(c)) == _lib.EINVAL
    assert L.rxb200_power_tile(C.byref(pc), C.byref(tl), 0, None, C.byref(e), C.byref(c)) == _lib.EINVAL


def test_named_shapes_have_several_tiles():
    got = {n: ptl.shape(n) for n in ptl.SHAPES}
    for name, (plan, _, tl, tiles, _, dd) in got.items():
        assert tl.n_tiles > 1, name
    assert got["one_hop"][2].decim == 1 and got["one_hop"][2].hops_per_tile == 1
    plan, _, tl, tiles, _, _ = got["hops300"]
    assert tl.hops_per_tile > 256 and tiles[1][0] > 0 and tiles[1][1] - tiles[1][0] > 256
    assert got["rms"][0].bin_e == 0 and got["peak_hold"][0].peak_hold == 1 and got["F9"][0].comp_fir_size == 9
    wide = got["wide_acc"][5]
    assert int(np.abs(wide[1].astype(np.int64)).sum()) * 32768 + (1 << (wide[2] - 1)) >= 1 << 31


@pytest.mark.parametrize("M,T", [(1, 1), (1, 33), (3, 17), (4, 129), (7, 8)])
def test_burst_model_is_the_stateless_ddc_past_the_lead(M, T):
    """Outputs G/M + u of the DDC from n = 0 over the burst; and the outputs before G/M are the ones whose windows reach
    before the burst, so the lead is the least that keeps zeros out."""
    rng = np.random.default_rng(M * 100 + T)
    buf_len, R, offs = 8, 1_000_000, [-300_000, 0, 123_457]
    dd = (M, rng.integers(-3000, 3000, size=T).astype(np.int32), 12)
    G = ptl.lead(M, T)
    assert G % M == 0 and G >= T - 1 and G - M < T - 1 or G == 0
    x = rng.integers(-30000, 30000, size=2 * (G + 3 * M * buf_len // 2)).astype(np.int16)
    hb = ptl.burst_buffers(x, R, offs, dd, buf_len)
    assert hb.shape == (3, 3, buf_len)
    for k, f in enumerate(offs):
        y, _ = pm.ddc(x, R, f, dd, 0)
        assert np.array_equal(hb[:, k, :].reshape(-1), y[2 * G // M:])
        # a different history before the burst changes none of the kept outputs
        junk = rng.integers(-30000, 30000, size=2 * (T - 1)).astype(np.int16)
        y2, _ = pm.ddc(x, R, f, dd, 0, pm.nco_mix(junk, R, f, -(T - 1)) if T > 1 else None)
        assert np.array_equal(y2[2 * G // M:], y[2 * G // M:])


@pytest.mark.parametrize("name", sorted(ptl.SHAPES))
def test_golden_hashes(name, port):
    g = json.load(open(GOLDEN))[name]
    plan, win, tl, tiles, offs, dd, bs = ptl.case_input(name)
    assert [plan.n_hops, plan.bin_e, plan.buf_len, plan.downsample, plan.downsample_passes] == g["plan"]
    assert [tl.n_tiles, tl.hops_per_tile, tl.decim, tl.capture_rate, dd[1].size, dd[2]] == g["tiling"]
    assert [pm.digest(b) for b in bs] == g["burst_sha256"]
    _, hb = ptl.tile_buffers(name)
    assert pm.digest(hb) == g["bufs_sha256"]
    avg, smp = pm.port_result(port, plan, win, hb)
    assert pm.digest(avg) == g["avg_sha256"] and smp.tolist() == g["samples"]
    csv = power.csv_rows(plan, avg, smp, TSTR)
    assert hashlib.sha256(csv.encode()).hexdigest() == g["csv_sha256"]


def test_golden_covers_every_shape():
    assert sorted(json.load(open(GOLDEN))) == sorted(ptl.SHAPES)


@pytest.mark.ref
@pytest.mark.parametrize("name", sorted(ptl.SHAPES))
def test_port_equals_reference(name, port, ref_power):
    s = ptl.SHAPES[name]
    plan, win = ptl.shape(name)[:2]
    rp = ref_power.setup(s["freq"], s["crop"], s["boxcar"], s["fir"], s["peak"], s["window"])
    assert (rp.tune_count, rp.bin_e, rp.buf_len, rp.rate) == (plan.n_hops, plan.bin_e, plan.buf_len, plan.rate)
    _, hb = ptl.tile_buffers(name)
    avg_r, smp_r = ref_power.scan(hb, hb.shape[0])
    avg_p, smp_p = pm.port_result(port, plan, win, hb)
    assert np.array_equal(smp_p, smp_r) and np.array_equal(avg_p, avg_r)
