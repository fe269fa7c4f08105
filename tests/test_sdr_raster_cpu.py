"""The shells' raster capture plan (rxb200_fm_plan_capture_raster) and rx_sdr raster I/Q handles without a GPU: the
planner against its rule restated over seeded frequency sets (grids of 5, 12.5, 25 and 200 kHz and arbitrary Hz), caps
at R and R - 1, K at 4096 and 4097, every bin against exact fractions, the same fc, M, R and T as the rx_fm and rx_sdr
single-stage plans, the header's worked examples; the create refusals (all before any device is touched); the shapes'
golden hashes in every format; and both shells' raster-mode refusals, none of which opens the device or creates a
file."""
import ctypes as C
import json
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import sdr_raster as sr
from rx_tools_b200 import _lib, fm, sdr

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = json.load(open(os.path.join(HERE, "golden", "sdr_raster_golden.json")))
RX_SDR = os.path.join(ROOT, "host", "rx_sdr_b200")
RX_FM = os.path.join(ROOT, "host", "rx_fm_b200")
RATES = (250_000, 25_000, 1_008_000, 48_000, 12_500, 200_000)


def _tuned_sets(n_sets, seed):
    """(tuned frequencies, chain rate): channels on a grid of 5, 12.5, 25 or 200 kHz, or at arbitrary Hz."""
    rng = np.random.default_rng(seed)
    for i in range(n_sets):
        k = int(rng.integers(1, 40))
        grid = [5_000, 12_500, 25_000, 200_000, None][i % 5]
        base = int(rng.integers(1_000_000, 3_000_000_000))
        if grid is None:
            t = base + rng.integers(0, int(rng.choice([3_000, 200_000, 5_000_000])), size=k)
        else:
            t = base - base % grid + grid * rng.choice(int(rng.choice([8, 100, 2000])), size=k)
        yield [int(v) for v in t], int(rng.choice(RATES))


def _check_plan(tuned, c, cap):
    want = sr.plan_restated(tuned, c, cap)
    if isinstance(want, str):
        with pytest.raises(_lib.Rxb200Error) as e:
            fm.plan_capture_raster(tuned, c, cap)
        assert e.value.code == _lib.EINVAL
        return want
    fc, M, R, T, K, bins = want
    plan, got = fm.plan_capture_raster(tuned, c, cap)
    assert (plan.centre_hz, plan.decim, plan.capture_rate, plan.n_taps, plan.n_bins, plan.shift) == (fc, M, R, T, K, 30)
    assert got == bins
    for t, b in zip(tuned, got):                       # b_k = (o_k K / R) mod K, exactly
        q = Fraction(t - fc) * K / R
        assert q.denominator == 1 and int(q) % K == b and 0 <= b < K
    # fc, M, R and T are the single-stage plans'
    sp, _ = sdr.plan_sdr_capture(tuned, c, cap)
    assert (sp.centre_hz, sp.decim, sp.capture_rate, sp.n_taps) == (fc, M, R, T)
    try:
        fp, _ = fm.plan_capture(tuned, c, cap)
        assert (fp.centre_hz, fp.decim, fp.capture_rate, fp.n_taps) == (fc, M, R, T)
    except _lib.Rxb200Error as e:                      # only the table mixer's period refusal differs
        assert e.code == _lib.EUNSUPPORTED
    return "ok"


def test_planner_equals_rule_restated():
    seen = {"ok": 0, "rate": 0, "bins": 0}
    for tuned, c in _tuned_sets(200, 17):
        want = sr.plan_restated(tuned, c, 1 << 40)
        if isinstance(want, str):
            seen[_check_plan(tuned, c, 1 << 40)] += 1
            continue
        R = want[2]
        for cap in (R, R - 1):
            if cap < R:
                with pytest.raises(_lib.Rxb200Error) as e:
                    fm.plan_capture_raster(tuned, c, cap)
                assert e.value.code == _lib.EINVAL and str(R) in str(e.value)
                continue
            seen[_check_plan(tuned, c, cap)] += 1
    assert seen["ok"] > 100 and seen["bins"] > 10, seen


@pytest.mark.parametrize("K", [4096, 4097])
def test_k_lands_on_4096_and_4097(K):
    """Two channels 100 Hz apart at c = 50 K: M = 2, R = 100 K, g = 100 Hz, so K0 = K."""
    tuned, c = [100_000_000, 100_000_100], 50 * K
    want = sr.plan_restated(tuned, c, 1 << 40)
    if K == 4096:
        plan, bins = fm.plan_capture_raster(tuned, c, 1 << 40)
        assert (plan.decim, plan.capture_rate, plan.n_bins) == (2, 100 * K, 4096) and want[4] == 4096
        assert bins == [0, 4096 * 100 // (100 * K)]
    else:
        assert want == "bins"
        with pytest.raises(_lib.Rxb200Error) as e:
            fm.plan_capture_raster(tuned, c, 1 << 40)
        assert e.value.code == _lib.EINVAL
        msg = str(e.value)
        assert "4097" in msg and "100 Hz" in msg and "RXB200_CAPTURE_STAGES=2" in msg


def test_small_grids_take_three_bins():
    """One frequency (g = 0, K0 = 1): K = 3 and the channel on bin 0."""
    plan, bins = fm.plan_capture_raster([100_000_000], 250_000, 1 << 40)
    assert (plan.n_bins, bins, plan.centre_hz, plan.decim) == (3, [0], 100_000_000, 1)
    plan, bins = fm.plan_capture_raster([100_000_000, 100_000_000], 250_000, 1 << 40)
    assert (plan.n_bins, bins) == (3, [0, 0])


@pytest.mark.parametrize("tuned,c,want", [
    ([88_100_000 + 200_000 * k for k in range(100)], 250_000, (97_900_000, 81, 20_250_000, 2593, 405)),
    ([162_400_000 + 25_000 * k for k in range(7)], 25_000, (162_475_000, 7, 175_000, 225, 7)),
    ([162_400_000 + 25_000 * k for k in range(7)], 1_008_000, (162_475_000, 2, 2_016_000, 65, 2016)),
])
def test_worked_examples(tuned, c, want):
    plan, bins = fm.plan_capture_raster(tuned, c, 1 << 40)
    assert (plan.centre_hz, plan.decim, plan.capture_rate, plan.n_taps, plan.n_bins) == want
    K = want[4]
    assert bins[0] == (tuned[0] - want[0]) * K // want[2] % K and tuned[bins.index(0)] == want[0]


def test_worked_example_refused():
    tuned = [162_400_000, 162_400_001, 162_550_000]
    assert sr.plan_restated(tuned, 25_000, 1 << 40) == "bins"
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.plan_capture_raster(tuned, 25_000, 1 << 40)
    assert e.value.code == _lib.EINVAL and "175000" in str(e.value)


def test_plan_refuses_bad_arguments():
    L = _lib.lib()
    out = _lib.FmRasterPlanC()
    t = np.array([100_000_000], np.int64)
    b = np.zeros(1, np.int32)
    pt, pb = t.ctypes.data_as(C.POINTER(C.c_int64)), b.ctypes.data_as(C.POINTER(C.c_int))
    assert L.rxb200_fm_plan_capture_raster(None, 1, 250_000, 1 << 40, C.byref(out), pb) == _lib.EINVAL
    assert L.rxb200_fm_plan_capture_raster(pt, 1, 250_000, 1 << 40, None, pb) == _lib.EINVAL
    assert L.rxb200_fm_plan_capture_raster(pt, 1, 250_000, 1 << 40, C.byref(out), None) == _lib.EINVAL
    assert L.rxb200_fm_plan_capture_raster(pt, 0, 250_000, 1 << 40, C.byref(out), pb) == _lib.EINVAL
    assert L.rxb200_fm_plan_capture_raster(pt, 1, 0, 1 << 40, C.byref(out), pb) == _lib.EINVAL
    t[0] = -1
    assert L.rxb200_fm_plan_capture_raster(pt, 1, 250_000, 1 << 40, C.byref(out), pb) == _lib.EINVAL
    # M > 256 and R above 2^31 - 1
    with pytest.raises(_lib.Rxb200Error):
        fm.plan_capture_raster([100_000_000, 100_000_000 + 300 * 10_000], 10_000, 1 << 40)
    with pytest.raises(_lib.Rxb200Error):
        fm.plan_capture_raster([1_000_000_000, 2_000_000_000], 1_000_000_000, 1 << 40)


def _create(K, bins, dd, out=True):
    L = _lib.lib()
    h = C.c_void_p()
    b = None if bins is None else np.ascontiguousarray(bins, dtype=np.int32)
    d, _t = fm._ddc_c(dd)
    rc = L.rxb200_sdr_mix_create_raster(K, None if b is None else b.ctypes.data_as(C.POINTER(C.c_int)),
                                        0 if b is None else b.size, C.byref(d), 0, C.byref(h) if out else None)
    assert not h.value
    return rc


def test_create_refusals_before_any_device():
    dd = (4, np.ones(9, np.int32), 3)
    assert _create(8, [0], dd, out=False) == _lib.EINVAL                 # NULL out
    assert _create(2, [0], dd) == _lib.EINVAL                            # K < 3
    assert _create(4097, [0], dd) == _lib.EINVAL                         # K > 4096
    assert _create(8, None, dd) == _lib.EINVAL                           # NULL bins
    assert _create(8, [], dd) == _lib.EINVAL                             # no channel
    assert _create(8, [0, 8], dd) == _lib.EINVAL                         # bin outside [0, K)
    assert _create(8, [-1], dd) == _lib.EINVAL
    assert _create(8, [0], (2, np.full(4, 1 << 20, np.int32), 30)) == _lib.EINVAL          # sum |h| = 2^22
    assert _create(8, [0], (0, np.ones(3, np.int32), 0)) == _lib.EINVAL                     # M out of range
    assert _create(8, [0], (2, np.ones(3, np.int32), 63)) == _lib.EINVAL                    # S out of range
    assert _create(8, [0], (2, np.ones(8192 + 1, np.int32), 0)) == _lib.EINVAL             # T > 8192
    with pytest.raises(ValueError):
        sdr.SdrMix(1000, [0], ddc=dd, raster=(8, [0]))


@pytest.mark.parametrize("name", list(sr.SHAPES))
def test_shape_hashes_every_format(name):
    g = GOLDEN[name]
    x = sr.case_capture(name)
    assert sr.digest(x) == g["input_sha256"]
    y, _ = sr.model(name, x)
    assert list(y.shape) == g["shape"]
    for fmt in sr.FORMATS:
        assert sr.digest(sr.convert(y, fmt)) == g[fmt], fmt


def test_golden_covers_every_shape():
    assert sorted(GOLDEN) == sorted(sr.SHAPES)


def test_unit_shape_bin0_is_the_capture():
    x = sr.case_capture("unit_k5")
    y, M = sr.model("unit_k5", x)
    assert M == 1 and np.array_equal(y[0], x)


_OFF_GRID = ["-f", "162400000", "-f", "162400001", "-f", "162550000"]


@pytest.mark.parametrize("shell,args,cap,needle", [
    (RX_SDR, _OFF_GRID + ["-s", "25k", "out"], "100000000", "175000 bins"),
    (RX_SDR, ["-f", "100M", "-f", "100.2M", "-s", "250k", "-"], "100000000", "not to '-'"),
    (RX_SDR, ["-f", "100M", "-f", "101M", "-s", "250k", "out"], "2249999", "2250000"),
    (RX_FM, _OFF_GRID + ["out"], "100000000", "2016000 bins"),
    (RX_FM, ["-f", "100M", "-f", "100.2M", "-"], "100000000", "'-' as the filename"),
    (RX_FM, ["-f", "100M", "-f", "101M", "out"], "3023999", "3024000"),
])
def test_shell_raster_refusals_create_no_file(tmp_path, shell, args, cap, needle):
    if not os.path.exists(shell):
        pytest.skip(f"{shell} not built")
    e = dict(os.environ, RXB200_CAPTURE_RATE=cap, RXB200_CAPTURE_STAGES="raster")
    r = subprocess.run([shell, "-d", "driver=file,path=" + str(tmp_path / "none.cs16")] + args, cwd=tmp_path, env=e,
                       capture_output=True, text=True, timeout=60)
    assert r.returncode == 1 and needle in r.stderr, r.stderr
    assert os.listdir(tmp_path) == []
