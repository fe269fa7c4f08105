"""Seeded sweeps of the rx_power accumulate paths (tests/power_paths.py) against the port, byte for byte.

Every draw runs as its calls (pass and hop sub-ranges, shard ranges, or back-to-back device calls without a sync) on
one handle; after every call ``last_path()`` must equal the path the launch rule gives.  The reassembled ``avg`` (int64)
and ``samples`` must equal the port's.  A second run of the same calls doubles the sums (or keeps the max under peak
hold), and ``reset()`` zeroes.  The named command lines of tests/golden/power_paths_golden.json are checked against the
reference's own bytes."""
import json
import os

import numpy as np
import pytest
import torch

import power_paths
from rx_tools_b200 import power
from rx_tools_b200.synth import digest

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "power_paths_golden.json")


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run_calls(sc, d, d_x=None):
    """Run the draw's calls; returns the paths the library reported."""
    got = []
    parts = [np.ascontiguousarray(d.x[p0:p1, h0:h1]) for p0, p1, h0, h1 in d.calls]
    if d.device:                                 # every upload done before the first call: the calls do not wait
        bufs = [torch.from_numpy(p.reshape(-1)).cuda() for p in parts]
        d_x.extend(bufs)                         # kept alive until the handle's stream is done with them
        torch.cuda.synchronize()
    for i, (p0, p1, h0, h1) in enumerate(d.calls):
        if d.device:
            sc.scanner_device(bufs[i].data_ptr(), p1 - p0, h0, h1, sync=False)
        else:
            sc.scanner(parts[i], p1 - p0, h0, h1)
        got.append(sc.last_path())
    return got


@pytest.mark.parametrize("family,seed", power_paths.all_ids(), ids=[f"{f}-{s}" for f, s in power_paths.all_ids()])
def test_power_path_draw(family, seed, port, monkeypatch):
    d = power_paths.draw(family, seed)
    if d.dropped:
        pytest.skip(f"dropped draw: {d.dropped}")
    for k, v in d.env.items():                   # read once, at create
        monkeypatch.setenv(k, v)
    n_sm = _n_sm()
    want_paths = [power_paths.expected_path(d.plan, d.env, p1 - p0, h1 - h0, n_sm) for p0, p1, h0, h1 in d.calls]
    want, want_smp = power_paths.port_result(port, d)
    sc = power.PowerScanner(d.plan, d.window, sinewave=d.sine)
    keep = []
    try:
        assert sc.last_path()["kernel"] == "none"
        got_paths = _run_calls(sc, d, keep)
        avg, smp = sc.read()
        assert got_paths == want_paths, (got_paths, want_paths, d.tags)
        assert np.array_equal(smp, want_smp), d.tags
        bad = np.argwhere(avg != want)
        assert bad.size == 0, (bad[:5].tolist(), avg[tuple(bad[0])], want[tuple(bad[0])], d.tags)
        _run_calls(sc, d, keep)
        avg2, smp2 = sc.read()
        assert np.array_equal(avg2, want if d.plan.peak_hold else 2 * want), d.tags
        assert np.array_equal(smp2, 2 * want_smp), d.tags
        sc.reset()
        z, zs = sc.read()
        assert not z.any() and not zs.any()
        if family == "cli" and d.plan.crop > 0 and seed % 4 == 0:
            sc.scanner(d.x, d.n_pass)
            assert sc.csv_rows_device() == power.csv_rows(d.plan, want, want_smp), d.tags
    finally:
        sc.close()


def test_power_paths_golden_cases():
    """The named command lines against the reference's own avg sha256 and samples (no reference on the GPU machine:
    its hashes travel)."""
    gold = json.load(open(GOLDEN))
    assert sorted(gold) == sorted(power_paths.GOLDEN_CASES)
    for name, c in power_paths.GOLDEN_CASES.items():
        plan = power_paths.golden_plan(c)
        win = power.window_table(c["window"], 1 << plan.bin_e)
        x = power_paths.golden_input(c, plan)
        sc = power.PowerScanner(plan, win)
        sc.scanner(x, c["n_pass"])
        avg, smp = sc.read()
        path = sc.last_path()
        sc.close()
        assert path == power_paths.expected_path(plan, {}, c["n_pass"], plan.n_hops, _n_sm()), name
        assert digest(avg) == gold[name]["avg_sha256"], name
        assert smp.tolist() == gold[name]["samples"], name


@pytest.mark.parametrize("bin_e,buf_len,env", [(10, 16384, {}), (10, 16384, {"RXB200_POWER_V1": "1"}),
                                               (16, 131072, {})], ids=["fft8", "generic", "big_load"])
def test_caller_sine_with_int16_min(bin_e, buf_len, env, port, monkeypatch):
    """A caller's Sinewave holding -32768 (the tables draws with random tables found it): the reference negates into an
    int16, so -(-32768) stays -32768 and wi = -16384.  Every kernel used to compute +16384 there."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    n = 1 << bin_e
    plan = power_paths.mkplan(bin_e, buf_len, n_hops=2)
    sine = power.sine_table(bin_e).copy()
    sine[[1, 3, n // 8, n // 2 + 5]] = -32768            # wi of twiddles 1, 3, N/8 and wr of N/4 + 5
    rng = np.random.default_rng(bin_e)
    x = power_paths.hop_input(rng, "noise", (2, 2, buf_len), False)
    win = power.window_table("hamming", n)
    want, want_smp = port.power_scan(power_paths.oracle_params(plan), win, x, 2, 2, sine=sine)
    plain, _ = port.power_scan(power_paths.oracle_params(plan), win, x, 2, 2, sine=np.maximum(sine, -32767))
    assert not np.array_equal(want, plain)            # the -32768 entries reach the result
    sc = power.PowerScanner(plan, win, sinewave=sine)
    sc.scanner(x, 2)
    avg, smp = sc.read()
    assert sc.last_path()["kernel"] == power_paths.expected_path(plan, env, 2, 2, _n_sm())["kernel"]
    sc.close()
    assert np.array_equal(smp, want_smp)
    assert np.array_equal(avg, want)


@pytest.mark.parametrize("buf_len", [116096, 116104], ids=["q_only", "i_and_q"])
def test_big_load_partial_last_slot(buf_len, port):
    """A ÷5 boxcar on a hop buffer just beyond shared memory (geometry draw 93 found it): the last slot is partial and
    lies past the int16 span remove_dc sums, buf_len/5 int16.  The global-memory path used to add that slot's Q (and,
    when buf_len/5 is even, its I) to the DC sums, and every bin differed."""
    plan = power_paths.mkplan(10, buf_len, ds=5, n_hops=1)
    used = buf_len // 5
    assert power_paths.is_big(plan) and -(-(buf_len // 2) // 5) > used // 2
    x = power_paths.hop_input(np.random.default_rng(buf_len), "dc", (2, 1, buf_len), False)
    win = power.window_table("blackman", 1024)
    want, want_smp = port.power_scan(power_paths.oracle_params(plan), win, x, 2, 1)
    sc = power.PowerScanner(plan, win)
    sc.scanner(x, 2)
    avg, smp = sc.read()
    assert sc.last_path()["kernel"] == "big_load"
    sc.close()
    assert np.array_equal(smp, want_smp)
    assert np.array_equal(avg, want)
