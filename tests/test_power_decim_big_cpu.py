"""rx_power -F on hop buffers beyond shared memory, CPU side: the port equals the unmodified reference at the
planner's shapes (bins of 50, 40, 10 and 1 Hz, -F 0 and -F 9, one with peak hold), and reproduces every hash of
tests/golden/power_decim_big_golden.json, so the fixture is pinned from both sides."""
import json
import os

import numpy as np
import pytest

import oracle
from rx_tools_b200.synth import digest

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLD = json.load(open(os.path.join(G, "power_decim_big_golden.json")))


def _input(e):
    rng = np.random.default_rng(e["seed"])
    return rng.integers(-3000, 3001, size=(e["n_pass"], e["n_hops"], e["buf_len"]), dtype=np.int32).astype(np.int16)


def _params(e):
    return oracle.PowerParams(bin_e=e["bin_e"], buf_len=e["buf_len"], downsample=e["downsample"],
                              downsample_passes=e["downsample_passes"], comp_fir_size=e["fir"], boxcar=0,
                              peak_hold=e["peak_hold"])


@pytest.mark.ref
@pytest.mark.parametrize("name", sorted(GOLD))
def test_port_equals_reference(name, port, ref_power):
    e = GOLD[name]
    plan = ref_power.setup(e["freq"], 0.0, 0, e["fir"], e["peak_hold"], e["window"])
    assert (plan.bin_e, plan.buf_len, plan.downsample, plan.downsample_passes) == \
        (e["bin_e"], e["buf_len"], e["downsample"], e["downsample_passes"])
    assert plan.buf_len * 2 > 227 * 1024
    x = _input(e)
    avg_r, smp_r = ref_power.scan(x, e["n_pass"])
    win, _ = ref_power.tables()
    assert np.array_equal(win, port.window_table(e["window"], 1 << e["bin_e"]))
    avg_p, smp_p = port.power_scan(_params(e), win, x, e["n_pass"], e["n_hops"])
    assert np.array_equal(smp_p, smp_r)
    assert np.array_equal(avg_p, avg_r)
    assert digest(avg_r) == e["avg_sha256"]


@pytest.mark.parametrize("name", sorted(GOLD))
def test_port_reproduces_golden(name, port):
    e = GOLD[name]
    win = port.window_table(e["window"], 1 << e["bin_e"])
    avg, smp = port.power_scan(_params(e), win, _input(e), e["n_pass"], e["n_hops"])
    assert avg.any()
    assert digest(avg) == e["avg_sha256"]
    assert smp.tolist() == e["samples"]


# -F geometries no planner makes, with a hop buffer beyond shared memory: power_big_decim does not serve them, so
# rxb200_power_create rejects them before it looks for a device (the accepted planner shapes run in
# tests/test_power_decim_big_gpu.py)
@pytest.mark.parametrize("bin_e,buf_len,ds,passes", [
    (14, 262144, 8, 2),      # downsample != 2^passes
    (12, 131080, 4, 2),      # buf_len not a multiple of 2 N downsample: the last block would read earlier passes' leftovers
    (14, 131072, 4, 0),      # downsample without passes or boxcar
])
def test_unsupported_big_geometries_are_rejected(bin_e, buf_len, ds, passes):
    from rx_tools_b200 import _lib, power
    plan = power.Plan(n_hops=1, bin_e=bin_e, buf_len=buf_len, downsample=ds, downsample_passes=passes, comp_fir_size=9,
                      boxcar=0, peak_hold=0, rate=2000000, crop=0.0, first_freq=100000000, freq_step=2000000,
                      bin_size_hz=0.0)
    with pytest.raises(_lib.Rxb200Error) as e:
        power.PowerScanner(plan, "hamming")
    assert e.value.code == _lib.EUNSUPPORTED
