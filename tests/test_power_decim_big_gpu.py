"""rx_power -F on hop buffers beyond shared memory (power_big_decim + the global-memory FFT path): PowerScanner is
bit-exact with the port oracle and with tests/golden/power_decim_big_golden.json (the reference's own hashes), for
the planner's shapes, for every pass count P = 1..10 with and without the droop FIR, for several N-blocks per hop
buffer, through csv_dbm on the device, and through the drop-in rx_power_b200."""
import json
import os
import subprocess

import numpy as np
import pytest

import oracle
from rx_tools_b200 import power
from rx_tools_b200.synth import digest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")
GOLD = json.load(open(os.path.join(G, "power_decim_big_golden.json")))
RX_POWER = os.path.join(ROOT, "host", "rx_power_b200")


def _input(e):
    rng = np.random.default_rng(e["seed"])
    return rng.integers(-3000, 3001, size=(e["n_pass"], e["n_hops"], e["buf_len"]), dtype=np.int32).astype(np.int16)


def _oracle_params(plan):
    return oracle.PowerParams(bin_e=plan.bin_e, buf_len=plan.buf_len, downsample=plan.downsample,
                              downsample_passes=plan.downsample_passes, comp_fir_size=plan.comp_fir_size,
                              boxcar=plan.boxcar, peak_hold=plan.peak_hold)


def _plan(e):
    plan = power.plan_range(e["freq"], 0.0, boxcar=0, comp_fir_size=e["fir"], peak_hold=e["peak_hold"])
    assert (plan.n_hops, plan.bin_e, plan.buf_len, plan.downsample, plan.downsample_passes) == \
        (e["n_hops"], e["bin_e"], e["buf_len"], e["downsample"], e["downsample_passes"])
    assert plan.buf_len * 2 > 227 * 1024
    return plan


def _check_twice(plan, win, x, n_pass, want, want_smp):
    """One scanner() call equals the port; a second one doubles the sums (or holds the max); reset() zeroes."""
    sc = power.PowerScanner(plan, win)
    sc.scanner(x, n_pass)
    avg, smp = sc.read()
    assert np.array_equal(smp, want_smp)
    bad = np.argwhere(avg != want)
    assert bad.size == 0, (bad[:4], avg[tuple(bad[0])], want[tuple(bad[0])])
    assert sc.kernel_ms() > 0.0
    assert _lib_launches(sc) == n_pass * plan.n_hops * (3 + plan.bin_e)
    sc.scanner(x, n_pass)
    avg2, smp2 = sc.read()
    assert np.array_equal(avg2, want if plan.peak_hold else 2 * want)
    assert np.array_equal(smp2, 2 * want_smp)
    sc.reset()
    z, zs = sc.read()
    assert not z.any() and not zs.any()
    sc.close()
    return avg


def _lib_launches(sc):
    from rx_tools_b200 import _lib
    return int(_lib.lib().rxb200_power_last_launches(sc._h))


@pytest.mark.parametrize("name", sorted(GOLD))
def test_planner_shapes(name, port):
    e = GOLD[name]
    plan = _plan(e)
    win = power.window_table(e["window"], 1 << plan.bin_e)
    x = _input(e)
    want, want_smp = port.power_scan(_oracle_params(plan), win, x, e["n_pass"], plan.n_hops)
    assert digest(want) == e["avg_sha256"]
    avg = _check_twice(plan, win, x, e["n_pass"], want, want_smp)
    assert digest(avg) == e["avg_sha256"]
    assert want_smp.tolist() == e["samples"]


def _explicit_plan(P, fir, peak, bin_e, buf_len, n_hops):
    return power.Plan(n_hops=n_hops, bin_e=bin_e, buf_len=buf_len, downsample=1 << P, downsample_passes=P,
                      comp_fir_size=fir, boxcar=0, peak_hold=peak, rate=2000000, crop=0.0, first_freq=100000000,
                      freq_step=2000000, bin_size_hz=0.0)


@pytest.mark.parametrize("fir", [0, 9])
@pytest.mark.parametrize("P", list(range(1, 11)))
def test_every_pass_count(P, fir, port):
    """bin_e = 16 - P, buf_len 131072, three hops: full-scale input wraps every pass and the FIR; peak hold on P = 3, 6, 9."""
    peak = 1 if P % 3 == 0 else 0
    plan = _explicit_plan(P, fir, peak, 16 - P, 131072, 3)
    rng = np.random.default_rng(1000 + 10 * P + fir)
    x = rng.integers(-32768, 32768, size=(2, 3, plan.buf_len), dtype=np.int32).astype(np.int16)
    win = power.window_table("hamming" if fir else "blackman", 1 << plan.bin_e)
    want, want_smp = port.power_scan(_oracle_params(plan), win, x, 2, 3)
    assert want.any()
    _check_twice(plan, win, x, 2, want, want_smp)


def test_several_blocks_per_hop_buffer(port):
    """P = 3, bin_e 12, buf_len 262144: the decimated span is four N-blocks."""
    plan = _explicit_plan(3, 9, 0, 12, 262144, 2)
    rng = np.random.default_rng(77)
    x = rng.integers(-32768, 32768, size=(3, 2, plan.buf_len), dtype=np.int32).astype(np.int16)
    win = power.window_table("hann-poisson", 1 << plan.bin_e)
    want, want_smp = port.power_scan(_oracle_params(plan), win, x, 3, 2)
    assert want_smp.tolist() == [3 * 4 * 8] * 2
    _check_twice(plan, win, x, 3, want, want_smp)


def test_csv_rows_on_device():
    e = GOLD["f10_fir9"]
    plan = _plan(e)
    sc = power.PowerScanner(plan, e["window"])
    sc.scanner(_input(e), e["n_pass"])
    avg, smp = sc.read()
    assert digest(avg) == e["avg_sha256"]
    assert sc.csv_rows_device() == power.csv_rows(plan, avg, smp)
    sc.close()


def _power_capture(plan, hop_bufs, n_pass):
    """What the shell reads: per hop a flush read of 16384 elements after every retune, then buf_len elements whose
    first buf_len int16 are the hop buffer."""
    parts = []
    rng = np.random.default_rng(5)
    for p in range(n_pass):
        for h in range(plan.n_hops):
            retune = plan.n_hops > 1 or p == 0
            if retune:
                parts.append(rng.integers(-50, 50, size=2 * 16384, dtype=np.int32).astype(np.int16))
            parts.append(hop_bufs[p, h])
            parts.append(rng.integers(-50, 50, size=plan.buf_len, dtype=np.int32).astype(np.int16))
    return np.concatenate(parts)


def test_dropin_rx_power(tmp_path, port):
    """rx_power_b200 -f 100M:100.1M:40 -F 9 -w hamming over the replay device writes csv_dbm's bytes of the port."""
    subprocess.run(["make", "-C", os.path.join(ROOT, "host"), "-s"], check=True)
    freq, n_pass = "100M:100.1M:40", 3
    plan = power.plan_range(freq, 0.0, boxcar=0, comp_fir_size=9)
    rng = np.random.default_rng(40)
    hb = rng.integers(-3000, 3001, size=(n_pass, plan.n_hops, plan.buf_len), dtype=np.int32).astype(np.int16)
    cap = tmp_path / "cap.cs16"
    _power_capture(plan, hb, n_pass).tofile(cap)
    out = tmp_path / "out.csv"
    env = dict(os.environ)
    env.update({"RXB200_MAX_SWEEPS": str(n_pass), "RXB200_FIXED_TIME": "2026-01-01, 00:00:00"})
    r = subprocess.run([RX_POWER, "-f", freq, "-c", "0%", "-F", "9", "-w", "hamming", "-i", "1h",
                        "-d", f"driver=file,path={cap}", str(out)], capture_output=True, env=env, timeout=300)
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    avg, smp = port.power_scan(_oracle_params(plan), power.window_table("hamming", 1 << plan.bin_e), hb, n_pass, plan.n_hops)
    assert open(out).read() == power.csv_rows(plan, avg, smp, "2026-01-01, 00:00:00")


@pytest.mark.parametrize("bin_e,buf_len", [(16, 262144), (12, 16384)])
def test_downsample_one_with_passes_is_not_decimated(bin_e, buf_len, port):
    """downsample 1 with downsample_passes set (no planner makes it): neither the global-memory path (bin_e 16) nor the
    shared-memory kernel (bin_e 12) runs a pass -- both transform the hop buffer as is, the same integers as a plan
    without passes."""
    plan = _explicit_plan(2, 9, 0, bin_e, buf_len, 1)
    plan.downsample = 1
    rng = np.random.default_rng(bin_e)
    x = rng.integers(-3000, 3001, size=(2, 1, buf_len), dtype=np.int32).astype(np.int16)
    win = power.window_table("hamming", 1 << bin_e)
    plain = oracle.PowerParams(bin_e=bin_e, buf_len=buf_len)
    want, want_smp = port.power_scan(plain, win, x, 2, 1)
    sc = power.PowerScanner(plan, win)
    sc.scanner(x, 2)
    avg, smp = sc.read()
    assert np.array_equal(avg, want) and np.array_equal(smp, want_smp)
    sc.close()


def test_interleaved_handles_with_different_spans(port):
    """Two scanners in one process whose power_big_decim tiles need very different shared memory (P = 8: ~70 KB,
    P = 4: a few KB), run alternately: each launch still gets the shared memory it planned."""
    big, small = GOLD["f1_fir9"], GOLD["f10_fir9"]
    plans = [_plan(big), _plan(small)]
    wins = [power.window_table(e["window"], 1 << p.bin_e) for e, p in zip((big, small), plans)]
    xs = [_input(big)[:1], _input(small)[:1]]
    wants = [port.power_scan(_oracle_params(p), w, x, 1, 1)[0] for p, w, x in zip(plans, wins, xs)]
    scs = [power.PowerScanner(p, w) for p, w in zip(plans, wins)]
    for k in (0, 1, 0, 1):
        scs[k].scanner(xs[k], 1)
    for sc, want in zip(scs, wants):
        avg, _ = sc.read()
        assert np.array_equal(avg, 2 * want)
        sc.close()
