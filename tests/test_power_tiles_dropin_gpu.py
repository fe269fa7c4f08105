"""The rx_power shell in tile mode (RXB200_TILE_RATE) on the replay device: per sweep and tile, one retune, one flush
read and one burst of the filter's lead plus one pass, gathered from reads whose caps do not divide a burst.  The file
is laid out the way the shell reads it, so the CSV bytes must equal csv_rows of the port on the model's hop buffers.  A
stream that runs dry mid-sweep reports what it got and exits 0; each refusal exits 1 before any output file exists."""
import os
import subprocess

import numpy as np
import pytest

import power_paths
import power_tiles as ptl
from rx_tools_b200 import power

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RX_POWER = os.path.join(ROOT, "host", "rx_power_b200")
TSTR = "2026-01-01, 00:00:00"
FLUSH = 16384                        # BUFFER_DUMP: complex elements of the flush read after each retune


@pytest.fixture(scope="module", autouse=True)
def built():
    subprocess.run(["make", "-C", os.path.join(ROOT, "host"), "-s"], check=True)


def _run(cmd, env):
    e = dict(os.environ)
    e.update(env)
    return subprocess.run(cmd, capture_output=True, env=e, timeout=300)


def _layout(bursts, reads, seed):
    """The replay file for bursts (in the order the shell takes them, every one after a retune): what each flush read
    takes, as the read caps cycle, then the burst."""
    rng = np.random.default_rng(seed)
    k, parts = 0, []

    def take(n):
        nonlocal k
        got = min(n, reads[k % len(reads)])
        k += 1
        return got

    for b in bursts:
        parts.append(rng.integers(-30000, 30000, size=2 * take(FLUSH), dtype=np.int32).astype(np.int16))
        need, have = b.size // 2, 0
        while have < need:
            have += take(need - have)
        parts.append(b)
    return np.concatenate(parts)


def _shell_case(name, n_sweeps):
    """The shape as the shell plans it (its own filter, one pass per burst) and n_sweeps sweeps of bursts."""
    plan, win, tl, tiles, offs, dd = ptl.shape(name)
    assert "taps" not in ptl.SHAPES[name] and tl.n_tiles > 1
    sweeps = [ptl.bursts(name, seed=100 * s, n_pass=1) for s in range(n_sweeps)]
    return plan, tl, tiles, offs, dd, sweeps


def _port_tiles(port, plan, window, tl, tiles, offs, dd, bursts):
    """The port's accumulators over (tile index, burst) pairs: each burst's hop buffers into its tile's rows."""
    n = 1 << plan.bin_e
    avg, smp = np.zeros((plan.n_hops, n), np.int64), np.zeros(plan.n_hops, np.int32)
    for t, x in bursts:
        b, e, _ = tiles[t]
        hb = ptl.burst_buffers(x, tl.capture_rate, offs[b:e], dd, plan.buf_len)
        port.power_scan(power_paths.oracle_params(plan), window, hb, hb.shape[0], e - b, avg[b:e], smp[b:e])
    return avg, smp


@pytest.mark.parametrize("name,crop,win,cap,reads", [("fm_band_6M", "0%", "hamming", "6000000", (5000, 12345, 777)),
                                                      ("hf_crop285_10M", "28.5%", "blackman", "10000000",
                                                       (40000, 3, 9999))])
def test_tile_mode_csv(tmp_path, port, name, crop, win, cap, reads):
    s = ptl.SHAPES[name]
    plan, tl, tiles, offs, dd, sweeps = _shell_case(name, 2)
    window = power.window_table(win, 1 << plan.bin_e)
    f = tmp_path / "cap.cs16"
    _layout([x for sw in sweeps for x in sw], reads, 3).tofile(f)
    out = tmp_path / "out.csv"
    r = _run([RX_POWER, "-f", s["freq"], "-c", crop, "-w", win, "-i", "1h",
              "-d", f"driver=file,path={f},reads={':'.join(map(str, reads))}", str(out)],
             {"RXB200_TILE_RATE": cap, "RXB200_MAX_SWEEPS": "2", "RXB200_FIXED_TIME": TSTR})
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    assert (f"Tile mode: {tl.n_tiles} tiles of up to {tl.hops_per_tile} hops, {tl.capture_rate} Hz, "
            f"decimation {tl.decim}, {tl.n_taps} taps") in r.stderr.decode()
    avg, smp = _port_tiles(port, plan, window, tl, tiles, offs, dd, [(t, x) for sw in sweeps for t, x in enumerate(sw)])
    assert (smp == smp[0]).all() and smp[0] > 0
    assert open(out).read() == power.csv_rows(plan, avg, smp, TSTR)


def test_tile_mode_stream_running_dry_mid_sweep(tmp_path, port):
    """One whole sweep, then the second sweep's first tile, then half a burst: the shell reports those and exits 0."""
    name = "peak_hold"
    s = ptl.SHAPES[name]
    plan, tl, tiles, offs, dd, sweeps = _shell_case(name, 2)
    window = power.window_table(s["window"], 1 << plan.bin_e)
    taken = sweeps[0] + sweeps[1][:1]
    data = _layout(taken + [sweeps[1][1]], (7000,), 4)
    f = tmp_path / "cap.cs16"
    data[:data.size - sweeps[1][1].size // 2].tofile(f)
    out = tmp_path / "out.csv"
    r = _run([RX_POWER, "-f", s["freq"], "-c", "10%", "-P", "-w", s["window"], "-i", "1h",
              "-d", f"driver=file,path={f},reads=7000", str(out)],
             {"RXB200_TILE_RATE": str(s["cap"]), "RXB200_FIXED_TIME": TSTR})
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    pairs = [(t, x) for t, x in enumerate(sweeps[0])] + [(0, sweeps[1][0])]
    avg, smp = _port_tiles(port, plan, window, tl, tiles, offs, dd, pairs)
    b, e, _ = tiles[0]
    assert (smp[b:e] == 2 * smp[-1]).all() and (smp[e:] == smp[-1]).all() and smp[-1] > 0
    assert open(out).read() == power.csv_rows(plan, avg, smp, TSTR)


@pytest.mark.parametrize("env", [{"RXB200_TILE_RATE": "6000000", "RXB200_CAPTURE_RATE": "40000000"},
                                 {"RXB200_TILE_RATE": "6000000", "RXB200_GPUS": "2"},
                                 {"RXB200_TILE_RATE": "2499999"},
                                 {"RXB200_TILE_RATE": "0"}])
def test_tile_mode_refusals_exit_before_any_output(tmp_path, env):
    f = tmp_path / "cap.cs16"
    np.zeros(1024, np.int16).tofile(f)
    out = tmp_path / "out.csv"
    r = _run([RX_POWER, "-f", "88M:108M:10k", "-d", f"driver=file,path={f}", str(out)], env)
    assert r.returncode == 1, r.stderr.decode()[-2000:]
    assert "Tile mode" in r.stderr.decode()
    assert not out.exists()
