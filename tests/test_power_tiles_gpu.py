"""Wide rx_power sweeps in tiles on the GPU (rxb200_power_mix_accumulate_burst*): every named shape and every tile
through the host and the device entries against the burst model, the port and the reference's golden hashes, with the
CSV of the whole tiled sweep; M = 1, T = 1 against a plain rx_power handle; a burst past the scratch bound; bursts
between continuous calls leaving the carried stream alone; and refusals that change nothing."""
import hashlib
import json
import os

import numpy as np
import pytest

import fm_ddc as fdd
import fm_handles as fh
import power_mix as pm
import power_paths
import power_tiles as ptl
from rx_tools_b200 import _lib, power

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "power_tiles_golden.json")
TSTR = "2026-01-01, 00:00:00"
SCRATCH = 64 << 20                   # RXB200_POWER_MIX_SCRATCH_BYTES


def _same(a, b):
    return all(np.array_equal(u, v) for u, v in zip(a.read(), b.read()))


def _device_copy(x):
    """x on the device 4 bytes past a tensor's start, and that pointer."""
    torch = fh.torch()
    buf = torch.from_numpy(np.concatenate([np.zeros(2, np.int16), np.asarray(x, np.int16)])).cuda()
    return buf, buf.data_ptr() + 4


@pytest.mark.parametrize("name", sorted(ptl.SHAPES))
def test_named_shape_every_tile_host_and_device(name, port):
    g = json.load(open(GOLDEN))[name]
    plan, win, tl, tiles, offs, dd, bs = ptl.case_input(name)
    assert [pm.digest(b) for b in bs] == g["burst_sha256"]
    host = power.PowerMix(plan, tl.capture_rate, offs, dd, win)
    dev = power.PowerMix(plan, tl.capture_rate, offs, dd, win)
    assert host.lead == ptl.lead(dd[0], dd[1].size)
    per, hb = ptl.tile_buffers(name)
    keep = []
    for (b, e, _), x, want in zip(tiles, bs, per):
        # each tile alone against the model through the port
        one = power.PowerMix(plan, tl.capture_rate, offs, dd, win)
        one.accumulate_burst(b, e, x)
        avg, smp = one.read()
        wavg, wsmp = port.power_scan(power_paths.oracle_params(plan), win, want, want.shape[0], e - b)
        assert np.array_equal(avg[b:e], wavg) and np.array_equal(smp[b:e], wsmp), (name, b, e)
        assert not avg[:b].any() and not avg[e:].any() and not smp[:b].any() and not smp[e:].any()
        one.close()
        host.accumulate_burst(b, e, x)
        buf, p = _device_copy(x)
        keep.append(buf)
        dev.accumulate_burst_device(b, e, p, x.size, sync=False)
    avg, smp = host.read()
    assert pm.digest(avg) == g["avg_sha256"] and smp.tolist() == g["samples"], name
    wavg, wsmp = pm.port_result(port, plan, win, hb)
    assert np.array_equal(avg, wavg) and np.array_equal(smp, wsmp)
    assert _same(host, dev)
    csv = dev.csv_rows_device(TSTR)
    assert csv == power.csv_rows(plan, wavg, wsmp, TSTR)
    assert hashlib.sha256(csv.encode()).hexdigest() == g["csv_sha256"]
    assert host.kernel_ms() > 0
    host.close()
    dev.close()


@pytest.mark.parametrize("path", ["rms", "fft8", "generic", "big_decim"])
def test_identity_burst_is_a_plain_power_handle(path):
    """M = 1, T = 1, h = {1}, S = 0 and offsets 0: G = 0, and each pass of the burst is the buffer of every hop in the
    range."""
    plan = dict(rms=power_paths.mkplan(0, 16384, n_hops=5), fft8=power_paths.mkplan(10, 16384, n_hops=5),
                generic=power_paths.mkplan(8, 4096, n_hops=5),
                big_decim=power_paths.mkplan(8, 1 << 17, ds=8, passes=3, fir=9, boxcar=0, n_hops=5))[path]
    rng = np.random.default_rng(len(path))
    n_pass, hb, he = 3, 1, 4
    x = rng.integers(-32768, 32768, size=n_pass * plan.buf_len, dtype=np.int32).astype(np.int16)
    win = power.window_table("hann", 1 << plan.bin_e)
    mx = power.PowerMix(plan, 2_000_000, [0] * plan.n_hops, (1, np.ones(1, np.int32), 0), win)
    assert mx.lead == 0
    sc = power.PowerScanner(plan, win)
    mx.accumulate_burst(hb, he, x)
    sc.scanner(np.repeat(x.reshape(n_pass, 1, plan.buf_len), he - hb, axis=1), n_pass, hb, he)
    assert mx.last_path()["kernel"] == path == sc.last_path()["kernel"]
    assert _same(mx, sc)
    mx.close()
    sc.close()


def test_burst_past_the_scratch_bound_equals_one_group():
    """A burst over 300 hops needs three groups of passes; over ranges of 4 hops the same burst is one group each."""
    plan = power_paths.mkplan(4, 16384, n_hops=300)
    rng = np.random.default_rng(5)
    R = 10_000_000
    offs = [int(v) for v in rng.integers(-R // 2 + 1, R // 2, size=plan.n_hops)]
    dd = (2, fdd.lowpass(9, 0.2), 15)
    n_pass = 2 * (SCRATCH // (plan.n_hops * plan.buf_len * 2)) + 3
    win = power.window_table("blackman", 16)
    big, small = power.PowerMix(plan, R, offs, dd, win), power.PowerMix(plan, R, offs, dd, win)
    x = rng.integers(-20000, 20000, size=big.burst_int16(n_pass), dtype=np.int32).astype(np.int16)
    assert 4 * plan.buf_len * 2 * n_pass <= SCRATCH
    big.accumulate_burst(0, plan.n_hops, x)
    for b in range(0, plan.n_hops, 4):
        small.accumulate_burst(b, b + 4, x)
    assert _same(big, small)
    big.close()
    small.close()


def test_burst_between_continuous_calls_leaves_the_stream_alone():
    """accumulate + burst + accumulate = the two accumulates alone + the burst alone (no -P, so the sums add)."""
    plan, win, tl, tiles, offs, dd, bs = ptl.case_input("fm_band_6M")
    R = tl.capture_rate
    x = pm.capture(3 * dd[0] * plan.buf_len // 2, R, offs, 31)
    cut = dd[0] * plan.buf_len
    b, e, _ = tiles[1]
    mixed, plain, burst = (power.PowerMix(plan, R, offs, dd, win) for _ in range(3))
    mixed.accumulate(x[:cut])
    mixed.accumulate_burst(b, e, bs[1])
    mixed.accumulate(x[cut:])
    plain.accumulate(x[:cut])
    plain.accumulate(x[cut:])
    burst.accumulate_burst(b, e, bs[1])
    (a1, s1), (a2, s2), (a3, s3) = mixed.read(), plain.read(), burst.read()
    assert np.array_equal(a1, a2 + a3) and np.array_equal(s1, s2 + s3)
    for h in (mixed, plain, burst):
        h.close()


def test_refusals_change_nothing():
    plan, win, tl, tiles, offs, dd, bs = ptl.case_input("peak_hold")
    R, n = tl.capture_rate, plan.n_hops
    b, e, _ = tiles[0]
    x = bs[0]
    x2 = ptl.bursts("peak_hold", seed=1)[0]
    h, ref = power.PowerMix(plan, R, offs, dd, win), power.PowerMix(plan, R, offs, dd, win)
    cont = pm.capture(2 * dd[0] * plan.buf_len // 2, R, offs, 41)
    cut = dd[0] * plan.buf_len
    for m in (h, ref):
        m.accumulate(cont[:cut])
        m.accumulate_burst(b, e, x)
    before = h.read()
    buf, p = _device_copy(x)
    G2, pas = 2 * h.lead, h.pass_int16
    assert x.size == G2 + ptl.SHAPES["peak_hold"]["n_pass"] * pas
    for hb, he in ((-1, e), (e, e), (e, b), (0, n + 1), (n, n)):
        for call in (lambda: h.accumulate_burst(hb, he, x), lambda: h.accumulate_burst_device(hb, he, p, x.size, True)):
            with pytest.raises(_lib.Rxb200Error) as ex:
                call()
            assert ex.value.code == _lib.EINVAL, (hb, he)
    for size in (0, G2, G2 + pas - 2, G2 + pas + 2, G2 + 2 * pas - 2, pas):
        with pytest.raises(_lib.Rxb200Error) as ex:
            h.accumulate_burst_device(b, e, p, size, sync=True)
        assert ex.value.code == _lib.EUNSUPPORTED, size
        with pytest.raises(_lib.Rxb200Error) as ex:
            h.accumulate_burst(b, e, x[:size] if size <= x.size else np.concatenate([x, x[:2]]))
        assert ex.value.code == _lib.EUNSUPPORTED, size
    with pytest.raises(_lib.Rxb200Error) as ex:
        h.accumulate_burst_device(b, e, p + 2, x.size, sync=True)
    assert ex.value.code == _lib.EINVAL
    L = _lib.lib()
    assert L.rxb200_power_mix_accumulate_burst(h._m, b, e, None, x.size) == _lib.EINVAL
    assert L.rxb200_power_mix_accumulate_burst_device(h._m, b, e, None, x.size, 1) == _lib.EINVAL
    assert L.rxb200_power_mix_accumulate_burst(None, b, e, x.ctypes.data, x.size) == _lib.EINVAL
    assert L.rxb200_power_mix_lead(None) == _lib.EINVAL
    after = h.read()
    assert all(np.array_equal(u, v) for u, v in zip(before, after))
    # nor did they move the carried stream: both handles go on alike
    for m in (h, ref):
        m.accumulate(cont[cut:])
        m.accumulate_burst(b, e, x2)
    assert _same(h, ref)
    h.close()
    ref.close()
