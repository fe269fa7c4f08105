"""rx_power hops of one capture (rxb200_power_mix_*) on the GPU: power_ddc_kernel alone (rxb200_power_ddc_device)
against the numpy model over every int16 value, phases near the 2^32 wrap and past 2^40, both accumulators and unaligned
sources; the identity handle against a plain rx_power handle on every accumulate path; the named shapes against the
model + port and the reference's golden hashes; the phase and history carry across calls, member resets, handle resets
and calls longer than the scratch bound; the device entry point; refusals that leave no trace; and the CSV."""
import hashlib
import json
import os

import numpy as np
import pytest

import fm_ddc as fdd
import fm_handles as fh
import power_mix as pm
import power_paths
from rx_tools_b200 import _lib, power

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "power_mix_golden.json")
TSTR = "2026-01-01, 00:00:00"
ONE = np.ones(1, np.int32)
SCRATCH = 64 << 20                   # RXB200_POWER_MIX_SCRATCH_BYTES


def _tap_sets(decim, n_taps, seed):
    """(taps, shift): a Q15 low-pass (int32 accumulator unless T is large) and large random taps at a small shift
    (int64 accumulator, saturating outputs)."""
    rng = np.random.default_rng(seed)
    return [(fdd.lowpass(n_taps, 0.45 / decim), 15),
            (rng.integers(-(1 << 20), 1 << 20, size=n_taps).astype(np.int32), 3)]


CASES = sorted({(m, t) for m in (1, 2, 7, 64, 4096) for t in (1, m, 4 * m + 1, 8192) if t <= 8192})


@pytest.mark.parametrize("decim,n_taps", CASES)
def test_kernel_entry_equals_model(decim, n_taps):
    torch = fh.torch()
    rate, f = 39_160_828, -9_790_207
    x = fh.every_int16(decim * 5 + n_taps)
    n_max = min(65536, max(decim + 3, (1 << 22) * decim // n_taps))
    srcs = {off16: torch.from_numpy(np.concatenate([np.zeros(off16, np.int16), x])).cuda() for off16 in (0, 2, 8)}
    dst = torch.zeros(2 * (65536 // decim) + 64, dtype=torch.int16, device="cuda")
    for taps, shift in _tap_sets(decim, n_taps, decim + n_taps):
        dd = (decim, taps, shift)
        assert fdd.wide(taps, shift) or shift == 15                 # the random taps take the int64 accumulator
        for n0 in (0, (1 << 32) - 3 * decim - 5, (1 << 40) + 3):
            for off16, src in srcs.items():
                for n in sorted({n_max, n_max - 1, decim - 1, 2 * decim + 1, 1}):
                    if n < 1:
                        continue
                    dst.fill_(0)
                    power.power_ddc_device(rate, f, n0, dd, src.data_ptr() + 2 * off16, n, dst.data_ptr())
                    torch.cuda.synchronize()
                    want, _ = pm.ddc(x[:2 * n], rate, f, dd, n0)
                    assert want.size == 2 * (n // decim)
                    got = dst[:want.size].cpu().numpy()
                    bad = np.flatnonzero(got != want)
                    assert bad.size == 0, (decim, n_taps, shift, n0, off16, n, bad[:4])
                    assert not dst[want.size:].any().item(), (decim, n_taps, n0, n)


def test_kernel_entry_offsets_and_refusals():
    torch = fh.torch()
    x = fh.every_int16(7)
    src = torch.from_numpy(x).cuda()
    dst = torch.zeros(x.size, dtype=torch.int16, device="cuda")
    dd = (3, fdd.lowpass(17, 0.1), 15)
    for rate, f in ((20_000_000, 5_000_000), (20_000_000, -5_000_000), (7, 3), (7, -3), (61_440_000, 30_719_999)):
        power.power_ddc_device(rate, f, 12345, dd, src.data_ptr(), 65536, dst.data_ptr())
        torch.cuda.synchronize()
        want, _ = pm.ddc(x, rate, f, dd, 12345)
        assert dst[:want.size].cpu().numpy().tobytes() == want.tobytes(), (rate, f)
    p = src.data_ptr()
    for args, code in (((20_000_000, 10_000_000, 0, dd, p, 8, p), _lib.EINVAL),
                       ((0, 0, 0, dd, p, 8, p), _lib.EINVAL),
                       ((20_000_000, 0, 0, (0, ONE, 0), p, 8, p), _lib.EINVAL),
                       ((20_000_000, 0, 0, dd, p + 2, 8, p), _lib.EINVAL),
                       ((20_000_000, 0, 0, dd, None, 8, p), _lib.EINVAL)):
        with pytest.raises(_lib.Rxb200Error) as e:
            power.power_ddc_device(*args)
        assert e.value.code == code, args


IDENTITY_PLANS = {
    "rms": power_paths.mkplan(0, 16384, n_hops=3),
    "fft8": power_paths.mkplan(10, 16384, n_hops=3),
    "generic": power_paths.mkplan(8, 4096, n_hops=3),
    "big_load": power_paths.mkplan(10, 1 << 17, n_hops=2),
    "big_decim": power_paths.mkplan(8, 1 << 17, ds=8, passes=3, fir=9, boxcar=0, n_hops=2),
}


@pytest.mark.parametrize("path", sorted(IDENTITY_PLANS))
def test_identity_is_a_plain_power_handle(path):
    """M = 1, h = {1}, S = 0 and every offset 0: each pass of the capture is every hop's buffer."""
    plan = IDENTITY_PLANS[path]
    n_pass = 3
    rng = np.random.default_rng(len(path))
    x = rng.integers(-32768, 32768, size=n_pass * plan.buf_len, dtype=np.int32).astype(np.int16)
    win = power.window_table("hamming", 1 << plan.bin_e)
    mx = power.PowerMix(plan, 2_000_000, [0] * plan.n_hops, (1, ONE, 0), win)
    sc = power.PowerScanner(plan, win)
    mx.accumulate(x)
    hb = np.repeat(x.reshape(n_pass, 1, plan.buf_len), plan.n_hops, axis=1)
    sc.scanner(hb, n_pass)
    assert mx.last_path()["kernel"] == path == sc.last_path()["kernel"]
    (a1, s1), (a2, s2) = mx.read(), sc.read()
    assert np.array_equal(s1, s2) and np.array_equal(a1, a2)
    mx.close()
    sc.close()


@pytest.mark.parametrize("name", sorted(pm.SHAPES))
def test_named_shape_equals_model_port_and_reference(name, port):
    g = json.load(open(GOLDEN))[name]
    plan, win, R, offs, dd, x = pm.case_input(name)
    assert pm.digest(x) == g["capture_sha256"]
    mx = power.PowerMix(plan, R, offs, dd, win)
    mx.accumulate(x)
    avg, smp = mx.read()
    assert pm.digest(avg) == g["avg_sha256"] and smp.tolist() == g["samples"], name
    hb = pm.Model(R, offs, dd, plan.buf_len).hop_buffers(x)
    wavg, wsmp = pm.port_result(port, plan, win, hb)
    assert np.array_equal(avg, wavg) and np.array_equal(smp, wsmp)
    csv = mx.csv_rows_device(TSTR)
    assert csv == power.csv_rows(plan, wavg, wsmp, TSTR)
    assert hashlib.sha256(csv.encode()).hexdigest() == g["csv_sha256"]
    assert mx.kernel_ms() > 0
    mx.close()


def _fm_band(n_pass, seed=0):
    plan, win, R, offs, dd = pm.shape("fm_band")
    x = pm.capture(n_pass * dd[0] * plan.buf_len // 2, R, offs, 2000 + seed)
    return plan, win, R, offs, dd, x


def test_calls_of_1_3_2_passes_equal_one_call_of_6():
    plan, win, R, offs, dd, x = _fm_band(6)
    pas = dd[0] * plan.buf_len
    one, split = power.PowerMix(plan, R, offs, dd, win), power.PowerMix(plan, R, offs, dd, win)
    one.accumulate(x)
    a = 0
    for k in (1, 3, 2):
        split.accumulate(x[a:a + k * pas])
        a += k * pas
    assert all(np.array_equal(u, v) for u, v in zip(one.read(), split.read()))
    one.close()
    split.close()


def test_member_reset_keeps_phases_and_history(port):
    plan, win, R, offs, dd, x = _fm_band(4, 1)
    pas = dd[0] * plan.buf_len
    mx = power.PowerMix(plan, R, offs, dd, win)
    model = pm.Model(R, offs, dd, plan.buf_len)
    mx.accumulate(x[:2 * pas])
    model.hop_buffers(x[:2 * pas])
    mx.reset_accumulators()
    mx.accumulate(x[2 * pas:])
    avg, smp = mx.read()
    wavg, wsmp = pm.port_result(port, plan, win, model.hop_buffers(x[2 * pas:]))
    assert np.array_equal(avg, wavg) and np.array_equal(smp, wsmp)
    # a handle reset is a fresh handle
    mx.reset()
    fresh = power.PowerMix(plan, R, offs, dd, win)
    mx.accumulate(x[pas:3 * pas])
    fresh.accumulate(x[pas:3 * pas])
    assert all(np.array_equal(u, v) for u, v in zip(mx.read(), fresh.read()))
    mx.close()
    fresh.close()


def test_call_beyond_the_scratch_bound_equals_per_pass_calls():
    plan = power_paths.mkplan(4, 16384, n_hops=300)
    rng = np.random.default_rng(3)
    R = 10_000_000
    offs = [int(v) for v in rng.integers(-R // 2 + 1, R // 2, size=plan.n_hops)]
    dd = (2, fdd.lowpass(9, 0.2), 15)
    per_pass = plan.n_hops * plan.buf_len * 2
    n_pass = 2 * (SCRATCH // per_pass) + 3                       # three groups, the last one partial
    x = rng.integers(-20000, 20000, size=n_pass * dd[0] * plan.buf_len, dtype=np.int32).astype(np.int16)
    win = power.window_table("blackman", 16)
    big, small = power.PowerMix(plan, R, offs, dd, win), power.PowerMix(plan, R, offs, dd, win)
    big.accumulate(x)
    pas = dd[0] * plan.buf_len
    for p in range(n_pass):
        small.accumulate(x[p * pas:(p + 1) * pas])
    assert all(np.array_equal(u, v) for u, v in zip(big.read(), small.read()))
    big.close()
    small.close()


def test_device_entry_at_a_4_byte_offset_and_refusals_that_change_nothing():
    torch = fh.torch()
    plan, win, R, offs, dd, x = _fm_band(3, 2)
    pas = dd[0] * plan.buf_len
    host, dev = power.PowerMix(plan, R, offs, dd, win), power.PowerMix(plan, R, offs, dd, win)
    buf = torch.from_numpy(np.concatenate([np.zeros(2, np.int16), x])).cuda()
    p = buf.data_ptr() + 4
    for bad, code in ((pas - 2, _lib.EUNSUPPORTED), (pas + 2 * plan.buf_len, _lib.EUNSUPPORTED)):
        with pytest.raises(_lib.Rxb200Error) as e:
            dev.accumulate_device(p, bad, sync=True)
        assert e.value.code == code
    with pytest.raises(_lib.Rxb200Error) as e:
        dev.accumulate_device(p + 2, pas, sync=True)
    assert e.value.code == _lib.EINVAL
    with pytest.raises(_lib.Rxb200Error) as e:
        host.accumulate(x[:pas + 2])
    assert e.value.code == _lib.EUNSUPPORTED
    dev.accumulate_device(p, 0, sync=True)
    host.accumulate(x[:0])
    dev.accumulate_device(p, pas, sync=False)
    dev.accumulate_device(p + 2 * pas, 2 * pas, sync=True)
    host.accumulate(x)
    assert all(np.array_equal(u, v) for u, v in zip(host.read(), dev.read()))
    assert host.csv_rows_device(TSTR) == dev.csv_rows_device(TSTR)
    host.close()
    dev.close()
