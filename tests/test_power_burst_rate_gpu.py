"""rx_power bursts at a device rate (include/rxb200.h, "Bursts at a device rate"): a handle with
rxb200_power_mix_set_burst_device_rate takes device-rate bursts, and each must accumulate exactly what the stateless
resampler (a fresh rxb200_resample handle, zeros before the burst) followed, from output E = ceil((J - 1) L / N) on, by
the capture-rate burst call of a handle without one would.  Ragged hop ranges, one and three passes, int32 and int64
DDC accumulators, a burst of the wrong length (refused, nothing changes), stream calls around bursts (unaffected) and
the exclusion of set_device_rate and set_burst_device_rate."""
import numpy as np
import pytest

import resample as rsm
from rx_tools_b200 import _lib, power
from rx_tools_b200 import resample as rs

pytestmark = pytest.mark.gpu

# (sweep, tile cap, device rate, ddc taps (T, S) or None for the planner's filter): tiles of several hops
CASES = {
    "fft_3.2M": ("100M:103M:1k", 10_000_000, 3_200_000, None),          # 2 hops of 2048 bins, one per tile, 15/16
    "rms_3.2M": ("100M:110M:1M", 10_000_000, 3_200_000, None),          # 10 hops at 1 M, 2 per tile, 15/16
    "rms_wide_acc": ("100M:110M:1M", 10_000_000, 4_400_000, (65, 17)),  # 3 per tile, 10/11, int64 DDC sums
    "rms_10.24M": ("100M:120M:2M", 12_000_000, 10_240_000, None),       # 4 per tile at 2 M, 125/128
}


def _case(name):
    freq, cap, R_dev, taps = CASES[name]
    plan = power.plan_range(freq)
    tl, tiles, offs = power.plan_tiles(plan, cap, device_rate=R_dev)
    assert tl.n_tiles > 1 and tl.capture_rate <= R_dev
    T, S = (tl.n_taps, 15) if taps is None else taps
    dd = (tl.decim, power.ddc_lowpass(tl.decim, T, S), S)
    c = (tl.hops_per_tile - 1) * plan.freq_step // 2
    span = 2 * max(c, (tl.hops_per_tile - 1) * plan.freq_step - c) + plan.rate
    r = rs.plan_resample(R_dev, tl.capture_rate, span)
    assert r.up <= r.down
    h = rs.lowpass(r.up, r.down, r.taps_per_phase)
    win = power.window_table("hamming", 1 << plan.bin_e)
    return plan, win, tl, tiles, offs, dd, (r.up, r.down, h)


def _handles(plan, win, tl, offs, dd, res):
    a = power.PowerMix(plan, tl.capture_rate, offs, dd, win)
    a.set_burst_device_rate(*res)
    b = power.PowerMix(plan, tl.capture_rate, offs, dd, win)
    return a, b


def _capture_burst(res, x_dev):
    """The stateless resampler over the burst, its first E outputs dropped."""
    L, N, h = res
    E = rsm.ceil_div((h.size // L - 1) * L, N)
    with rs.Resampler(L, N, h) as r:
        y = r.process(x_dev)
    return y[2 * E:]


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("n_pass", [1, 3])
def test_bursts_equal_resampler_then_capture_rate_burst(name, n_pass):
    plan, win, tl, tiles, offs, dd, res = _case(name)
    a, b = _handles(plan, win, tl, offs, dd, res)
    assert a.burst_in_len(n_pass) != b.burst_in_len(n_pass) == b.burst_int16(n_pass)
    rng = np.random.default_rng(len(name) + 10 * n_pass)
    # every tile, then ragged hop ranges inside tiles
    ranges = [(hb, he) for hb, he, _ in tiles]
    for hb, he, _ in tiles[:2]:
        lo = int(rng.integers(hb, he))
        ranges.append((lo, int(rng.integers(lo + 1, he + 1))))
    for hb, he in ranges:
        x = rng.integers(-20000, 20001, size=a.burst_in_len(n_pass), dtype=np.int32).astype(np.int16)
        y = _capture_burst(res, x)
        assert y.size == b.burst_int16(n_pass)
        a.accumulate_burst(hb, he, x)
        b.accumulate_burst(hb, he, y)
    ga, gb = a.read(), b.read()
    assert np.array_equal(ga[0], gb[0]) and np.array_equal(ga[1], gb[1])
    assert gb[1].sum() > 0
    assert a.kernel_ms() > 0.0
    a.close(); b.close()


def test_wrong_length_refused_and_stream_unaffected():
    plan, win, tl, tiles, offs, dd, res = _case("fft_3.2M")
    a, b = _handles(plan, win, tl, offs, dd, res)
    rng = np.random.default_rng(3)
    pass_ = lambda: rng.integers(-20000, 20001, size=dd[0] * plan.buf_len, dtype=np.int32).astype(np.int16)  # noqa
    s0, s1 = pass_(), pass_()
    x = rng.integers(-20000, 20001, size=a.burst_in_len(1), dtype=np.int32).astype(np.int16)
    hb, he, _ = tiles[0]
    # stream, burst, stream: the stream calls take capture-rate samples and see one unbroken stream
    a.accumulate(s0); b.accumulate(s0)
    before = a.read()
    for bad in (x[:-2], np.concatenate([x, x[:2]]), x[:a.burst_in_len(1) // 2 & ~1]):
        with pytest.raises(_lib.Rxb200Error) as e:
            a.accumulate_burst(hb, he, bad)
        assert e.value.code == _lib.EUNSUPPORTED
    after = a.read()
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    a.accumulate_burst(hb, he, x); b.accumulate_burst(hb, he, _capture_burst(res, x))
    a.accumulate(s1); b.accumulate(s1)
    ga, gb = a.read(), b.read()
    assert np.array_equal(ga[0], gb[0]) and np.array_equal(ga[1], gb[1])
    # reset keeps the burst resampler: the same burst again gives the same accumulators
    a.reset(); b.reset()
    a.accumulate_burst(hb, he, x); b.accumulate_burst(hb, he, _capture_burst(res, x))
    ga, gb = a.read(), b.read()
    assert np.array_equal(ga[0], gb[0]) and np.array_equal(ga[1], gb[1])
    a.close(); b.close()


def test_device_rate_and_burst_device_rate_exclude_each_other():
    plan, win, tl, tiles, offs, dd, res = _case("fft_3.2M")
    a, b = _handles(plan, win, tl, offs, dd, res)
    for call in (a.set_device_rate, a.set_burst_device_rate):
        with pytest.raises(_lib.Rxb200Error) as e:
            call(*res)
        assert e.value.code == _lib.EINVAL
    b.set_device_rate(*res)
    with pytest.raises(_lib.Rxb200Error) as e:
        b.set_burst_device_rate(*res)
    assert e.value.code == _lib.EINVAL
    # the stream resampler still refuses bursts, whatever their length
    with pytest.raises(_lib.Rxb200Error) as e:
        b.accumulate_burst(0, 1, np.zeros(b.burst_int16(1), np.int16))
    assert e.value.code == _lib.EUNSUPPORTED
    with pytest.raises(_lib.Rxb200Error):
        a.burst_in_len(0)
    a.close(); b.close()
