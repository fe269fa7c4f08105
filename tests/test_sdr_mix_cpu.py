"""rx_sdr I/Q down-converter handles without a GPU: the capture planner against its rule restated over seeded frequency
sets, offsets it takes that the rx_fm planner refuses for the mixer table's period, the refusals of both create calls
(all before any device is touched), and the model's anchors and formats against the port's rx_sdr conversions."""
import ctypes as C

import numpy as np
import pytest

import sdr_mix as sm
from rx_tools_b200 import _lib, fm, sdr


def _tuned_sets(n_sets, seed):
    rng = np.random.default_rng(seed)
    for _ in range(n_sets):
        k = int(rng.integers(1, 12))
        base = int(rng.integers(0, 3_000_000_000))
        span = int(rng.choice([10_000, 1_000_000, 20_000_000, 200_000_000]))
        yield [base + int(v) for v in rng.integers(0, span, size=k)], int(rng.choice([250_000, 1_000_000, 48_000]))


def test_planner_equals_rule_restated():
    n_ok = 0
    for tuned, s in _tuned_sets(200, 5):
        want = sm.plan_restated(tuned, s, 1 << 40)
        if want is None:
            with pytest.raises(_lib.Rxb200Error) as e:
                sdr.plan_sdr_capture(tuned, s, 1 << 40)
            assert e.value.code == _lib.EINVAL
            continue
        fc, M, R, T, offs = want
        for cap in (R, R - 1):
            if cap < R:
                with pytest.raises(_lib.Rxb200Error) as e:
                    sdr.plan_sdr_capture(tuned, s, cap)
                assert e.value.code == _lib.EINVAL and str(R) in str(e.value)
                continue
            plan, got = sdr.plan_sdr_capture(tuned, s, cap)
            assert (plan.centre_hz, plan.decim, plan.capture_rate, plan.n_taps) == (fc, M, R, T)
            assert got == offs and all(2 * abs(o) < R for o in got)
            n_ok += 1
    assert n_ok > 100


def test_planner_takes_offsets_the_table_mixer_refuses():
    """An offset whose table period exceeds 2^20 is refused by the rx_fm plan but not by the rx_sdr plan (the NCO)."""
    tuned = [100_000_000, 100_000_001, 100_731_119]
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.plan_capture(tuned, 1_000_003, 1 << 40)
    assert e.value.code == _lib.EUNSUPPORTED
    plan, offs = sdr.plan_sdr_capture(tuned, 1_000_003, 1 << 40)
    fplan, foffs = sm.plan_restated(tuned, 1_000_003, 1 << 40)[:2], sm.plan_restated(tuned, 1_000_003, 1 << 40)[4]
    assert (plan.centre_hz, plan.decim) == fplan and offs == foffs


def _create(rate, offs, ddc=None, two=None):
    L = _lib.lib()
    h = C.c_void_p()
    o = np.ascontiguousarray(offs, dtype=np.int32)
    if ddc is not None:
        d, _t = fm._ddc_c(ddc)
        rc = L.rxb200_sdr_mix_create(rate, o.ctypes.data_as(C.POINTER(C.c_int)), o.size, C.byref(d), 0, C.byref(h))
    else:
        K, c1, c2 = two
        d1, _t1 = fm._ddc_c(c1)
        d2, _t2 = fm._ddc_c(c2)
        rc = L.rxb200_sdr_mix_create_two_stage(rate, K, o.ctypes.data_as(C.POINTER(C.c_int)), o.size, C.byref(d1),
                                               C.byref(d2), 0, C.byref(h))
    assert not h.value
    return rc


def test_create_refusals_before_any_device():
    dd = (4, np.ones(9, np.int32), 3)
    assert _create(0, [0], ddc=dd) == _lib.EINVAL                       # R <= 0
    assert _create(1000, [500], ddc=dd) == _lib.EINVAL                  # |f| >= R/2
    assert _create(1000, [-500], ddc=dd) == _lib.EINVAL
    assert _create(1000, [], ddc=dd) == _lib.EINVAL                     # no channel
    assert _create(1000, [1], ddc=(0, np.ones(3, np.int32), 0)) == _lib.EINVAL          # M out of range
    assert _create(1000, [1], ddc=(2, np.ones(3, np.int32), 63)) == _lib.EINVAL         # S out of range
    assert _create(1000, [1], ddc=(2, np.ones(8192 + 1, np.int32), 0)) == _lib.EINVAL   # T > 8192
    c = (2, np.ones(5, np.int32), 15)
    f = (2, np.ones(5, np.int32), 15)
    assert _create(48_000, [0], two=(2, c, f)) == _lib.EINVAL           # K < 3
    assert _create(48_000, [0], two=(4097, c, f)) == _lib.EINVAL        # K > 4096
    assert _create(48_000, [24_000], two=(8, c, f)) == _lib.EINVAL      # |f| >= R/2
    assert _create(48_000, [0], two=(8, (2, np.full(4, 1 << 20, np.int32), 15), f)) == _lib.EINVAL   # sum |h1| >= 2^22
    assert _create(48_000, [0], two=(8, (128, np.ones(5, np.int32), 15), (64, np.ones(5, np.int32), 15))) == _lib.EINVAL
    assert _create(48_000, [0], two=(8, c, (0, np.ones(5, np.int32), 15))) == _lib.EINVAL


def test_null_handle_calls_refuse():
    L = _lib.lib()
    n = C.c_size_t(0)
    assert L.rxb200_sdr_mix_decimated_len(None, 8, C.byref(n)) == _lib.EINVAL
    assert L.rxb200_sdr_mix_process(None, None, 8, sdr.OUT_CS16, None, 0, 0, None) == _lib.EINVAL
    assert L.rxb200_sdr_mix_process_device(None, None, 8, sdr.OUT_CS16, None, 0, 0, None, 1) == _lib.EINVAL
    assert L.rxb200_sdr_mix_reset(None) == _lib.EINVAL
    L.rxb200_sdr_mix_destroy(None)


def test_identity_shape_is_the_capture():
    x = sm.case_capture("identity")
    y, M = sm.model("identity", x)
    assert M == 1 and np.array_equal(y[0], x)


def test_wide_shape_needs_a_64_bit_accumulator():
    h = sm.SHAPES["wide_acc"][3][1]
    assert int(np.abs(h.astype(np.int64)).sum()) * 32768 + (1 << 20) >= 1 << 31


def test_model_formats_equal_the_port(port):
    """The model's conversions over every int16 value equal the port's rx_sdr conversions (pinned to the reference)."""
    x = np.arange(-32768, 32768, dtype=np.int32).astype(np.int16)
    for fmt, name, dt in (("CS8", "orx_sdr_cs16_to_cs8", np.uint8), ("CU8", "orx_sdr_cs16_to_cu8", np.uint8),
                          ("CF32", "orx_sdr_cs16_to_cf32", np.float32)):
        f = getattr(port.L, name)
        f.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
        f.restype = None
        want = np.empty(x.size, dt)
        f(x.ctypes.data, x.size, want.ctypes.data)
        assert np.array_equal(sm.convert(x, fmt).view(np.uint8), want.view(np.uint8)), fmt
