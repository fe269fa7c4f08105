"""The rational resampler without a GPU: the numpy model against the rule term by term (L = 1, N = 1, L > N, L < N,
non-coprime L/N, J = 1; single calls and ragged splits), both anchors (the identity, and L = 1 against the DDC model with
M - 1 leading zeros), the library's prototype filter (every phase sums to 2^15, a constant comes back exactly, the named
plans' passband and stopband, its refusals), the planner against its restatement (seeded spans and rates, the worked
examples, the guard-band edge, every refusal), and the create and device-entry refusals, which come before any device
work."""
import ctypes as C
import random

import numpy as np
import pytest

import fm_ddc as fd
import resample as rm
from rx_tools_b200 import _lib, resample


def _rand_taps(rng, L, J, lim=3000):
    return rng.integers(-lim, lim + 1, size=L * J).astype(np.int32)


def _stream(rng, c):
    return rng.integers(-32768, 32768, size=2 * c).astype(np.int16)


@pytest.mark.parametrize("L,N,J,S", [(1, 1, 1, 0), (1, 1, 5, 12), (1, 4, 7, 13), (5, 1, 3, 14), (5, 8, 6, 15),
                                     (8, 5, 4, 15), (6, 4, 5, 16), (21, 25, 1, 3), (3, 7, 9, 20)])
def test_model_equals_rule(L, N, J, S):
    rng = np.random.default_rng(L * 1000 + N * 10 + J)
    h = _rand_taps(rng, L, J)
    x = _stream(rng, 97)
    for n0 in (0, 1, 13, (1 << 40) + 3):
        y, _ = rm.resample_model(x, L, N, h, S, n0)
        assert np.array_equal(y, rm.resample_rule(x, L, N, h, S, n0)), n0
        assert y.size == 2 * rm.out_count(n0, 97, L, N)


@pytest.mark.parametrize("L,N,J", [(1, 3, 4), (7, 2, 5), (21, 25, 6), (6, 9, 3), (1, 1, 1)])
def test_model_ragged_splits_equal_one_call(L, N, J):
    rng = np.random.default_rng(5 + L + N + J)
    h = _rand_taps(rng, L, J)
    x = _stream(rng, 400)
    one, _ = rm.resample_model(x, L, N, h, 15)
    assert np.array_equal(one, rm.resample_rule(x, L, N, h, 15))
    for lens in ([2], [6, 2, 14], [2 * 37, 2 * 3, 2 * 101], [2 * 1000]):
        assert np.array_equal(rm.calls_model(x, L, N, h, 15, lens), one), lens


def test_identity_anchor():
    x = _stream(np.random.default_rng(1), 1000)
    y, _ = rm.resample_model(x, 1, 1, np.array([1 << 15], np.int32), 15)
    assert np.array_equal(y, x)


@pytest.mark.parametrize("M,T,S", [(2, 9, 15), (7, 33, 13), (5, 1, 0), (3, 4, 15)])
def test_decimation_anchor_against_ddc_model(M, T, S):
    """L = 1, N = M, J = T: output m is output m of the DDC at offset 0 over the stream with M - 1 zeros prepended."""
    rng = np.random.default_rng(M * T)
    h = _rand_taps(rng, 1, T)
    x = _stream(rng, 333)
    y, _ = rm.resample_model(x, 1, M, h, S)
    ident = np.array([[32768, 0]], np.int64)                # offset 0: the mixer is the identity
    z = np.concatenate([np.zeros(2 * (M - 1), np.int16), x])
    d, _ = fd.ddc_model(z, ident, h, M, S)
    n = min(y.size, d.size)
    assert n >= 2 * (333 // M)
    assert np.array_equal(y[:n], d[:n])


@pytest.mark.parametrize("L,N,J", [(1, 1, 1), (1, 7, 8), (7, 1, 8), (5, 8, 48), (21, 25, 24), (504, 625, 24),
                                   (187, 256, 136), (3, 3, 16)])
def test_lowpass_phases_sum_to_unity_and_constants_pass(L, N, J):
    h = resample.lowpass(L, N, J)
    assert h.size == L * J
    for p in range(L):
        assert int(h[p::L].astype(np.int64).sum()) == 1 << 15, p
    for v in (-32768, -1, 12345, 32767):
        x = np.full(2 * (J + 3 * N + 5), v, np.int16)
        y, _ = rm.resample_model(x, L, N, h, 15)
        q = (np.arange(y.size // 2) * N) // L
        steady = y.reshape(-1, 2)[q >= J - 1]
        assert steady.size and np.all(steady == v), v


@pytest.mark.parametrize("name,R_dev,R,span,LN,J", rm.NAMED, ids=[n[0] for n in rm.NAMED])
def test_named_plans(name, R_dev, R, span, LN, J):
    p = resample.plan_resample(R_dev, R, span)
    assert (p.up, p.down) == LN and p.taps_per_phase == J and p.shift == 15
    assert tuple(p) == rm.plan_rule(R_dev, R, span)
    h = resample.lowpass(p.up, p.down, J)
    ripple, stop = rm.response_db(h, p.up, R_dev, span, R)
    assert ripple <= 0.01, ripple
    assert stop <= -70.0, stop


def test_named_refusal_names_the_span():
    with pytest.raises(_lib.Rxb200Error) as e:
        resample.plan_resample(*rm.REFUSED)
    assert e.value.code == _lib.EINVAL
    assert "21020000" in str(e.value) and "20000000" in str(e.value) and str(20_000_000 - 625_000) in str(e.value)


DEVICE_RATES = [2_048_000, 2_400_000, 2_500_000, 3_200_000, 6_000_000, 10_000_000, 20_000_000, 30_720_000, 56_000_000,
                61_440_000]
CHAIN_RATES = [25_000, 48_000, 170_000, 240_000, 250_000, 300_000, 1_008_000, 1_020_000, 2_400_000]


def _capture_case(rnd):
    """A device rate and what a capture plan would ask of it: a chain rate c, channels out to A from the centre, and
    R = M c with M large enough that the resampler's guard band fits (min(R, R_dev) - (2A + c) >= G)."""
    R_dev = rnd.choice(DEVICE_RATES)
    c = rnd.choice([v for v in CHAIN_RATES if v < R_dev // 2])
    G = -(-R_dev // 32)
    A = rnd.randrange(0, (R_dev - G - c) // 2 + 1)
    span = 2 * A + c
    M = -(-(span + G) // c)
    return R_dev, M * c, span


def test_plan_matches_restatement_over_seeded_capture_cases():
    """Cases shaped like capture plans: nearly all are accepted, and every one matches the restatement."""
    rnd = random.Random(2026)
    accepted = 0
    for _ in range(400):
        R_dev, R, span = _capture_case(rnd)
        want = rm.plan_rule(R_dev, R, span)
        assert want is not None
        if want[2] * want[0] > (1 << 22):
            with pytest.raises(_lib.Rxb200Error) as e:
                resample.plan_resample(R_dev, R, span)
            assert e.value.code == _lib.EUNSUPPORTED and f"{want[0]}/{want[1]}" in str(e.value)
            continue
        got = resample.plan_resample(R_dev, R, span)
        assert tuple(got) == want
        assert 8 <= got.taps_per_phase <= 192
        accepted += 1
    assert accepted >= 300, accepted


def test_plan_matches_restatement_over_seeded_ratios():
    """Arbitrary rates and spans: mostly refusals (coprime ratios, spans without a guard band), each as restated."""
    rnd = random.Random(2026)
    for _ in range(400):
        R_dev = rnd.choice(DEVICE_RATES)
        R = rnd.randrange(R_dev // 3, 2 * R_dev)
        span = rnd.randrange(0, min(R, R_dev))
        want = rm.plan_rule(R_dev, R, span)
        if want is not None and want[2] * want[0] > (1 << 22):
            with pytest.raises(_lib.Rxb200Error) as e:
                resample.plan_resample(R_dev, R, span)
            assert e.value.code == _lib.EUNSUPPORTED and f"{want[0]}/{want[1]}" in str(e.value)
        elif want is None:
            with pytest.raises(_lib.Rxb200Error) as e:
                resample.plan_resample(R_dev, R, span)
            assert e.value.code == _lib.EINVAL
        else:
            got = resample.plan_resample(R_dev, R, span)
            assert tuple(got) == want
            assert 8 <= got.taps_per_phase <= 192


@pytest.mark.parametrize("R_dev", [2_400_000, 2_500_000, 30_720_000, 61_440_000, 2_048_001])
def test_plan_guard_band_edge(R_dev):
    G = -(-R_dev // 32)
    p = resample.plan_resample(R_dev, R_dev, R_dev - G)
    assert (p.up, p.down, p.taps_per_phase) == (1, 1, 192)
    with pytest.raises(_lib.Rxb200Error) as e:
        resample.plan_resample(R_dev, R_dev, R_dev - G + 1)
    assert e.value.code == _lib.EINVAL


def test_plan_refusals():
    L = _lib.lib()
    out = _lib.ResamplerC()
    assert L.rxb200_plan_resample(2_400_000, 2_016_000, 1_000_000, None) == _lib.EINVAL
    for args in ((0, 1, 0), (1, 0, 0), (1 << 31, 1000, 0), (1000, 1 << 31, 0), (1000, 1000, -1)):
        assert L.rxb200_plan_resample(*args, C.byref(out)) == _lib.EINVAL, args
    # a ratio whose prototype would pass 2^22 taps: L = 2^21 + 1 over a coprime N
    assert L.rxb200_plan_resample(2_000_000, 2_097_153, 0, C.byref(out)) == _lib.EUNSUPPORTED


def test_lowpass_refusals():
    L = _lib.lib()
    t = np.zeros(16, np.int32)
    tp = t.ctypes.data_as(C.POINTER(C.c_int32))
    assert L.rxb200_resample_lowpass(1, 1, 1, None) == _lib.EINVAL
    for args in ((0, 1, 1), (1, 0, 1), (1, 1, 0), (1, 1, 1025), (4097, 1, 1024)):
        assert L.rxb200_resample_lowpass(*args, tp) == _lib.EINVAL, args


def _rs(up, down, J, taps, shift):
    return _lib.ResamplerC(up, down, J, taps.ctypes.data_as(C.POINTER(C.c_int32)) if taps is not None else None, shift)


def test_create_and_device_refusals_before_any_device_work():
    """Every refusal comes before any device is touched, so it holds on a machine without a GPU too."""
    L = _lib.lib()
    h = np.ones(4096, np.int32)
    big = np.full(1024, (1 << 31) - 1, np.int32)
    bad = [None, _rs(1, 1, 1, None, 15), _rs(0, 1, 1, h, 15), _rs(1, 0, 1, h, 15), _rs(1, 1, 0, h, 15),
           _rs(1, 1, 1025, h, 15), _rs(4097, 1, 1024, h, 15), _rs(1, 1, 1, h, -1), _rs(1, 1, 1, h, 63)]
    out = C.c_void_p()
    for rs in bad:
        arg = None if rs is None else C.byref(rs)
        assert L.rxb200_resample_create(arg, 0, C.byref(out)) == _lib.EINVAL
        assert L.rxb200_resample_device(arg, 0, 16, 4, 16, None) == _lib.EINVAL
    assert L.rxb200_resample_create(C.byref(_rs(1, 1, 1, h, 15)), 0, None) == _lib.EINVAL
    ok = _rs(1, 1, 1024, big, 62)                       # 1024 (2^31 - 1) 2^15 + 2^61 < 2^63: accepted by the check
    for src, dst in ((None, 16), (16, None), (18, 16), (16, 18)):
        assert L.rxb200_resample_device(C.byref(ok), 0, src, 4, dst, None) == _lib.EINVAL, (src, dst)
    for fn in (L.rxb200_resample_reset,):
        assert fn(None) == _lib.EINVAL
    assert L.rxb200_resample_out_len(None, 4, C.byref(C.c_size_t())) == _lib.EINVAL
    assert L.rxb200_resample_process(None, 16, 4, 16, 8, None) == _lib.EINVAL
    assert L.rxb200_resample_process_device(None, 16, 4, 16, 8, None, 1) == _lib.EINVAL
    assert L.rxb200_resample_kernel_ms(None, C.byref(C.c_float())) == _lib.EINVAL
    assert L.rxb200_resample_stream(None) is None


def test_wide_rule_matches_the_fm_ddc_rule_at_one_phase():
    h = fd.lowpass(33, 0.1, gain_bits=17)
    assert rm.wide(h, 1, 13) == fd.wide(h, 13)
