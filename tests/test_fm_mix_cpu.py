"""Several rx_fm channels of one capture, on the CPU: the properties of the library's mixer table, the numpy mixer model,
the port against the unmodified reference on every channel of every shape (read by read over a ragged sequence, so the
mixer's phase runs on across reads), their -L levels, the golden hashes tests/golden/fm_mix_golden.json records of the
reference, and the handle's refusals that need no device."""
import hashlib
import json
import os

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_mix as fmx
from rx_tools_b200 import _lib, fm

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "fm_mix_golden.json")


@pytest.mark.parametrize("rate,f", [(2_400_000, 12500), (2_400_000, -12500), (2_400_000, 37500), (1_008_000, 24000),
                                    (1_000_000, 33000), (48_000, 1), (2_400_000, 1_199_000), (7, 3), (1, 0)])
def test_table_period_and_first_entry(rate, f):
    t = fm.mix_table(rate, f)
    assert t.shape == (rate // np.gcd(rate, abs(f)), 2)
    assert t[0].tolist() == [32768, 0]
    assert np.all(np.abs(t) <= 32768)
    # every entry is the rounded Q15 point of its angle (within rounding of a correct fp64 cos / sin)
    m = np.arange(t.shape[0], dtype=np.int64)
    ang = -2.0 * np.pi * ((m * f) % rate) / rate
    assert np.abs(t[:, 0] - 32768.0 * np.cos(ang)).max() <= 0.5 + 1e-6
    assert np.abs(t[:, 1] - 32768.0 * np.sin(ang)).max() <= 0.5 + 1e-6


def test_table_zero_offset_is_the_identity():
    for rate in (1, 1_008_000, 2_400_000):
        assert fm.mix_table(rate, 0).tolist() == [[32768, 0]]
    x = np.arange(-32768, 32768, dtype=np.int16)
    assert np.array_equal(fmx.mix_model(x, fm.mix_table(2_400_000, 0)), x)


@pytest.mark.parametrize("rate", [4, 1_008_000, 2_400_000])
def test_table_quarter_rate_is_an_exact_rotation(rate):
    assert fm.mix_table(rate, rate // 4).tolist() == [[32768, 0], [0, -32768], [-32768, 0], [0, 32768]]
    assert fm.mix_table(rate, -(rate // 4)).tolist() == [[32768, 0], [0, 32768], [-32768, 0], [0, -32768]]
    # (I, Q) -> (Q, -I) -> (-I, -Q) -> (-Q, I) for every value but -32768, whose negation wraps
    x = np.arange(-32767, 32767, dtype=np.int16)
    y = fmx.mix_model(x, fm.mix_table(rate, rate // 4)).reshape(-1, 2)
    xi = x.reshape(-1, 2).astype(np.int32)
    k = (np.arange(xi.shape[0]) % 4)[:, None]
    want = np.select([k == 0, k == 1, k == 2, k == 3],
                     [xi, np.stack([xi[:, 1], -xi[:, 0]], 1), -xi, np.stack([-xi[:, 1], xi[:, 0]], 1)])
    assert np.array_equal(y.astype(np.int32), want)


@pytest.mark.parametrize("rate,f", [(2_400_000, 12500), (1_008_000, 24000), (1_000_000, 33000), (48_000, 7),
                                    (2_400_000, 1_199_000)])
def test_table_of_minus_f_is_the_conjugate(rate, f):
    a, b = fm.mix_table(rate, f), fm.mix_table(rate, -f)
    assert np.array_equal(a[:, 0], b[:, 0]) and np.array_equal(a[:, 1], -b[:, 1])


@pytest.mark.parametrize("rate,f,code", [(2_400_000, 1_200_000, _lib.EINVAL), (2_400_000, -1_200_000, _lib.EINVAL),
                                         (2_400_000, 2_000_000, _lib.EINVAL), (0, 0, _lib.EINVAL),
                                         (-48_000, 100, _lib.EINVAL), (2_400_001, 1, _lib.EUNSUPPORTED),
                                         ((1 << 20) + 1, 1, _lib.EUNSUPPORTED)])
def test_table_refusals(rate, f, code):
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.mix_table(rate, f)
    assert e.value.code == code


def test_table_capacity():
    import ctypes as C
    period = C.c_size_t(0)
    t = np.zeros(2 * 192 - 1, dtype=np.int32)
    rc = _lib.lib().rxb200_fm_mix_table(2_400_000, 12500, t.ctypes.data_as(C.POINTER(C.c_int32)), t.size,
                                        C.byref(period))
    assert rc == _lib.ECAPACITY and period.value == 192
    assert fm.mix_table(1 << 20, 1).shape == (1 << 20, 2)      # the longest period taken


def test_model_phase_carries():
    """Mixing a stream in pieces with the phase carried equals mixing it at once."""
    x = fmx.capture(5000, 1_008_000, [10000], 3)
    t = fm.mix_table(1_008_000, 24000)
    whole = fmx.mix_model(x, t)
    parts, ph = [], 0
    for a, b in ((0, 2 * 1021), (2 * 1021, 2 * 1354), (2 * 1354, x.size)):
        parts.append(fmx.mix_model(x[a:b], t, ph))
        ph += (b - a) // 2
    assert np.array_equal(np.concatenate(parts), whole)


def _assert_same(a, b, what):
    assert a[0].size == b[0].size, what
    bad = np.flatnonzero(a[0] != b[0])
    assert bad.size == 0, (what, bad[:5])
    assert np.array_equal(a[1], b[1]), what
    assert np.array_equal(a[2], b[2]), what


@pytest.mark.ref
@pytest.mark.parametrize("name", sorted(fmx.SHAPES))
def test_channels_port_equals_reference(name, port, ref_fm):
    p, rate, offs, x = fmx.case_input(name, seed=1)
    for f in offs:
        y = fmx.mix_model(x, fm.mix_table(rate, f))
        a = fac.port_run_seq(port, p, y, fmx.READS, return_chunks=True)
        b = fac.ref_run_seq(ref_fm, p, y, fmx.READS, return_chunks=True)
        _assert_same(a, b, (name, f))


@pytest.mark.ref
def test_channel_levels_port_equals_reference(port, ref_fm):
    p, rate, offs, x = fmx.case_input("fm_lut_d42_squelch", seed=2)
    for f in offs:
        y = fmx.mix_model(x, fm.mix_table(rate, f))
        assert np.array_equal(fac.port_levels_seq(port, p, y, fmx.READS), fac.ref_levels_seq(ref_fm, p, y, fmx.READS))


def test_port_matches_reference_golden(port):
    gold = json.load(open(GOLDEN))
    assert sorted(gold) == sorted(fmx.SHAPES)
    for name in fmx.SHAPES:
        p, rate, offs, x = fmx.case_input(name)
        g = gold[name]
        assert g["params"] == {k: int(v) for k, v in vars(p).items()}, name
        assert g["capture_rate"] == rate and g["lens_int16"] == fmx.READS and g["n_int16"] == x.size, name
        assert g["capture_sha256"] == hashlib.sha256(x.tobytes()).hexdigest(), name
        assert [c["offset_hz"] for c in g["channels"]] == offs, name
        for c in g["channels"]:
            y = fmx.mix_model(x, fm.mix_table(rate, c["offset_hz"]))
            got, rl, _ = fac.port_run_seq(port, p, y, fmx.READS, return_chunks=True)
            assert rl.tolist() == c["result_len"], (name, c["offset_hz"])
            assert hashlib.sha256(got.tobytes()).hexdigest() == c["sha256"], (name, c["offset_hz"])


def test_create_refuses_offsets_before_looking_for_a_device():
    p = fmx.SHAPES["fm5a_lut_d100"][0]
    for offs, code in (([0, 1_200_000], _lib.EINVAL), ([3], _lib.EUNSUPPORTED)):
        with pytest.raises(_lib.Rxb200Error) as e:
            fm.FmMix(p, 2_400_001 if code == _lib.EUNSUPPORTED else 2_400_000, offs)
        assert e.value.code == code
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.FmMix(p, 2_400_000, [])
    assert e.value.code == _lib.EINVAL


def test_create_without_device():
    if _lib.lib().rxb200_device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.FmMix(fmx.SHAPES["fm5a_lut_d100"][0], 2_400_000, [0, 12500])
    assert e.value.code == _lib.ENODEV
