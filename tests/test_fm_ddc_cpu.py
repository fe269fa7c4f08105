"""Decimating mixing handles on the CPU: the numpy DDC model (the identity against the mixer model, any split of a
capture against the whole, hand-computed rounding and saturation), the port against the unmodified reference on every
channel's decimated stream of every shape (read by read over reads that are not multiples of M, skipping reads with no
output), the golden hashes tests/golden/fm_ddc_golden.json records, and the refusals that need no device."""
import hashlib
import json
import os

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_ddc as fdd
import fm_mix as fmx
from rx_tools_b200 import _lib, fm

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "fm_ddc_golden.json")
ONE = np.ones(1, np.int32)


@pytest.mark.parametrize("rate,f,phase", [(2_400_000, 12500, 0), (1_008_000, -24000, 17), (19_200_000, 9_000_000, 5)])
def test_model_identity_is_the_mixer(rate, f, phase):
    x = fmx.capture(4001, rate, [f], 11)
    t = fm.mix_table(rate, f)
    y, hist = fdd.ddc_model(x, t, ONE, 1, 0, phase)
    assert np.array_equal(y, fmx.mix_model(x, t, phase)) and hist.size == 0


@pytest.mark.parametrize("decim,n_taps,shift", [(1, 1, 0), (3, 17, 13), (8, 33, 15), (64, 257, 15), (7, 5, 0)])
def test_model_over_any_split_equals_the_whole(decim, n_taps, shift):
    rng = np.random.default_rng(decim * 100 + n_taps)
    x = fmx.capture(9001, 1_008_000, [24000, -100000], 12)
    t = fm.mix_table(1_008_000, 24000)
    taps = fdd.lowpass(n_taps, 0.4 / decim, gain_bits=shift + 2)
    whole, _ = fdd.ddc_model(x, t, taps, decim, shift)
    for _ in range(4):
        cuts = np.sort(rng.choice(np.arange(1, 9001), size=6, replace=False))
        parts, pos, hist = [], 0, None
        for a, b in zip(np.r_[0, cuts], np.r_[cuts, 9001]):
            y, hist = fdd.ddc_model(x[2 * a:2 * b], t, taps, decim, shift, pos, hist)
            assert y.size == fdd.decimated_len(pos, 2 * (b - a), decim)
            parts.append(y)
            pos += b - a
        assert np.array_equal(np.concatenate(parts), whole)


def test_model_rounding_and_saturation_by_hand():
    t = fm.mix_table(1_000_000, 0)                           # the identity mixer: z = x
    x = np.array([1, -1, 3, -3, 5, 2, -5, 0, 20000, -20000, 11, -11], np.int16)
    # T = 1, h = {3}, S = 1: (3x + 1) >> 1, arithmetic (floor) shift
    y, _ = fdd.ddc_model(x, t, np.array([3], np.int32), 1, 1)
    assert y.tolist() == [2, -1, 5, -4, 8, 3, -7, 0, 30000, -30000, 17, -16]
    # h = {2}, S = 0: 2x saturates
    y, _ = fdd.ddc_model(x, t, np.array([2], np.int32), 1, 0)
    assert y.tolist() == [2, -2, 6, -6, 10, 4, -10, 0, 32767, -32768, 22, -22]
    # M = 2, h = {1, 1}, S = 1: outputs at samples 1, 3, 5 of (x[n] + x[n-1] + 1) >> 1
    y, _ = fdd.ddc_model(x, t, np.array([1, 1], np.int32), 2, 1)
    assert y.tolist() == [2, -2, 0, 1, 10006, -10005]   # ((3+1+1)>>1, (-3-1+1)>>1), ((-5+5+1)>>1, (0+2+1)>>1), ...
    # M = 3, h = {1, 0, 4}, S = 2 after one sample n = 0 of (7, -9): the history holds n = -1 (zero) and n = 0.  The
    # call's samples are n = 1, 2, 3 and its one emission n = 2: z[2] + 4 z[0] = (3 + 28, -3 - 36)
    y, h = fdd.ddc_model(x[:6], t, np.array([1, 0, 4], np.int32), 3, 2, pos=1, hist=np.array([0, 0, 7, -9], np.int16))
    assert y.tolist() == [(31 + 2) >> 2, (-39 + 2) >> 2] == [8, -10]
    assert h.tolist() == [3, -3, 5, 2]


def test_wide_flag_matches_the_shapes():
    assert not fdd.wide(*fdd.SHAPES["nbfm_m64_t257"][3][1:])
    assert fdd.wide(*fdd.SHAPES["raw_wide_m3"][3][1:])


def _channel_reads(name, seed=0):
    p, rate, offs, ddc, x, reads = fdd.case_input(name, seed)
    for f in offs:
        yield p, f, fdd.decimated_reads(x, fm.mix_table(rate, f), ddc, reads)


@pytest.mark.ref
@pytest.mark.parametrize("name", sorted(fdd.SHAPES))
def test_channels_port_equals_reference(name, port, ref_fm):
    for p, f, reads in _channel_reads(name, seed=1):
        y, lens = fdd.nonempty(reads)
        a = fac.port_run_seq(port, p, y, lens, return_chunks=True)
        b = fac.ref_run_seq(ref_fm, p, y, lens, return_chunks=True)
        assert a[0].tobytes() == b[0].tobytes(), (name, f)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]), (name, f)


@pytest.mark.ref
def test_channel_levels_port_equals_reference(port, ref_fm):
    for p, f, reads in _channel_reads("fm_lut_squelch_m4", seed=2):
        y, lens = fdd.nonempty(reads)
        assert np.array_equal(fac.port_levels_seq(port, p, y, lens), fac.ref_levels_seq(ref_fm, p, y, lens)), f


def test_port_matches_reference_golden(port):
    gold = json.load(open(GOLDEN))
    assert sorted(gold) == sorted(fdd.SHAPES)
    for name in fdd.SHAPES:
        p, rate, offs, ddc, x, reads = fdd.case_input(name)
        g = gold[name]
        assert g["params"] == {k: int(v) for k, v in vars(p).items()}, name
        assert g["capture_rate"] == rate and g["lens_int16"] == reads and g["n_int16"] == x.size, name
        assert g["ddc"] == {"decim": ddc[0], "taps": ddc[1].tolist(), "shift": ddc[2]}, name
        assert g["capture_sha256"] == hashlib.sha256(x.tobytes()).hexdigest(), name
        assert [c["offset_hz"] for c in g["channels"]] == offs, name
        for c in g["channels"]:
            dec = fdd.decimated_reads(x, fm.mix_table(rate, c["offset_hz"]), ddc, reads)
            assert [int(r.size) for r in dec] == c["dec_len"], (name, c["offset_hz"])
            y, lens = fdd.nonempty(dec)
            assert hashlib.sha256(y.tobytes()).hexdigest() == c["dec_sha256"], (name, c["offset_hz"])
            got, rl, _ = fac.port_run_seq(port, p, y, lens, return_chunks=True)
            assert rl.tolist() == c["result_len"], (name, c["offset_hz"])
            assert hashlib.sha256(got.tobytes()).hexdigest() == c["sha256"], (name, c["offset_hz"])


@pytest.mark.parametrize("ddc", [(0, [1], 0), (4097, [1], 0), (1, [], 0), (1, [1] * 8193, 0), (1, [1], -1),
                                 (1, [1], 63)])
def test_create_refuses_bad_ddc_before_looking_for_a_device(ddc):
    p = fmx.SHAPES["fm5a_lut_d100"][0]
    for cls in (fm.FmMix, fm.FmMixGroup):
        with pytest.raises(_lib.Rxb200Error) as e:
            cls(p, 2_400_000, [0, 12500], ddc=ddc)
        assert e.value.code == _lib.EINVAL, (cls, ddc)


def test_create_refuses_null_taps_and_keeps_the_mixer_refusals():
    import ctypes as C
    p = fm.FmParams.from_any(fmx.SHAPES["fm5a_lut_d100"][0]).to_c()
    offs = np.array([0, 12500], np.int32)
    d = _lib.DdcC(4, 3, None, 0)
    h = C.c_void_p()
    assert _lib.lib().rxb200_fm_mix_create_ddc(C.byref(p), 2_400_000, offs.ctypes.data_as(C.POINTER(C.c_int)), 2,
                                               C.byref(d), 0, C.byref(h)) == _lib.EINVAL
    assert _lib.lib().rxb200_fm_mix_create_ddc(C.byref(p), 2_400_000, offs.ctypes.data_as(C.POINTER(C.c_int)), 2,
                                               None, 0, C.byref(h)) == _lib.EINVAL
    for rate, offs, code in ((2_400_000, [0, 1_200_000], _lib.EINVAL), (2_400_001, [3], _lib.EUNSUPPORTED)):
        for cls in (fm.FmMix, fm.FmMixGroup):
            with pytest.raises(_lib.Rxb200Error) as e:
                cls(fmx.SHAPES["fm5a_lut_d100"][0], rate, offs, ddc=(4, [1, 2, 1], 2))
            assert e.value.code == code


def test_max_output_and_decimated_len_refuse_null():
    import ctypes as C
    n = C.c_size_t(0)
    assert _lib.lib().rxb200_fm_mix_decimated_len(None, 100, C.byref(n)) == _lib.EINVAL
    assert _lib.lib().rxb200_fm_mix_max_output(None, 100, 100) == 0


def test_create_without_device():
    if _lib.lib().rxb200_device_count() > 0:
        pytest.skip("a GPU is present")
    p, rate, offs, ddc, _, _ = fdd.SHAPES["nbfm_m64_t257"]
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.FmMix(p, rate, offs, ddc=ddc)
    assert e.value.code == _lib.ENODEV
