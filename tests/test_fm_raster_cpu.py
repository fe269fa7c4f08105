"""Raster mixing handles on the CPU: the numpy model against a direct Python-integer evaluation of the rule, the
polyphase regrouping the kernels use against the direct sum, the two exact anchors against the decimating handle's
model (bin 0 at every shift, bin K/4 where the quarter-turn mixer does not wrap), the port against the unmodified
reference on every channel's decimated stream of every shape, the golden hashes tests/golden/fm_raster_golden.json
records, and the refusals, which come before any device work."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_ddc as fdd
import fm_mix as fmx
import fm_raster as frs
from rx_tools_b200 import _lib, fm

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "fm_raster_golden.json")


def direct(x, n_bins, bins, taps, decim, shift, phase=0, raw=False):
    """The rule term by term in Python integers over a whole capture (sample i has index phase + i; none before).
    raw: the sums A as (I, Q) pairs, before the shift and the saturation."""
    tw = frs.table(n_bins).tolist()
    xs = np.asarray(x, dtype=np.int64).reshape(-1, 2).tolist()
    out = []
    for k in bins:
        row = []
        for m in range(len(xs) // decim):
            e = m * decim + decim - 1
            ai = aq = 0
            for j, h in enumerate(int(v) for v in taps):
                if e - j < 0:
                    continue
                xi, xq = xs[e - j]
                c, s = tw[(k * (phase + e - j)) % n_bins]
                ai += h * (xi * c - xq * s)
                aq += h * (xi * s + xq * c)
            if raw:
                row.append((ai, aq))
                continue
            for a in (ai, aq):
                y = a if shift == 0 else (a + (1 << (shift - 1))) >> shift
                row.append(max(-32768, min(32767, y)))
        out.append(row)
    return out


def _random(n, seed, amp=32768):
    return np.random.default_rng(seed).integers(-amp, amp, size=2 * n).astype(np.int16)


@pytest.mark.parametrize("K,bins,decim,n_taps,shift", [(3, [0, 1, 2], 1, 1, 0), (4, [1, 3, 2, 1], 3, 7, 17),
                                                       (7, [5, 0], 2, 16, 31), (12, [3, 11, 6], 5, 30, 40),
                                                       (16, [4], 4, 3, 62)])
def test_model_equals_the_rule_over_any_split(K, bins, decim, n_taps, shift):
    rng = np.random.default_rng(K * 100 + n_taps)
    taps = rng.integers(-30000, 30000, size=n_taps).astype(np.int32)
    x = _random(301, K + n_taps)
    want = np.array(direct(x, K, bins, taps, decim, shift), dtype=np.int16)
    whole, _ = frs.raster_model(x, K, bins, taps, decim, shift)
    assert whole.tolist() == want.tolist()
    for _ in range(3):
        cuts = np.sort(rng.choice(np.arange(1, 301), size=5, replace=False))
        parts, pos, hist = [], 0, None
        for a, b in zip(np.r_[0, cuts], np.r_[cuts, 301]):
            y, hist = frs.raster_model(x[2 * a:2 * b], K, bins, taps, decim, shift, pos, hist)
            assert y.shape == (len(bins), fdd.decimated_len(pos, 2 * (b - a), decim))
            parts.append(y)
            pos += b - a
        assert np.concatenate(parts, axis=1).tolist() == want.tolist()


def test_model_phase_is_the_first_sample_residue():
    x, taps = _random(97, 3), np.array([3, -1, 4, 1, -5], np.int32)
    for phase in (0, 5, (1 << 64) - 11, (1 << 40) + 3):
        y, _ = frs.raster_model(x, 11, [0, 2, 9], taps, 2, 9, phase=phase)
        assert y.tolist() == direct(x, 11, [0, 2, 9], taps, 2, 9, phase=phase % 11)


@pytest.mark.parametrize("K,decim,n_taps", [(3, 1, 1), (8, 3, 5), (8, 4, 40), (12, 7, 12), (5, 2, 23)])
def test_polyphase_regrouping_equals_the_direct_sum(K, decim, n_taps):
    rng = np.random.default_rng(K + decim + n_taps)
    taps = rng.integers(-(1 << 16), 1 << 16, size=n_taps).astype(np.int64)         # sum |h| < 2^22
    bins = list(range(K)) + [1]
    x = _random(200, n_taps)
    n_out = 200 // decim
    ext = np.concatenate([np.zeros(2 * (n_taps - 1), np.int16), x])
    for res0 in (0, 2):
        v = frs.branch_sums(ext, taps, decim, K, res0 - (n_taps - 1), n_out)
        assert np.abs(v).max() < (1 << 37)
        got = frs.dft(v, K, bins)
        want = direct(x, K, bins, taps, decim, 0, phase=res0, raw=True)
        assert [[tuple(a) for a in ch] for ch in got.tolist()] == want
        full = frs.raster_model(x, K, bins, taps, decim, 0, phase=res0)[0]
        assert np.clip(got, -32768, 32767).reshape(len(bins), -1).tolist() == full.tolist()


def test_anchor_bin_zero_is_the_ddc_at_dc_for_every_shift():
    rate, K = 2_400_000, 48
    taps = fdd.lowpass(33, 0.05, gain_bits=21)
    assert frs.sum_abs(taps) < (1 << 22)
    x = _random(2001, 7)
    t0 = fm.mix_table(rate, 0)
    for shift in range(48):
        got, _ = frs.raster_model(x, K, [0], taps, 4, shift + 15)
        want, _ = fdd.ddc_model(x, t0, taps, 4, shift)
        assert got[0].tobytes() == want.tobytes(), shift


@pytest.mark.parametrize("K", [4, 8, 768])
def test_anchor_bin_quarter_is_the_ddc_at_a_quarter_turn(K):
    rate = 2_400_000
    taps = fdd.lowpass(17, 0.1, gain_bits=18)
    tq = fm.mix_table(rate, rate // 4)
    assert tq.shape[0] == 4
    x = _random(3001, K)
    x[x == -32768] = -32767
    for shift in (0, 12, 20):
        for pos in (0, 1, 2, 3):
            got, _ = frs.raster_model(x, K, [K // 4], taps, 3, shift + 15, pos=pos)
            want, _ = fdd.ddc_model(x, tq, taps, 3, shift, pos=pos)
            assert got[0].tobytes() == want.tobytes(), (shift, pos)
    # a -32768 in I (sample 9: the entry that negates I) or in Q (sample 10) wraps the mixer, not the raster
    for comp in (0, 1):
        y = np.zeros(2 * 16, np.int16)
        y[2 * (9 + comp) + comp] = -32768
        got, _ = frs.raster_model(y, K, [K // 4], np.ones(1, np.int32), 1, 15)
        want, _ = fdd.ddc_model(y, tq, np.ones(1, np.int32), 1, 0)
        assert got[0].tobytes() != want.tobytes(), comp


def test_shapes_cover_the_named_cases():
    Ks = {s[2] for s in frs.SHAPES.values()}
    assert {3, 4096, 768} <= Ks and any(k & (k - 1) for k in Ks)
    b = frs.SHAPES["raw_k4096_m64"][3]
    assert {0, 1, 2048, 4095} <= set(b) and len(set(b)) < len(b)
    dd = frs.SHAPES["raw_sat_k3_m3"][4]
    assert frs.sum_abs(dd[1]) == (1 << 22) - 1
    _, K, bins, ddc, x, reads = frs.case_input("raw_sat_k3_m3")
    y = frs.decimated_reads(x, K, bins, ddc, reads)
    assert any((np.abs(np.concatenate(r).astype(np.int32)) >= 32767).any() for r in y)   # outputs saturate


def _channel_reads(name, seed=0):
    p, K, bins, ddc, x, reads = frs.case_input(name, seed)
    return p, frs.decimated_reads(x, K, bins, ddc, reads)


@pytest.mark.ref
@pytest.mark.parametrize("name", sorted(frs.SHAPES))
def test_channels_port_equals_reference(name, port, ref_fm):
    p, chans = _channel_reads(name, seed=1)
    for c, reads in enumerate(chans):
        y, lens = fdd.nonempty(reads)
        a = fac.port_run_seq(port, p, y, lens, return_chunks=True)
        b = fac.ref_run_seq(ref_fm, p, y, lens, return_chunks=True)
        assert a[0].tobytes() == b[0].tobytes(), (name, c)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2]), (name, c)


@pytest.mark.ref
def test_channel_levels_port_equals_reference(port, ref_fm):
    p, chans = _channel_reads("fm_lut_squelch_k504_m4", seed=2)
    for c, reads in enumerate(chans):
        y, lens = fdd.nonempty(reads)
        assert np.array_equal(fac.port_levels_seq(port, p, y, lens), fac.ref_levels_seq(ref_fm, p, y, lens)), c


def test_port_matches_reference_golden(port):
    gold = json.load(open(GOLDEN))
    assert sorted(gold) == sorted(frs.SHAPES)
    for name in frs.SHAPES:
        p, K, bins, ddc, x, reads = frs.case_input(name)
        g = gold[name]
        assert g["params"] == {k: int(v) for k, v in vars(p).items()}, name
        assert g["n_bins"] == K and g["bins"] == bins and g["lens_int16"] == reads and g["n_int16"] == x.size, name
        assert g["ddc"] == {"decim": ddc[0], "taps": [int(v) for v in ddc[1]], "shift": ddc[2]}, name
        assert g["capture_sha256"] == hashlib.sha256(x.tobytes()).hexdigest(), name
        for c, dec in enumerate(frs.decimated_reads(x, K, bins, ddc, reads)):
            gc = g["channels"][c]
            assert [int(r.size) for r in dec] == gc["dec_len"], (name, c)
            y, lens = fdd.nonempty(dec)
            assert hashlib.sha256(y.tobytes()).hexdigest() == gc["dec_sha256"], (name, c)
            got, rl, _ = fac.port_run_seq(port, p, y, lens, return_chunks=True)
            assert rl.tolist() == gc["result_len"], (name, c)
            assert hashlib.sha256(got.tobytes()).hexdigest() == gc["sha256"], (name, c)


P0 = fmx.SHAPES["fm5a_lut_d100"][0]
GOOD = (4, np.array([1, 2, 1], np.int32), 2)


@pytest.mark.parametrize("raster,ddc", [((2, [0]), GOOD), ((4097, [0]), GOOD), ((8, [8]), GOOD), ((8, [-1]), GOOD),
                                        ((8, []), GOOD), ((8, [0]), (4, np.full(4, 1 << 20, np.int32), 2)),
                                        ((8, [0]), (0, [1], 0)), ((8, [0]), (4, [1] * 8193, 0)),
                                        ((8, [0]), (4, [1], 63))])
def test_create_and_device_entry_refuse_before_looking_for_a_device(raster, ddc):
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.FmMix(P0, ddc=ddc, raster=raster)
    assert e.value.code == _lib.EINVAL
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.raster_device(raster[0], raster[1], 0, ddc, 16, 1000, 16)     # never dereferenced
    assert e.value.code == _lib.EINVAL


def test_create_refuses_null_bins_and_ddc_and_keeps_the_params_refusals():
    p = fm.FmParams.from_any(P0).to_c()
    taps = np.array([1, 2, 1], np.int32)
    d = _lib.DdcC(4, 3, taps.ctypes.data_as(C.POINTER(C.c_int32)), 2)
    bins = np.array([0, 3], np.int32)
    h = C.c_void_p()
    L = _lib.lib()
    pb = bins.ctypes.data_as(C.POINTER(C.c_int))
    assert L.rxb200_fm_mix_create_raster(C.byref(p), 8, None, 2, C.byref(d), 0, C.byref(h)) == _lib.EINVAL
    assert L.rxb200_fm_mix_create_raster(C.byref(p), 8, pb, 0, C.byref(d), 0, C.byref(h)) == _lib.EINVAL
    assert L.rxb200_fm_mix_create_raster(C.byref(p), 8, pb, 2, None, 0, C.byref(h)) == _lib.EINVAL
    assert L.rxb200_fm_mix_create_raster(None, 8, pb, 2, C.byref(d), 0, C.byref(h)) == _lib.EINVAL
    assert L.rxb200_fm_mix_create_raster(C.byref(p), 8, pb, 2, C.byref(d), 0, None) == _lib.EINVAL
    assert L.rxb200_raster_device(8, pb, 2, 0, C.byref(d), None, 100, 16, None) == _lib.EINVAL
    assert L.rxb200_raster_device(8, pb, 2, 0, C.byref(d), 18, 100, 16, None) == _lib.EINVAL   # 2-byte aligned
    assert L.rxb200_raster_device(8, pb, 2, 0, C.byref(d), 16, 100, 18, None) == _lib.EINVAL
    # a chain parameter the member refuses: the same code as a decimating handle's
    bad = fm.FmParams.from_any(fac.with_(P0, downsample=0)).to_c()
    offs = np.array([0], np.int32)
    want = L.rxb200_fm_mix_create_ddc(C.byref(bad), 2_400_000, offs.ctypes.data_as(C.POINTER(C.c_int)), 1,
                                      C.byref(d), 0, C.byref(h))
    assert want != _lib.OK
    assert L.rxb200_fm_mix_create_raster(C.byref(bad), 8, pb, 2, C.byref(d), 0, C.byref(h)) == want


def test_create_without_device():
    if _lib.lib().rxb200_device_count() > 0:
        pytest.skip("a GPU is present")
    p, _, K, bins, ddc, _, _ = frs.SHAPES["nbfm_k768_m64_t257"]
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.FmMix(p, ddc=ddc, raster=(K, bins))
    assert e.value.code == _lib.ENODEV
