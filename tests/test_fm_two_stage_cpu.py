"""Two-stage mixing handles on the CPU: the numpy model against the rule evaluated term by term in Python integers, the
bins and words the library computes against exact rational arithmetic, both exact anchors against the raster and the
rx_power DDC models, the shell's two-stage capture plan and its refusals, the port against the unmodified reference on
every channel's decimated stream of every shape, the golden hashes tests/golden/fm_two_stage_golden.json records, and
the refusals of create and of the stateless entry, which come before any device work."""
import ctypes as C
import hashlib
import json
import os
from fractions import Fraction

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_ddc as fdd
import fm_mix as fmx
import fm_raster as frs
import fm_two_stage as fts
import power_mix as pmx
from rx_tools_b200 import _lib, fm, power

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "fm_two_stage_golden.json")


def _sat(a, shift):
    y = a if shift == 0 else (a + (1 << (shift - 1))) >> shift
    return max(-32768, min(32767, y))


def _wrap16(v):
    return (v + 32768) % 65536 - 32768


def direct(x, rate, K, offsets, coarse, fine, n0=0):
    """The rule term by term in Python integers over a whole capture (sample i is index n0 + i; none before)."""
    (M1, h1, S1), (M2, h2, S2) = coarse, fine
    tw = frs.table(K).tolist()
    nco = pmx.nco_table().tolist()
    xs = np.asarray(x, dtype=np.int64).reshape(-1, 2).tolist()
    n1 = len(xs) // M1
    out = []
    for f in offsets:
        b, w = fts.bin_word(rate, K, M1, f)
        y = []
        for m in range(n1):
            e = m * M1 + M1 - 1
            ai = aq = 0
            for j, h in enumerate(int(v) for v in h1):
                if e - j < 0:
                    continue
                xi, xq = xs[e - j]
                c, s = tw[(b * (n0 + e - j)) % K]
                ai += h * (xi * c - xq * s)
                aq += h * (xi * s + xq * c)
            y.append((_sat(ai, S1), _sat(aq, S1)))
        z = []
        for m, (yi, yq) in enumerate(y):
            th = ((n0 // M1 + m) * w) % (1 << 32)
            c, s = nco[((th + 32768) % (1 << 32)) >> 16]
            z.append((_wrap16((yi * c - yq * s + 16384) >> 15), _wrap16((yi * s + yq * c + 16384) >> 15)))
        row = []
        for q in range(n1 // M2):
            e = q * M2 + M2 - 1
            ai = aq = 0
            for j, h in enumerate(int(v) for v in h2):
                if e - j >= 0:
                    ai += h * z[e - j][0]
                    aq += h * z[e - j][1]
            row += [_sat(ai, S2), _sat(aq, S2)]
        out.append(row)
    return out


def _random(n, seed, amp=32768):
    return np.random.default_rng(seed).integers(-amp, amp, size=2 * n).astype(np.int16)


@pytest.mark.parametrize("rate,K,offsets,M1,T1,S1,M2,T2,S2", [
    (1000, 3, [0, 333, -499, 170], 1, 1, 15, 1, 1, 0),
    (48_000, 4, [12_000, -5_001, 23_999], 3, 7, 20, 2, 5, 17),
    (7_000, 7, [1234, -3499, 500, 0], 2, 16, 33, 3, 4, 16),
    (96_000, 12, [47_999, -1, 4_000, 4_001], 5, 30, 40, 2, 9, 19),
    (16_000, 16, [-8_000 + 1, 999], 4, 3, 30, 1, 3, 14),
])
def test_model_equals_the_rule(rate, K, offsets, M1, T1, S1, M2, T2, S2):
    rng = np.random.default_rng(K * 100 + T1)
    h1 = rng.integers(-(1 << 22) // (T1 + 1), (1 << 22) // (T1 + 1), size=T1).astype(np.int32)
    h2 = rng.integers(-30000, 30000, size=T2).astype(np.int32)
    x = _random(241, K + T1)
    for n0 in (0, 5 * M1 * M2, (1 << 40) + 3):
        want = direct(x, rate, K, offsets, (M1, h1, S1), (M2, h2, S2), n0)
        got = fts.two_stage_model(x, rate, K, offsets, (M1, h1, S1), (M2, h2, S2), n0)
        assert got.tolist() == want, n0


def _exact(rate, K, M1, f):
    """b_c and w_c through Fraction: the nearest bin centre (ties up), the residual as a fraction of the coarse rate."""
    r = Fraction(f * K, rate)
    bm = int((r + Fraction(rate // 2, rate)).__floor__()) % K
    bp = bm - K if 2 * bm > K else bm
    resid = (Fraction(f) - Fraction(bp * rate, K)) / Fraction(rate, M1)          # cycles per coarse sample
    w = ((resid * (1 << 32)) + Fraction((K * rate) // 2, K * rate)).__floor__() % (1 << 32)
    return bm, int(w)


def test_bins_and_words_against_fractions():
    rng = np.random.default_rng(11)
    cases = [(19_200_000, 32, 16), (2_400_000, 50, 25), (2_048_000, 4096, 64), (1_008_000, 3, 3), (8_064_001, 7, 1),
             (2_304_000, 48, 24), (2_147_483_647, 4096, 4096)]
    for rate, K, M1 in cases:
        lim = (rate - 1) // 2
        offs = [int(v) for v in rng.integers(-lim, lim + 1, size=300)] + [0, lim, -lim]
        offs += [int(k * rate // K) for k in range(-(K // 2), K // 2 + 1) if abs(k * rate // K) <= lim][:200]
        bins, words = fm.two_stage_word(rate, K, M1, offs)
        for f, b, w in zip(offs, bins, words):
            assert (b, w) == fts.bin_word(rate, K, M1, f) == _exact(rate, K, M1, f), (rate, K, M1, f)


def test_ties_round_up_and_centres_have_word_zero():
    rate, K, M1 = 2_304_000, 48, 24
    step = rate // K
    bins, words = fm.two_stage_word(rate, K, M1, [k * step for k in range(-23, 24)])
    assert bins == [k % K for k in range(-23, 24)] and set(words) == {0}
    edges = [k * step + step // 2 for k in range(-24, 23)]
    bins, _ = fm.two_stage_word(rate, K, M1, edges)
    assert bins == [(k + 1) % K for k in range(-24, 23)]
    assert fm.two_stage_word(rate, K, M1, [step // 2 - 1])[0] == [0]


def test_anchor_identity_coarse_stage_is_the_power_ddc():
    """M1 = 1, T1 = 1, h1 = {1}, S1 = 15, channels on bin 0: rx_power's DDC of the same offset (even R)."""
    rate, K = 2_400_000, 16
    offs = [0, 17, -74_999, 74_998, 31_415]
    x = _random(4001, 3)
    for M2, T2, S2 in ((1, 1, 0), (4, 33, 15), (7, 64, 20)):
        h2 = fdd.lowpass(T2, 0.1, gain_bits=S2) if T2 > 1 else np.ones(1, np.int32)
        for n0 in (0, 12345, (1 << 40) + 3):
            got = fts.two_stage_model(x, rate, K, offs, (1, np.ones(1, np.int32), 15), (M2, h2, S2), n0)
            for c, f in enumerate(offs):
                assert fm.two_stage_word(rate, K, 1, [f])[0] == [0]
                want, _ = pmx.ddc(x, rate, f, (M2, h2, S2), n0)
                assert got[c].tobytes() == want.tobytes(), (M2, n0, f)


def test_anchor_unit_fine_stage_is_the_raster():
    """M2 = 1, T2 = 1, h2 = {1}, S2 = 0 and channels on bin centres: the raster rule with those bins."""
    rate, K = 2_400_000, 48
    bins = [0, 1, 23, 47, 25, 1]
    offs = [int(k * rate // K) if 2 * k <= K else int((k - K) * rate // K) for k in bins]
    x = _random(3001, 5)
    h1 = fdd.lowpass(65, 0.02, gain_bits=20)
    for M1, S1 in ((1, 20), (3, 35), (8, 30)):
        got = fts.two_stage_model(x, rate, K, offs, (M1, h1, S1), (1, np.ones(1, np.int32), 0), n0=0)
        want, _ = frs.raster_model(x, K, bins, h1, M1, S1)
        assert got.tobytes() == want.tobytes(), M1
        assert fm.two_stage_word(rate, K, M1, offs) == (bins, [0] * len(bins))


def test_planner_against_the_restated_rule():
    rng = np.random.default_rng(3)
    for i in range(200):
        c = int(rng.choice([24_000, 48_000, 170_000, 300_000, 2_400_000, 1_008_000]))
        base = int(rng.integers(50_000_000, 1_000_000_000))
        grid = int(rng.choice([5_000, 12_500, 25_000, 100_000, 1]))
        t = [base + grid * int(k) for k in rng.integers(0, int(rng.integers(1, 400)), size=int(rng.integers(1, 12)))]
        want = fts.plan_restated(t, c, 1 << 62)
        for cap in ((want[1], want[1] - 1) if want else (1 << 62,)):
            w = fts.plan_restated(t, c, cap)
            if w is None:
                with pytest.raises(_lib.Rxb200Error) as e:
                    fm.plan_capture_two_stage(t, c, cap)
                assert e.value.code == _lib.EINVAL
                continue
            p, offs = fm.plan_capture_two_stage(t, c, cap)
            fc, R, K, M1, T1, o = w
            assert (p.centre_hz, p.capture_rate, p.n_bins, p.coarse_decim, p.coarse_taps) == (fc, R, K, M1, T1), (t, c)
            assert (p.coarse_shift, p.fine_decim, p.fine_taps, p.fine_shift) == (30, 4, 129, 15)
            assert offs == o
            # the same centre and offsets as the single-stage plan wherever that one plans
            try:
                q, o1 = fm.plan_capture(t, c, 1 << 40)
            except _lib.Rxb200Error:
                continue
            assert q.centre_hz == fc and o1 == o and 4 * -(-q.decim // 4) == 4 * M1


def test_planner_refusals():
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.plan_capture_two_stage([100_000_000], 300_000, 1 << 40)          # M' = 4 < 8
    assert e.value.code == _lib.EINVAL
    t = [100_000_000, 104_500_000, 109_000_000]                             # M = 31 -> M' = 32, R = 9.6 Msps
    p, offs = fm.plan_capture_two_stage(t, 300_000, 9_600_000)
    assert (p.capture_rate, p.n_bins, p.coarse_decim) == (9_600_000, 16, 8) and offs == [-4_500_000, 0, 4_500_000]
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.plan_capture_two_stage(t, 300_000, 9_599_999)
    assert e.value.code == _lib.EINVAL and b"9600000" in _lib.lib().rxb200_last_error()
    for bad in (([], 300_000), ([100], 0), ([-1, 5], 300_000)):
        with pytest.raises(_lib.Rxb200Error) as e:
            fm.plan_capture_two_stage(bad[0], bad[1], 1 << 40)
        assert e.value.code == _lib.EINVAL
    with pytest.raises(_lib.Rxb200Error):
        fm.plan_capture_two_stage([0, 80_000_000], 300_000, 1 << 40)        # M' = 536 > 256
    plan, _ = fm.plan_capture_two_stage(t, 300_000, 1 << 40)
    K, coarse, fine = fts.plan_stages(4 * plan.coarse_decim)
    assert K == plan.n_bins and frs.sum_abs(coarse[1]) < (1 << 22)
    assert np.array_equal(coarse[1], power.ddc_lowpass(plan.coarse_decim, plan.coarse_taps, 15))


def test_shapes_cover_the_named_cases():
    assert len(fts.SHAPES["nbfm_19m2_c256"][3]) == 256 and fts.SHAPES["nbfm_19m2_c256"][1] == 19_200_000
    Ks = {s[2] for s in fts.SHAPES.values()}
    assert {3, 4096} <= Ks
    for name in ("raw_sat_k3", "raw_sat_k4096"):
        assert frs.sum_abs(fts.SHAPES[name][4][1]) == (1 << 22) - 1
    _, rate, K, offs, coarse, fine, x, reads = fts.case_input("raw_sat_k3")
    y = fts.coarse_streams(x, K, [0, 1, 2], coarse, x.size // 2 // coarse[0])
    assert any((np.abs(v.astype(np.int32)) >= 32767).any() for v in y.values())          # coarse outputs saturate
    rate, K, offs = fts.SHAPES["raw_centres_edges"][1:4]
    bins, words = fm.two_stage_word(rate, K, fts.SHAPES["raw_centres_edges"][4][0], offs)
    assert words.count(0) >= 4 and 24 in bins                                            # centres, and the K/2 tie
    rate, K, offs = fts.SHAPES["nbfm_19m2_c256"][1:4]
    _, words = fm.two_stage_word(rate, K, 16, offs)
    assert 0 not in words                                                                # none on the grid


def _channel_reads(name, seed=0):
    p, rate, K, offs, coarse, fine, x, reads = fts.case_input(name, seed)
    return p, fts.decimated_reads(x, rate, K, offs, coarse, fine, reads)


@pytest.mark.ref
@pytest.mark.parametrize("name", sorted(fts.SHAPES))
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
    p, chans = _channel_reads("fm_lut_squelch", seed=2)
    for c, reads in enumerate(chans):
        y, lens = fdd.nonempty(reads)
        assert np.array_equal(fac.port_levels_seq(port, p, y, lens), fac.ref_levels_seq(ref_fm, p, y, lens)), c


def test_port_matches_reference_golden(port):
    gold = json.load(open(GOLDEN))
    assert sorted(gold) == sorted(fts.SHAPES)
    for name in fts.SHAPES:
        p, rate, K, offs, coarse, fine, x, reads = fts.case_input(name)
        g = gold[name]
        assert g["params"] == {k: int(v) for k, v in vars(p).items()}, name
        assert (g["capture_rate"], g["n_bins"], g["offsets_hz"]) == (rate, K, offs), name
        assert g["lens_int16"] == reads and g["n_int16"] == x.size, name
        for key, d in (("coarse", coarse), ("fine", fine)):
            assert g[key] == {"decim": d[0], "taps": [int(v) for v in d[1]], "shift": d[2]}, name
        assert g["capture_sha256"] == hashlib.sha256(x.tobytes()).hexdigest(), name
        for c, dec in enumerate(fts.decimated_reads(x, rate, K, offs, coarse, fine, reads)):
            gc = g["channels"][c]
            assert [int(r.size) for r in dec] == gc["dec_len"], (name, c)
            y, lens = fdd.nonempty(dec)
            assert hashlib.sha256(y.tobytes()).hexdigest() == gc["dec_sha256"], (name, c)
            got, rl, _ = fac.port_run_seq(port, p, y, lens, return_chunks=True)
            assert rl.tolist() == gc["result_len"], (name, c)
            assert hashlib.sha256(got.tobytes()).hexdigest() == gc["sha256"], (name, c)


P0 = fmx.SHAPES["fm5a_lut_d100"][0]
C1 = (4, np.array([1, 2, 1], np.int32), 17)
F1 = (2, np.array([1, 1], np.int32), 1)


@pytest.mark.parametrize("rate,K,offs,coarse,fine", [
    (2_400_000, 2, [0], C1, F1), (2_400_000, 4097, [0], C1, F1),                          # K
    (2_400_000, 8, [0], (4, np.full(4, 1 << 20, np.int32), 30), F1),                      # sum |h1| = 2^22
    (2_400_000, 8, [0], (0, [1], 0), F1), (2_400_000, 8, [0], C1, (2, [1] * 8193, 0)),    # the ddc ranges
    (2_400_000, 8, [0], C1, (4, [1], 63)),
    (0, 8, [0], C1, F1), (-5, 8, [0], C1, F1),                                            # R
    (2_400_000, 8, [1_200_000], C1, F1), (2_400_000, 8, [-1_200_000], C1, F1),            # |f| >= R/2
    (2_400_000, 8, [], C1, F1),                                                           # no channel
    (2_400_000, 8, [0], (64, [1], 16), (65, [1], 0)),                                     # M1 M2 = 4160 > 4096
])
def test_create_and_device_entry_refuse_before_looking_for_a_device(rate, K, offs, coarse, fine):
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.FmMix(P0, rate, offs, two_stage=(K, coarse, fine))
    assert e.value.code == _lib.EINVAL
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.two_stage_device(rate, K, offs, 0, coarse, fine, 16, 1000, 16)     # never dereferenced
    assert e.value.code == _lib.EINVAL


def test_create_refuses_null_arguments_and_keeps_the_params_refusals():
    p = fm.FmParams.from_any(P0).to_c()
    t1, t2 = np.array([1, 2, 1], np.int32), np.array([1, 1], np.int32)
    d1 = _lib.DdcC(4, 3, t1.ctypes.data_as(C.POINTER(C.c_int32)), 17)
    d2 = _lib.DdcC(2, 2, t2.ctypes.data_as(C.POINTER(C.c_int32)), 1)
    offs = np.array([0, 3000], np.int32)
    po = offs.ctypes.data_as(C.POINTER(C.c_int))
    h = C.c_void_p()
    L = _lib.lib()
    R = 2_400_000
    assert L.rxb200_fm_mix_create_two_stage(C.byref(p), R, 8, None, 2, C.byref(d1), C.byref(d2), 0, C.byref(h)) == _lib.EINVAL
    assert L.rxb200_fm_mix_create_two_stage(C.byref(p), R, 8, po, 2, None, C.byref(d2), 0, C.byref(h)) == _lib.EINVAL
    assert L.rxb200_fm_mix_create_two_stage(C.byref(p), R, 8, po, 2, C.byref(d1), None, 0, C.byref(h)) == _lib.EINVAL
    assert L.rxb200_fm_mix_create_two_stage(None, R, 8, po, 2, C.byref(d1), C.byref(d2), 0, C.byref(h)) == _lib.EINVAL
    assert L.rxb200_fm_mix_create_two_stage(C.byref(p), R, 8, po, 2, C.byref(d1), C.byref(d2), 0, None) == _lib.EINVAL
    assert L.rxb200_two_stage_device(R, 8, po, 2, 0, C.byref(d1), C.byref(d2), None, 100, 16, None) == _lib.EINVAL
    assert L.rxb200_two_stage_device(R, 8, po, 2, 0, C.byref(d1), C.byref(d2), 18, 100, 16, None) == _lib.EINVAL
    assert L.rxb200_two_stage_device(R, 8, po, 2, 0, C.byref(d1), C.byref(d2), 16, 100, 18, None) == _lib.EINVAL
    b, w = (C.c_int * 2)(), (C.c_uint32 * 2)()
    assert L.rxb200_two_stage_word(R, 8, 4, po, 2, None, w) == _lib.EINVAL
    assert L.rxb200_two_stage_word(R, 8, 4, po, 0, b, w) == _lib.EINVAL
    assert L.rxb200_two_stage_word(R, 8, 0, po, 2, b, w) == _lib.EINVAL
    # a chain parameter the member refuses: the same code as a decimating handle's
    bad = fm.FmParams.from_any(fac.with_(P0, downsample=0)).to_c()
    want = L.rxb200_fm_mix_create_ddc(C.byref(bad), R, po, 1, C.byref(d2), 0, C.byref(h))
    assert want != _lib.OK
    assert L.rxb200_fm_mix_create_two_stage(C.byref(bad), R, 8, po, 2, C.byref(d1), C.byref(d2), 0, C.byref(h)) == want


def test_create_without_device():
    if _lib.lib().rxb200_device_count() > 0:
        pytest.skip("a GPU is present")
    p, rate, K, offs, coarse, fine, _, _ = fts.SHAPES["fm2b_f9"]
    with pytest.raises(_lib.Rxb200Error) as e:
        fm.FmMix(p, rate, offs, two_stage=(K, coarse, fine))
    assert e.value.code == _lib.ENODEV
