"""rx_power hops of one capture on the CPU: the numpy NCO model (f = 0, the quarter turn, conjugate tables, the frequency
word at negative offsets and at the band edges), the port against the unmodified reference on every named shape's hop
buffers, the golden hashes tests/golden/power_mix_golden.json records, the shell's channel filter from
rxb200_ddc_lowpass, and the refusals that need no device."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

import power_mix as pm
from rx_tools_b200 import _lib, power

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "power_mix_golden.json")
TSTR = "2026-01-01, 00:00:00"


def every_int16(seed):
    """Every int16 value in I and in Q, shuffled: int16[2 * 65536]."""
    rng = np.random.default_rng(seed)
    v = np.arange(-32768, 32768, dtype=np.int32)
    x = np.empty(2 * 65536, dtype=np.int16)
    x[0::2], x[1::2] = rng.permutation(v), rng.permutation(v)
    return x


def test_nco_table_entries():
    t = pm.nco_table()
    assert t.shape == (65536, 2)
    assert t[0].tolist() == [32768, 0] and t[16384].tolist() == [0, -32768]
    assert t[32768].tolist() == [-32768, 0] and t[49152].tolist() == [0, 32768]
    j = np.arange(1, 65536)
    assert np.array_equal(t[65536 - j, 0], t[j, 0]) and np.array_equal(t[65536 - j, 1], -t[j, 1])
    assert np.abs(t).max() == 32768


@pytest.mark.parametrize("n0", [0, 12345, (1 << 32) - 7, (1 << 40) + 3])
def test_model_f0_is_the_identity(n0):
    x = every_int16(1)
    assert np.array_equal(pm.nco_mix(x, 20_000_000, 0, n0), x)
    y, _ = pm.ddc(x, 20_000_000, 0, (1, np.ones(1, np.int32), 0), n0)
    assert np.array_equal(y, x)


@pytest.mark.parametrize("sign", [1, -1])
def test_model_quarter_rate_is_an_exact_quarter_turn(sign):
    R = 20_000_000
    assert pm.nco_word(R, sign * R // 4) == (1 << 30 if sign > 0 else 3 << 30)
    x = every_int16(2)
    y = pm.nco_mix(x, R, sign * R // 4, 5).reshape(-1, 2).astype(np.int64)
    xi, xq = x.reshape(-1, 2).astype(np.int64).T
    k = (5 + np.arange(xi.size)) % 4
    # multiply by exp(-j sign pi/2 k): k = 1 takes (I, Q) to (Q, -I) for +R/4
    want = np.stack([xi, xq], 1)
    for kk, (a, b) in enumerate([((1, 0), (0, 1)), ((0, 1), (-1, 0)), ((-1, 0), (0, -1)), ((0, -1), (1, 0))]):
        if sign < 0 and kk % 2:
            a, b = (-a[0], -a[1]), (-b[0], -b[1])
        m = k == kk
        want[m, 0] = a[0] * xi[m] + a[1] * xq[m]
        want[m, 1] = b[0] * xi[m] + b[1] * xq[m]
    assert np.array_equal(y, want.astype(np.int16).astype(np.int64))


@pytest.mark.parametrize("R,f", [(20_000_000, 1_234_567), (39_160_828, 9_790_207), (61_440_000, 30_719_999),
                                 (7, 3), (22_222_216, 1)])
def test_model_f_and_minus_f_are_conjugates(R, f):
    """The words of f and -f are negatives mod 2^32, so the phases are too, and the entries they pick are conjugates
    wherever the phase is not a rounding tie (theta mod 2^16 == 2^15 rounds up on both sides)."""
    assert (pm.nco_word(R, f) + pm.nco_word(R, -f)) % 2**32 == 0 or (f * 2**32 + R // 2) % R == 0
    n = np.arange(0, 50_000, dtype=np.uint64) * np.uint64(977)
    t = pm.nco_table()
    idx, ths = [], []
    for g in (f, -f):
        w = np.uint64(pm.nco_word(R, g))
        th = ((n & np.uint64(0xffffffff)) * w) & np.uint64(0xffffffff)
        ths.append(th)
        idx.append((((th + np.uint64(32768)) & np.uint64(0xffffffff)) >> np.uint64(16)).astype(np.int64))
    keep = (ths[0] & np.uint64(0xffff)) != np.uint64(0x8000)
    assert keep.sum() > 45_000
    assert np.array_equal(t[idx[0][keep], 0], t[idx[1][keep], 0])
    assert np.array_equal(t[idx[0][keep], 1], -t[idx[1][keep], 1])


def test_model_frequency_word():
    """w against exact rational arithmetic, at negative offsets and at +-(R/2 - 1)."""
    from fractions import Fraction
    import math
    for R in (7, 2_400_000, 20_000_000, 22_222_216, 39_160_828, 61_440_000, 2**31 - 1):
        for f in (0, 1, -1, R // 3, -(R // 3), R // 2 - 1 if R % 2 == 0 else R // 2, -(R // 2 - 1) if R % 2 == 0 else -(R // 2)):
            if 2 * abs(f) >= R:
                continue
            exact = math.floor(Fraction(f * 2**32 + R // 2, R)) % 2**32
            assert pm.nco_word(R, f) == exact, (R, f)
            # the frequency the word runs at is within R / 2^33 of f
            ff = ((exact + 2**31) % 2**32 - 2**31) * R / 2**32
            assert abs(ff - f) <= R / 2**33 + 1e-9, (R, f)
    assert pm.nco_word(20_000_000, -1) == 2**32 - 215    # floor(-2^32 / R + 1/2) = -215 (C's truncation would give -214)


@pytest.mark.parametrize("name", sorted(pm.SHAPES))
def test_golden_hashes(name, port):
    """The model's hop buffers and the port's result over them are the ones the reference saw and made."""
    g = json.load(open(GOLDEN))[name]
    plan, win, R, offs, dd, x = pm.case_input(name)
    assert [plan.n_hops, plan.bin_e, plan.buf_len, plan.downsample, plan.downsample_passes] == g["plan"]
    assert (R, dd[0], dd[1].size, dd[2]) == (g["capture_rate"], g["decim"], g["n_taps"], g["shift"])
    assert pm.digest(x) == g["capture_sha256"]
    hb = pm.Model(R, offs, dd, plan.buf_len).hop_buffers(x)
    assert pm.digest(hb) == g["bufs_sha256"]
    avg, smp = pm.port_result(port, plan, win, hb)
    assert pm.digest(avg) == g["avg_sha256"] and smp.tolist() == g["samples"]
    csv = power.csv_rows(plan, avg, smp, TSTR)
    assert hashlib.sha256(csv.encode()).hexdigest() == g["csv_sha256"]


def test_golden_covers_every_shape():
    assert sorted(json.load(open(GOLDEN))) == sorted(pm.SHAPES)
    plans = {n: pm.shape(n) for n in pm.SHAPES}
    assert plans["fm_band"][2] == 20_000_000 and plans["fm_band"][0].n_hops == 8
    assert plans["hf_crop285"][2] == 39_160_828 and plans["hf_crop285"][0].n_hops == 18
    assert plans["hops260"][0].n_hops > 256
    assert plans["rms"][0].bin_e == 0 and plans["peak_hold"][0].peak_hold == 1
    assert plans["small_F9"][0].downsample_passes > 0 and plans["small_boxcar"][0].downsample > 1
    assert fdd_wide(plans["wide_acc"][4]) and not fdd_wide(plans["fm_band"][4])
    # the table mixer refuses at least one offset of the cropped plan
    p, _, R, offs, _ = plans["uhf_crop25"]
    codes = set()
    for f in offs:
        period = C.c_size_t(0)
        codes.add(_lib.lib().rxb200_fm_mix_table(R, f, None, 0, C.byref(period)))
    assert _lib.EUNSUPPORTED in codes


def fdd_wide(dd):
    return int(np.abs(dd[1].astype(np.int64)).sum()) * 32768 + ((1 << (dd[2] - 1)) if dd[2] else 0) >= (1 << 31)


@pytest.mark.ref
@pytest.mark.parametrize("name", sorted(pm.SHAPES))
def test_port_equals_reference(name, port, ref_power):
    c = pm.SHAPES[name]
    plan, win, R, offs, dd, x = pm.case_input(name)
    rp = ref_power.setup(c["freq"], c["crop"], c["boxcar"], c["fir"], c["peak"], c["window"])
    assert (rp.tune_count, rp.bin_e, rp.buf_len, rp.rate) == (plan.n_hops, plan.bin_e, plan.buf_len, plan.rate)
    assert np.array_equal(ref_power.hop_freqs(), [plan.hop_freq(i) for i in range(plan.n_hops)])
    hb = pm.Model(R, offs, dd, plan.buf_len).hop_buffers(x)
    avg_r, smp_r = ref_power.scan(hb, hb.shape[0])
    avg_p, smp_p = pm.port_result(port, plan, win, hb)
    assert np.array_equal(smp_p, smp_r) and np.array_equal(avg_p, avg_r)


def test_model_split_calls_equal_one_call():
    plan, win, R, offs, dd, x = pm.case_input("peak_hold")
    whole = pm.Model(R, offs, dd, plan.buf_len).hop_buffers(x)
    m, pass16 = pm.Model(R, offs, dd, plan.buf_len), dd[0] * plan.buf_len
    parts = [m.hop_buffers(x[:pass16]), m.hop_buffers(x[pass16:])]
    assert np.array_equal(np.concatenate(parts), whole)


# ------------------------------------------------------------------------------------------------ rxb200_ddc_lowpass
@pytest.mark.parametrize("M,T,S", [(1, 1, 0), (1, 33, 15), (2, 65, 15), (8, 257, 15), (14, 449, 15), (64, 2049, 15),
                                   (4096, 8191, 15), (3, 7, 30), (5, 11, 0)])
def test_lowpass_symmetric_with_exact_dc_gain(M, T, S):
    h = power.ddc_lowpass(M, T, S).astype(np.int64)
    assert h.size == T and h.sum() == 1 << S
    assert np.array_equal(h, h[::-1])


def _response_db(h, freqs):
    n = np.arange(h.size) - (h.size - 1) / 2
    H = np.abs(np.exp(-2j * np.pi * np.outer(freqs, n)) @ h.astype(np.float64)) / h.sum()
    return 20 * np.log10(np.maximum(H, 1e-30))


@pytest.mark.parametrize("M", [2, 8, 14])
def test_lowpass_response_of_the_shell_filter(M):
    h = power.ddc_lowpass(M, min(8191, 32 * M + 1), 15)
    pb = _response_db(h, np.linspace(0, 0.4 / M, 400))
    sb = _response_db(h, np.linspace(0.6 / M, 0.5, 4000))
    assert np.abs(pb).max() <= 0.01, np.abs(pb).max()
    assert sb.max() <= -60.0, sb.max()


def test_lowpass_refusals():
    t = np.zeros(8200, np.int32)
    p = t.ctypes.data_as(C.POINTER(C.c_int32))
    L = _lib.lib()
    for args in ((0, 3, 15), (4097, 3, 15), (2, 0, 15), (2, 4, 15), (2, 8193, 15), (2, 5, -1), (2, 5, 31)):
        assert L.rxb200_ddc_lowpass(*args, p) == _lib.EINVAL, args
    assert L.rxb200_ddc_lowpass(2, 5, 15, None) == _lib.EINVAL


# ------------------------------------------------------------------------------------------------ refusals
def _create(plan, R, offs, dd, window=True):
    pc = plan.to_c()
    win = power.window_table("hamming", 1 << plan.bin_e)
    taps = None if dd[1] is None else np.ascontiguousarray(dd[1], np.int32)
    d = _lib.DdcC(dd[0], 0 if taps is None else taps.size,
                  None if taps is None else taps.ctypes.data_as(C.POINTER(C.c_int32)), dd[2])
    o = None if offs is None else np.ascontiguousarray(offs, np.int32)
    h = C.c_void_p()
    rc = _lib.lib().rxb200_power_mix_create(C.byref(pc), win.ctypes.data_as(C.POINTER(C.c_int)) if window else None,
                                            None, R, None if o is None else o.ctypes.data_as(C.POINTER(C.c_int)),
                                            C.byref(d), 0, C.byref(h))
    if rc == _lib.OK:
        _lib.lib().rxb200_power_mix_destroy(h)
    return rc


def test_create_refusals_before_any_device():
    plan, _, R, offs, dd = pm.shape("fm_band")
    bad_plan = power.Plan(**{**vars(plan), "buf_len": 12})
    one = np.ones(1, np.int32)
    cases = [
        (plan, R, None, dd, _lib.EINVAL),                                   # NULL offsets
        (plan, 0, offs, dd, _lib.EINVAL),                                   # R <= 0
        (plan, -5, offs, dd, _lib.EINVAL),
        (plan, R, offs[:-1] + [R // 2], dd, _lib.EINVAL),                   # |f| >= R/2
        (plan, R, [-(R // 2)] + offs[1:], dd, _lib.EINVAL),
        (plan, R, offs, (0, one, 0), _lib.EINVAL),                          # the ddc's refusals
        (plan, R, offs, (2, one, 63), _lib.EINVAL),
        (plan, R, offs, (2, np.ones(8193, np.int32), 0), _lib.EINVAL),
        (plan, R, offs, (2, None, 0), _lib.EINVAL),
        (bad_plan, R, offs, dd, _lib.EINVAL),                               # the params' refusals
    ]
    for p, r, o, d, code in cases:
        assert _create(p, r, o, d) == code, (r, d[0], d[2])
    assert _create(plan, R, offs, dd, window=False) == _lib.EINVAL
    if _lib.lib().rxb200_device_count() == 0:
        assert _create(plan, R, offs, dd) == _lib.ENODEV
        with pytest.raises(_lib.Rxb200Error) as e:
            power.PowerMix(plan, R, offs, dd)
        assert e.value.code == _lib.ENODEV
