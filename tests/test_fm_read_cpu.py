"""One full_demod per device read with fifth_order passes, on the CPU: the slot-level model of the reference's in-place
passes that the read kernel's counts rest on, the port against the unmodified reference over read sequences that meet
every residue of the read length, their -L levels, and the golden hashes tests/golden/fm_read_golden.json records of
the reference."""
import hashlib
import json
import os
import zlib

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_read as frd

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "fm_read_golden.json")
SHAPES = frd.shapes()


@pytest.mark.parametrize("p_", range(1, 11))
def test_pass_model(p_):
    """For every even read of at least 2^(P+1) int16 up to 8192: no pass reads a slot its predecessor did not write in
    the same read, pass l runs over ceil(L_l / 2) I and floor(L_l / 2) Q samples (the read kernel's pairs n >> l plus a
    lone I when n >> (l-1) is odd), takes the first of the previous pass's outputs and loses at most its last one."""
    for n16 in range(2 << p_, 8193, 2):
        rows, _ = frd.pass_model(n16, p_)
        for l, (ni, nq, oi, oq, stale) in enumerate(rows):
            assert stale == 0, (n16, l)
            length = n16 >> l
            assert (ni, nq) == ((length + 1) // 2, length // 2) == frd.stream_counts(n16, p_, l), (n16, l)
            if l + 1 < p_:
                nxt_i, nxt_q = frd.stream_counts(n16, p_, l + 1)
            else:
                nxt_i, nxt_q = frd.stream_counts(n16, p_, p_)
            assert 0 <= oi - nxt_i <= 1 and 0 <= oq - nxt_q <= 1, (n16, l)
        lp = n16 >> p_
        assert frd.stream_counts(n16, p_, p_) == ((lp + 1) // 2, lp // 2)


def test_read_lens_cover_every_residue():
    for p_ in range(1, 11):
        lens = frd.read_lens(p_, p_)
        g = 2 << p_
        assert {n % g for n in lens} == set(range(0, g, 2)) and g in lens and min(lens) >= g
        assert any((n >> p_) & 1 for n in lens[:-1]), p_       # an odd L_P that a later read follows
    assert all(((n // 2) >> 2) % 2 == 0 for n in frd.read_lens(2, 5, even_dec=True))


def _assert_same(a, b, what):
    assert a[0].size == b[0].size, what
    bad = np.flatnonzero(a[0] != b[0])
    assert bad.size == 0, (what, bad[:5])
    assert np.array_equal(a[1], b[1]), what
    assert np.array_equal(a[2], b[2]), what


@pytest.mark.ref
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_reads_port_equals_reference(name, port, ref_fm):
    p = SHAPES[name]
    lens = frd.read_lens(p.downsample_passes, zlib.crc32(name.encode()), even_dec=p.post_downsample > 1)
    x = frd.stream_for(lens, 30, quiet_half=bool(p.squelch_level))
    a = fac.port_run_seq(port, p, x, lens, return_chunks=True)
    b = fac.ref_run_seq(ref_fm, p, x, lens, return_chunks=True)
    _assert_same(a, b, (name, lens))


@pytest.mark.ref
@pytest.mark.parametrize("name", ["fm2b", "fm_lut_p4_squelch", "usb_p2_squelch_adc", "am_p5_rdc_adc", "raw_p5",
                                  "fm_fast_p10_fir"])
def test_read_levels_port_equals_reference(name, port, ref_fm):
    p = SHAPES[name]
    lens = frd.read_lens(p.downsample_passes, 11)
    x = frd.stream_for(lens, 31, quiet_half=True)
    assert np.array_equal(fac.port_levels_seq(port, p, x, lens), fac.ref_levels_seq(ref_fm, p, x, lens))


def test_port_matches_reference_golden(port):
    gold = json.load(open(GOLDEN))
    cases = frd.golden_cases()
    assert sorted(gold) == sorted(cases)
    for name, (p, x, lens) in cases.items():
        g = gold[name]
        assert g["params"] == {k: int(v) for k, v in vars(p).items()}, name
        assert g["lens_int16"] == list(lens) and g["n_int16"] == x.size, name
        got, rl, _ = fac.port_run_seq(port, p, x, lens, return_chunks=True)
        assert rl.tolist() == g["result_len"], name
        assert hashlib.sha256(got.tobytes()).hexdigest() == g["sha256"], name
