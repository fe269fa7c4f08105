"""The port against the unmodified reference on chunks of any whole number of complex samples, for every shape without
fifth_order passes: uniform chunk lengths that are not multiples of 8 complex (the stream not a multiple of the chunk
either), ragged sequences of chunk lengths with one run call per chunk on one configured state, the -L levels of
both, and the golden hashes tests/golden/fm_any_chunk_golden.json records of the reference."""
import hashlib
import json
import os
import zlib

import numpy as np
import pytest

import fm_any_chunk as fac

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "fm_any_chunk_golden.json")
SHAPES = fac.shapes()
UNIFORM_CHUNKS = [997, 1001, 1002, 1003, 4093]     # complex samples


def _input(name, n_complex, seed):
    p = SHAPES[name]
    return fac.loud_quiet(n_complex, seed) if p.squelch_level else fac.signal(n_complex, seed)


def _assert_same(a, b, what):
    assert a[0].size == b[0].size, what
    bad = np.flatnonzero(a[0] != b[0])
    assert bad.size == 0, (what, bad[:5])
    assert np.array_equal(a[1], b[1]), what        # result_len per chunk
    assert np.array_equal(a[2], b[2]), what        # squelch_hits per chunk


@pytest.mark.ref
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_uniform_odd_chunks_port_equals_reference(name, port, ref_fm):
    p = SHAPES[name]
    for i, c in enumerate(UNIFORM_CHUNKS):
        n = 7 * c + 2 * p.downsample + 3 * i + 1          # a short last chunk, still at least one boxcar long
        x = _input(name, n, 10 + i)
        a = port.fm_run(p, x, 2 * c, return_chunks=True)
        b = ref_fm.run(p, x, 2 * c, return_chunks=True)
        _assert_same(a, b, (name, c))


@pytest.mark.ref
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_ragged_sequences_port_equals_reference(name, port, ref_fm):
    p = SHAPES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    for k in range(3):
        lens = fac.ragged_lens(rng, 12, fac.shortest(p), 6000 if k else 300)
        x = _input(name, fac.seq_len(lens), 50 + k)
        a = fac.port_run_seq(port, p, x, lens, return_chunks=True)
        b = fac.ref_run_seq(ref_fm, p, x, lens, return_chunks=True)
        _assert_same(a, b, (name, k, lens))


# chunks that complete no boxcar, in runs: (parameters, chunk lengths in complex samples, stream length)
EMPTY_RUNS = {
    "fm5a_chunks_of_1": (fac.FM5A, [1], 2500),
    "lut_d12_chunks_of_8": (fac.NBFM12, [8], 1603),
    "lut_d12_mixed": (fac.NBFM12, [8, 1, 3, 40, 2, 2, 5, 11, 24], 3001),
    **{f"{an}_d10_mixed": (fac.with_(fac.SHORT_STD, custom_atan=a), [3, 4, 9, 1, 16, 2, 7], 2001)
       for a, an in ((0, "std"), (1, "fast"), (2, "lut"), (3, "ale"))},
    "fast_d6_deemph_resample": (fac.WBFM, [2, 3, 1, 5, 13], 3000),
    "lut_d3_deemph_even": (fac.shapes()["fm_lut_d3_deemph_even"], [1, 1, 2, 1, 4], 1000),
    "am_d42": (fac.AM, [8, 30, 1, 50], 3000),
    "raw_d42": (fac.RAW, [8, 30, 1, 50], 3000),
    # -o 2 at D = 12: the boxcar phase returns to 0 every cycle, every chunk decimates to 0 or 2
    "lut_d12_o2": (fac.with_(fac.NBFM12, post_downsample=2), fac.O2_CYCLE, 20 * sum(fac.O2_CYCLE)),
    "std_d12_o2_deemph": (fac.with_(fac.NBFM12, custom_atan=0, post_downsample=2, deemph=1, deemph_a=7),
                          fac.O2_CYCLE, 20 * sum(fac.O2_CYCLE)),
}


@pytest.mark.ref
@pytest.mark.parametrize("name", sorted(EMPTY_RUNS))
def test_empty_chunk_runs_port_equals_reference(name, port, ref_fm):
    """Runs of chunks too short to complete a boxcar: after each, fm_demod carries (0, 0) in the reference, and the next
    emitting chunk's first output is exactly 0."""
    p, chunks, n = EMPTY_RUNS[name]
    lens = [2 * c for c in chunks]
    x = fac.signal(n, zlib.crc32(name.encode()) % 1000)
    a = fac.port_run_seq(port, p, x, lens, return_chunks=True)
    b = fac.ref_run_seq(ref_fm, p, x, lens, return_chunks=True)
    _assert_same(a, b, name)
    assert np.any(a[1] == 0) and np.any(a[1] > 0), name
    if p.mode == fac.M_FM and not (p.deemph or p.rate_out2 > 0 or p.post_downsample > 1):
        zero = fac.after_empty(a[1])
        assert zero.size and np.all(a[0][zero] == 0), name


@pytest.mark.ref
@pytest.mark.parametrize("name", ["fm_lut_d42_squelch", "usb_d5_squelch_adc", "wbfm", "am_d42_rdc_adc", "raw"])
def test_levels_port_equals_reference(name, port, ref_fm):
    """-L's per-chunk rms() on uniform odd chunks and on a ragged sequence."""
    p = SHAPES[name]
    x = _input(name, 5 * 1001 + 321, 7)
    assert np.array_equal(port.fm_levels(p, x, 2 * 1001), ref_fm.levels(p, x, 2 * 1001))
    lens = fac.ragged_lens(np.random.default_rng(3), 12, 2 * p.downsample, 3000)
    x = _input(name, fac.seq_len(lens), 8)
    assert np.array_equal(fac.port_levels_seq(port, p, x, lens), fac.ref_levels_seq(ref_fm, p, x, lens))


def test_chunk_sequence_bounds():
    assert fac.seq_bounds(20, [6, 4]) == [(0, 6), (6, 4), (10, 6), (16, 4)]
    assert fac.seq_bounds(11 * 2, [6]) == [(0, 6), (6, 6), (12, 6), (18, 4)]
    with pytest.raises(AssertionError):
        fac.seq_bounds(10, [3])                 # half a complex sample


def test_port_matches_reference_golden(port):
    """The port against the reference's sha256 of the benchmark shapes at odd chunks and the ragged sequences (minted by
    golden/make_fm_any_chunk_golden.py)."""
    gold = json.load(open(GOLDEN))
    cases = fac.golden_cases()
    assert sorted(gold) == sorted(cases)
    for name, (p, x, lens) in cases.items():
        g = gold[name]
        assert g["params"] == {k: int(v) for k, v in vars(p).items()}, name
        assert g["lens_int16"] == list(lens) and g["n_int16"] == x.size, name
        got, rl, _ = fac.port_run_seq(port, p, x, lens, return_chunks=True)
        assert rl.tolist() == g["result_len"], name
        assert hashlib.sha256(got.tobytes()).hexdigest() == g["sha256"], name


def test_golden_covers_the_shapes():
    cases = fac.golden_cases()
    assert {n for n in cases if n.startswith("fm1_")} == {"fm1_std_c131071", "fm1_fast_c131071", "fm1_lut_c131071"}
    assert all(lens == [2 * 131071] for n, (_, _, lens) in cases.items() if n.startswith(("fm1", "fm2a")))
    assert all(lens == [2 * 131069] for n, (_, _, lens) in cases.items() if n.startswith("fm5a"))
    seq = [c for n, c in cases.items() if n.startswith("seq_")]
    assert {p.mode for p, _, _ in seq} == {0, 1, 2, 3, 4} and {p.custom_atan for p, _, _ in seq if p.mode == 0} == {0, 1, 2, 3}
    assert all(len(set(lens)) > 1 and any(v % 16 for v in lens) for _, _, lens in seq)
