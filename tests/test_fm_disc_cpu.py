"""The port's discriminators (oracle/rx_oracle.c) against the reference's own polar_discriminant, polar_disc_fast,
polar_disc_lut and esbensen (src/rtl_fm.c:476-582, compiled unmodified into oracle/_ref) over every operand class of
fm_disc.py -- except the quads the reference cannot evaluate, which the harness marks and never hands to it; the port's
std value against the exact truncation from mpmath wherever it is not near an integer; the guard-band fixture's
distances; the port's defined result where the reference crashes in -A lut, alone and through a chain; and the port's
count of near-integer polar_discriminant evaluations, which the GPU comparisons of -A std use to decide whether a 1-LSB
difference is allowed at all."""
import importlib.util
import os

import numpy as np
import pytest

import fm_any_chunk as fac
import fm_disc as fd

HERE = os.path.dirname(os.path.abspath(__file__))


def _exact(cr, cj):
    """(trunc(V), |V - round(V)|, V > round(V)) of V = atan2(cj, cr) / 3.14159 * 2^14 at 50 digits (3.14159 as the C
    double)"""
    import mpmath
    with mpmath.workdps(50):
        v = mpmath.atan2(int(cj), int(cr)) / mpmath.mpf(3.14159) * 16384
        r = v - mpmath.nint(v)
        return int(mpmath.floor(v) if v >= 0 else mpmath.ceil(v)), float(abs(r)), bool(r > 0)


def _ref_forms(q):
    """the reference forms that apply to quads q: esbensen only on int16 samples (its int32 divisor is the point)"""
    forms = [fd.STD, fd.FAST, fd.LUT]
    return forms + [fd.ALE] if np.all(fd.in_int16(q)) else forms


def _port_vs_ref(port, ref_fm, form, q, what):
    got, _ = port.disc_many(form, q, want_near=False)
    want, skipped = ref_fm.disc_many(form, q)
    cr, cj = fd.conj(q)
    crash = (form == fd.LUT) & (np.abs(cr.astype(np.int64)) == 1) & ((cj.astype(np.int64) & 0xFFFFFF) == 1 << 23)
    assert np.array_equal(skipped, crash), (what, form)
    bad = np.flatnonzero((got != want) & ~skipped)
    assert bad.size == 0, (what, fd.FORM_NAMES[form], q[bad[:5]], got[bad[:5]], want[bad[:5]])
    return int(skipped.sum())


def test_port_equals_reference_small_operands(port, ref_fm):
    """every (cr, cj) with |cr|, |cj| <= 2048 through all four reference discriminators"""
    for q in fd.small_slices():
        for form in (fd.STD, fd.FAST, fd.LUT, fd.ALE):
            assert _port_vs_ref(port, ref_fm, form, q, "small") == 0


@pytest.mark.parametrize("name", sorted(fd.random_classes()))
def test_port_equals_reference_by_class(name, port, ref_fm):
    q = fd.random_classes()[name]
    skipped = sum(_port_vs_ref(port, ref_fm, form, q, name) for form in _ref_forms(q))
    if name == "lut_crash":
        assert skipped == q.shape[0] == 256                   # every one of them crashes the reference
    elif name.startswith("lut_shift_wrap"):
        assert skipped > 0                                    # cr = +-1 against cj = +-2^23 is among them
    else:
        assert skipped == 0, name


def test_port_equals_reference_on_edges_and_stream(port, ref_fm):
    for name, q in fd.edges().items():
        for form in (fd.STD, fd.FAST, fd.LUT):
            _port_vs_ref(port, ref_fm, form, q, name)
    q = fd.stream_class()
    for form in (fd.STD, fd.FAST, fd.LUT, fd.ALE):
        _port_vs_ref(port, ref_fm, form, q, "stream")


def test_lut_crash_pairs_return_linear_range(port):
    """Where the reference crashes (cj << 8 == INT_MIN, |cr| = 1) the port returns cj > 0 ? 8192 : -8192, like the
    library; every other int16 quad of the search's neighbourhood keeps the reference's rule (checked above)."""
    q = fd.lut_crash_quads()
    cr, cj = fd.conj(q)
    assert np.all(np.abs(cr) == 1) and np.all((cj.astype(np.int64) << 8).astype(np.int32) == fd.INT_MIN)
    got, _ = port.disc_many(fd.LUT, q, want_near=False)
    assert np.array_equal(got, np.where(cj > 0, 8192, -8192))
    # the two pairs of the issue's example: (-2047, 2048) after (2049, 2048), and (-2047, -2048) after (-2049, 2048)
    got, _ = port.disc_many(fd.LUT, [[-2047, 2048, 2049, 2048], [-2047, -2048, -2049, 2048]], want_near=False)
    assert got.tolist() == [8192, 8192]


def test_std_equals_exact_truncation(port):
    """The port's std value (glibc's atan2, the reference's expression) is trunc(V) of the exact V wherever V is not
    within 2^-30 of an integer, and the near flag is set exactly where mpmath puts V that close: so the 'truth' the
    device forms are held to is the exact value, not one more libm."""
    rng = np.random.default_rng(fd.SEED + 7)
    sets = dict(fd.edges())
    for name, q in fd.random_classes().items():
        sets[name] = q[rng.choice(q.shape[0], min(q.shape[0], 1500), replace=False)]
    small = next(iter(fd.small_slices(64)))
    sets["small"] = small[rng.choice(small.shape[0], 3000, replace=False)]
    sets["near_pair"] = fd.pairs([fd.NEAR_PAIR[0], fd.NEAR_PAIR[0]], [fd.NEAR_PAIR[1], -fd.NEAR_PAIR[1]])
    n_near = 0
    for name, q in sets.items():
        got, near = port.disc_many(fd.STD, q)
        cr, cj = fd.conj(q)
        for i in range(q.shape[0]):
            if cr[i] == 0 and cj[i] == 0:
                continue                                      # atan2(0, 0) = 0: no exact value to compare
            t, d, _ = _exact(cr[i], cj[i])
            assert bool(near[i]) == (d < 2.0 ** -30 and not (cj[i] == 0 and cr[i] > 0)), (name, cr[i], cj[i], d)
            if not near[i]:
                assert got[i] == t, (name, cr[i], cj[i], got[i], t)
        n_near += int(near.sum())
    assert n_near >= 2                                        # the near pair, both signs (and what the libm edges hold)


def _edge_buckets():
    spec = importlib.util.spec_from_file_location("make_disc_edges", os.path.join(HERE, "golden", "make_disc_edges.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m.BUCKETS


def test_edge_fixture_distances():
    """every pair of golden/disc_edges.npz lies where its name says: operand range and exact distance band"""
    z = np.load(fd.EDGES)
    buckets = _edge_buckets()
    assert sorted(z.files) == sorted(name for name, *_ in buckets)
    for name, _, (lo, hi), below in buckets:
        a = z[name].astype(np.int64)
        assert a.shape == (256, 2) and len({tuple(r) for r in a.tolist()}) == 256, name
        big = np.abs(a).max(axis=1)
        assert np.all(big < (1 << 24)) if below else np.all((big >= (1 << 24)) & (big < (1 << 31))), name
        sides = set()
        for cr, cj in a:
            _, d, above = _exact(cr, cj)
            assert lo <= d < hi, (name, cr, cj, d)
            sides.add(above)
        assert sides == {False, True}, name                 # just below and just above an integer


def _near_chain_input(port, D):
    """decimated samples (1, 0) then NEAR_PAIR somewhere inside the first chunk, zeros elsewhere: one near-integer
    polar_discriminant evaluation in the whole run (every other conjugate product is (0, 0) or on the positive axis)"""
    dec = np.zeros((64, 2), dtype=np.int64)
    dec[20] = (1, 0)
    dec[21] = fd.NEAR_PAIR
    return fd.crafted_capture(port, D, dec)


def test_std_near_counter_counts(port):
    p = fac.with_(fac.SHORT_STD, downsample=256, offset_tuning=1)
    port.std_near_count()                                     # read and reset whatever ran before
    x = fac.signal(20000, 3)
    port.fm_run(p, x, 2 * 4096)
    assert port.std_near_count() == 0                         # a plain run meets none
    y = _near_chain_input(port, 256)
    out = port.fm_run(p, y, 2 * 8192)
    t, d, _ = _exact(*fd.NEAR_PAIR)
    assert d < 2.0 ** -30 and out.size == 64
    assert int(out[21]) in (t, t + 1)                         # V is 4.6e-10 below t + 1: glibc truncates one way
    assert port.std_near_count() == 1
    assert port.std_near_count() == 0                         # read and reset
    port.fm_run(fac.with_(p, custom_atan=1), y, 2 * 8192)
    assert port.std_near_count() == 0                         # -A fast: only the chunk's first sample is atan2's
    port.fm_run(fac.with_(p, custom_atan=1), y, 2 * 256 * 21)
    assert port.std_near_count() == 1                         # ... and F8 counts: a chunk that starts at the near pair


def test_lut_chain_on_crash_pairs(port):
    """-A lut through the port's chain on a capture whose decimated samples carry every crash pair: each gives
    cj > 0 ? 8192 : -8192, and the run completes (the reference's process would not)"""
    D, chunk_c = 100, 25000
    dec, placed = fd.crash_sequence(D, 2000, chunk_c // D)
    x = fd.crafted_capture(port, D, dec, chunk_complex=chunk_c)
    out = port.fm_run(fac.FM5A, x, 2 * chunk_c)
    assert out.size == 2000
    for n, pos in placed:
        assert int(out[n]) == (8192 if pos else -8192), n
