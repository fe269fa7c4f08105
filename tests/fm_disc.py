"""Operand classes of the discriminator tests (test_fm_disc_cpu.py, test_fm_disc_gpu.py): seeded quads (ar, aj, br, bj)
of int32, the sample x[n] and the one before it, at the operands where the device forms of the discriminators could go
wrong.  A quad (cr, cj, 1, 0) hands the pair (cr, cj) straight to a discriminator as its conjugate product.

Classes (name -> int32 [n][4]):
  small:      every (cr, cj) with |cr|, |cj| <= 2048, in slices (small_slices)
  mag_*:      random pairs by magnitude class: < 2^16, [2^16, 2^19), [2^19, 2^24), exactly +-2^24, >= 2^24, INT_MIN
  octant:     |cr| = |cj| and +-1 around it, cr = 0, cj = 0 with either sign of cr
  fast_*:     fast_atan2: ||cr| - |cj|| at 2^19 - 1 .. 2^19 + 1 (4096 n leaves int32), divisors |cr| + |cj| that wrap to
              <= 0, quotients 4096 n / den that are exact integers (and one off)
  lut_*:      polar_disc_lut: |x| = |(cj << 8) / cr| at 131071 / 131072, cj around +-2^23 where the shift wraps, and the
              int16 quads whose (cj << 8) is INT_MIN with |cr| = 1 (the reference crashes there: lut_crash)
  i16_*:      int16 quads: random, and the +-32768 corners where AM's and esbensen's int32 sums wrap
  stream:     every 8-bit-range (di, dq) in [-127, 128]^2 against a few hundred previous samples, extremes included
The guard-band edges, pairs whose exact value lies at a set distance from an integer, are a committed fixture
(golden/disc_edges.npz, made by golden/make_disc_edges.py) so that only numpy is needed to read them.
No class holds cr == cj == INT_MIN (fast_atan2's C division by zero, unreachable from int16 samples).
"""
import os

import numpy as np

SEED = 1017
INT_MIN = -(1 << 31)
I32_MAX = (1 << 31) - 1
HERE = os.path.dirname(os.path.abspath(__file__))
EDGES = os.path.join(HERE, "golden", "disc_edges.npz")

# forms of rxb200_fm_disc_device / orx_disc_many
STD, FAST, LUT, ALE, ATAN2, STD_FP64, ROWS, STREAM, AM = range(9)
FORM_NAMES = ["std", "fast", "lut", "ale", "atan2", "std_fp64", "rows", "stream", "am"]
STD_FORMS = (STD, ATAN2, STD_FP64)


def pairs(cr, cj):
    """quads (cr, cj, 1, 0): the conjugate product of x[n] = (cr, cj) and x[n-1] = (1, 0) is (cr, cj)"""
    cr = np.asarray(cr, dtype=np.int64).reshape(-1)
    cj = np.asarray(cj, dtype=np.int64).reshape(-1)
    q = np.zeros((cr.size, 4), dtype=np.int32)
    q[:, 0] = cr.astype(np.int32)
    q[:, 1] = cj.astype(np.int32)
    q[:, 2] = 1
    return q


def small_slices(n_slices=8):
    """every (cr, cj) with |cr|, |cj| <= 2048 (4097^2 = 16.8 M pairs), as n_slices quad arrays by rows of cr"""
    v = np.arange(-2048, 2049, dtype=np.int64)
    for rows in np.array_split(v, n_slices):
        cr, cj = np.meshgrid(rows, v, indexing="ij")
        yield pairs(cr, cj)


def _mag(rng, n, lo_bits, hi_bits):
    """n magnitudes log-uniform in [2^lo_bits, 2^hi_bits), with the class ends themselves included"""
    m = np.floor(np.exp2(rng.uniform(lo_bits, hi_bits, n))).astype(np.int64)
    m[:4] = [1 << lo_bits if lo_bits > 0 else 0, (1 << lo_bits) + 1, (1 << hi_bits) - 2, (1 << hi_bits) - 1]
    return np.clip(m, 0, (1 << hi_bits) - 1)


def _sign(rng, v):
    return np.where(rng.random(v.size) < 0.5, -v, v)


def _no_double_int_min(q):
    cr, cj = q[:, 0].astype(np.int64), q[:, 1].astype(np.int64)
    keep = ~((cr == INT_MIN) & (cj == INT_MIN) & (q[:, 2] == 1) & (q[:, 3] == 0))
    return q[keep]


def magnitude_classes(n=200_000, seed=SEED):
    """random int32 pairs: both components in the class, and one in the class with the other anywhere below it"""
    rng = np.random.default_rng(seed)
    out = {}
    for name, lo, hi in (("mag_lt16", 0, 16), ("mag_16_19", 16, 19), ("mag_19_24", 19, 24), ("mag_ge24", 24, 31)):
        a = _sign(rng, _mag(rng, n, lo, hi))
        b = _sign(rng, _mag(rng, n, lo, hi))
        c = _sign(rng, _mag(rng, n, 0, hi))
        swap = rng.random(n) < 0.5
        both = pairs(a, b)
        one = pairs(np.where(swap, a, c), np.where(swap, c, a))
        out[name] = np.concatenate([both, one])
    # exactly +-2^24 in one or both components (disc_std_f32 takes [-2^24, 2^24) and leaves +2^24 to the fp64 form)
    e = np.array([1 << 24, -(1 << 24)], dtype=np.int64)
    o = _sign(rng, _mag(rng, n, 0, 31))
    k = rng.integers(0, 2, n)
    swap = rng.random(n) < 0.5
    exact = pairs(np.where(swap, e[k], o), np.where(swap, o, e[k]))
    grid = np.array([-(1 << 24) - 1, -(1 << 24), -(1 << 24) + 1, -1, 0, 1, (1 << 24) - 1, 1 << 24, (1 << 24) + 1])
    gr, gj = np.meshgrid(grid, grid, indexing="ij")
    out["mag_eq24"] = np.concatenate([exact, pairs(gr, gj)])
    # INT_MIN in either component
    o = _sign(rng, _mag(rng, n, 0, 31))
    o[:8] = [0, 1, -1, I32_MAX, -I32_MAX, 1 << 24, -(1 << 24), 1 << 30]
    swap = rng.random(n) < 0.5
    out["mag_int_min"] = _no_double_int_min(pairs(np.where(swap, INT_MIN, o), np.where(swap, o, INT_MIN)))
    return out


def octant_class(n=100_000, seed=SEED + 1):
    """|cr| = |cj| + d (d in -1..1) at every magnitude and sign; cr = 0; cj = 0 with either sign of cr"""
    rng = np.random.default_rng(seed)
    m = _mag(rng, n, 0, 31)
    d = rng.integers(-1, 2, n)
    a = np.clip(m + d, 0, I32_MAX)
    sr, sj = rng.random(n) < 0.5, rng.random(n) < 0.5
    diag = pairs(np.where(sr, -a, a), np.where(sj, -m, m))
    z = _sign(rng, _mag(rng, n // 4, 0, 31))
    axes = [pairs(np.zeros_like(z), z), pairs(z, np.zeros_like(z)), pairs([0, 0, INT_MIN, I32_MAX], [INT_MIN, 0, 0, 0])]
    return np.concatenate([diag] + axes)


def fast_classes(n=100_000, seed=SEED + 2):
    rng = np.random.default_rng(seed)
    out = {}
    # n = ||x| - |y|| at 2^19 - 1, 2^19, 2^19 + 1 (4096 n leaves int32 from 2^19 on), both branches and signs
    nn = (1 << 19) + rng.integers(-1, 2, n)
    small = _mag(rng, n, 0, 30)
    big = np.minimum(small + nn, I32_MAX)
    xb = rng.random(n) < 0.5                 # which component is the larger one
    ax, ay = np.where(xb, big, small), np.where(xb, small, big)
    out["fast_n_2e19"] = pairs(_sign(rng, ax), _sign(rng, ay))
    # divisors |x| + |y| that wrap to <= 0: |x| + |y| >= 2^31
    ax = _mag(rng, n, 30, 31)
    ay = np.clip((1 << 31) - ax + rng.integers(-2, 1 << 20, n), 0, I32_MAX)
    out["fast_den_wrap"] = _no_double_int_min(pairs(_sign(rng, ax), _sign(rng, ay)))
    # exact quotients: den = |x| + |y| = 4096 m (m even), n = T m, so 4096 n / den = T, and n +- 1 beside them
    m = 2 * rng.integers(1, 1 << 9, n)
    T = rng.integers(0, 4097, n)
    den, nv = 4096 * m, T * m + rng.integers(-1, 2, n) * 2
    ax, ay = (den + nv) // 2, (den - nv) // 2
    ok = (ax >= 0) & (ay >= 0)
    xb = rng.random(n) < 0.5
    out["fast_exact_q"] = pairs(_sign(rng, np.where(xb, ax, ay)[ok]), _sign(rng, np.where(xb, ay, ax)[ok]))
    return out


def lut_crash_quads():
    """int16 quads whose conjugate product has |cr| = 1 and cj = k 2^23 with k odd -- (cj << 8) is INT_MIN: with
    s = 2048 k' (k' odd), x[n] = (-(s -+ 1), s) after x[n-1] = (s +- 1, s) gives cr = 1, cj = 2 s^2, and the pair with
    x[n-1]'s real part and x[n]'s imaginary part negated gives cr = -1.  Every common rotation by a quarter turn and the
    conjugate of both samples keep |cr| = 1 and (cj << 8) = INT_MIN."""
    out = []
    for kk in range(1, 16, 2):
        s = 2048 * kk
        if s + 1 > 32767:
            break
        for e in (1, -1):
            base = [((-(s - e), s), (s + e, s)),          # cr = 1
                    ((-(s - e), -s), (-(s + e), s))]      # cr = -1
            for a, b in base:
                for rot in range(4):
                    for conj in (False, True):
                        aa, bb = a, b
                        for _ in range(rot):
                            aa, bb = (-aa[1], aa[0]), (-bb[1], bb[0])
                        if conj:
                            aa, bb = (aa[0], -aa[1]), (bb[0], -bb[1])
                        out.append((aa[0], aa[1], bb[0], bb[1]))
    return np.array(out, dtype=np.int32)


def lut_classes(n=100_000, seed=SEED + 3):
    rng = np.random.default_rng(seed)
    out = {}
    # |x| = |(cj << 8) / cr| at 131071 and 131072 (the table's end), with cj one either side of the boundary
    cr = _sign(rng, rng.integers(1, 1 << 14, n))
    k = rng.integers(131071, 131073, n)
    cj = (k * np.abs(cr)) // 256 + rng.integers(-1, 2, n)
    out["lut_end"] = pairs(cr, _sign(rng, cj))
    # cj around +-2^23, where cj << 8 wraps, against small and random divisors
    cj = _sign(rng, (1 << 23) + rng.integers(-3, 4, n))
    cr = np.where(rng.random(n) < 0.3, _sign(rng, rng.integers(1, 4, n)), _sign(rng, _mag(rng, n, 0, 31)))
    out["lut_shift_wrap"] = pairs(cr, cj)
    out["lut_crash"] = lut_crash_quads()
    return out


def int16_classes(n=400_000, seed=SEED + 4):
    rng = np.random.default_rng(seed)
    out = {"i16_random": rng.integers(-32768, 32768, (n, 4)).astype(np.int32)}
    corner = np.array([-32768, -32767, -1, 0, 1, 32766, 32767], dtype=np.int32)
    g = np.stack(np.meshgrid(corner, corner, corner, corner, indexing="ij"), axis=-1).reshape(-1, 4)
    out["i16_corners"] = np.ascontiguousarray(g)
    return out


def stream_class(n_prev=300, seed=SEED + 5):
    """every 8-bit-range sample (di, dq) in [-127, 128]^2 against n_prev previous samples, the extremes among them"""
    rng = np.random.default_rng(seed)
    ext = np.array([(-127, -127), (-127, 128), (128, -127), (128, 128), (0, 0), (1, 0), (0, -127), (128, 0)])
    prev = np.concatenate([ext, rng.integers(-127, 129, (n_prev - len(ext), 2))])
    v = np.arange(-127, 129, dtype=np.int32)
    di, dq = np.meshgrid(v, v, indexing="ij")
    cur = np.stack([di.reshape(-1), dq.reshape(-1)], axis=1)
    q = np.empty((len(prev), cur.shape[0], 4), dtype=np.int32)
    q[:, :, 0:2] = cur[None]
    q[:, :, 2:4] = prev[:, None, :]
    return q.reshape(-1, 4)


# an int16 pair whose std value V = 4934.99999999954... lies 4.6e-10 (< 2^-30) below an integer (mpmath, 50 digits)
NEAR_PAIR = (15954, 22135)


def crafted_capture(port, D, dec, chunk_complex=None):
    """A CS16 capture whose boxcar of length D (no passes) decimates to exactly dec (int [n][2], |component| <= 127 D):
    each decimated sample is D scaled samples in [-127, 127] that sum to it, every scaled value the least int16 the
    port's scale table maps to it.  chunk_complex: the rotation rotate16_90 applies per chunk (src/rtl_fm.c:309-327,
    restarting at every chunk) is undone, so that the boxcar sees dec; None for offset tuning (no rotation)."""
    dec = np.asarray(dec, dtype=np.int64).reshape(-1, 2)
    assert np.all(np.abs(dec) <= 127 * D)
    q, r = np.divmod(dec, D)                                          # r samples of q + 1, D - r of q
    j = np.arange(D)[None, :, None]
    s = (q[:, None, :] + (j < r[:, None, :])).reshape(-1, 2)          # scaled samples, in order
    if chunk_complex is not None:
        n = np.arange(s.shape[0]) % chunk_complex                     # in-chunk index: x[n] = s[n] * j^-n before rotation
        re, im = s[:, 0].copy(), s[:, 1].copy()
        ph = n & 3
        s[ph == 1] = np.stack([im, -re], axis=1)[ph == 1]
        s[ph == 2] = np.stack([-re, -im], axis=1)[ph == 2]
        s[ph == 3] = np.stack([-im, re], axis=1)[ph == 3]
    table = port.scale_table().astype(np.int64)                       # scaled value of int16 x at x + 32768
    raw = np.searchsorted(table, s.reshape(-1), side="left") - 32768
    assert np.array_equal(table[raw + 32768], s.reshape(-1))
    return raw.astype(np.int16)


def crash_sequence(D, n_dec, chunk_dec, seed=SEED + 6):
    """Decimated samples (int [n_dec][2]) that carry every lut_crash quad whose samples fit a boxcar of D (|v| <= 127 D)
    as two consecutive samples, x[n-1] then x[n], away from every chunk's first sample (where F8 takes the atan2 form),
    over a quiet random background.  Returns (samples, [(n, cj > 0) of each x[n]])."""
    rng = np.random.default_rng(seed)
    dec = rng.integers(-40, 41, (n_dec, 2))
    quads = [q for q in lut_crash_quads() if np.abs(q).max() <= 127 * D]
    placed, n = [], 5
    for a0, a1, b0, b1 in quads:
        while n % chunk_dec in (0, 1) or (n + 1) % chunk_dec == 0:
            n += 1
        assert n + 1 < n_dec
        dec[n - 1] = (b0, b1)
        dec[n] = (a0, a1)
        cj = int(a1) * int(b0) - int(a0) * int(b1)
        placed.append((n, cj > 0))
        n += 7
    return dec, placed


_NEAR = {"test": None, "met": False}


def port_met_near_integer():
    """Whether the port's chain runs of the running test so far evaluated polar_discriminant within 2^-30 of an integer
    (oracle.Port.std_near_count, read and reset, remembered until the next test: a test may compare several outputs
    against port runs it made beforehand).  Only then may a -A std result of the library differ from the port's:
    elsewhere CUDA's atan2 and glibc's, a few ulps apart at most, truncate to the same integer."""
    import oracle
    test = os.environ.get("PYTEST_CURRENT_TEST", "").split(" (")[0]
    if _NEAR["test"] != test:
        _NEAR.update(test=test, met=False)
    _NEAR["met"] = _NEAR["met"] or oracle.port().std_near_count() > 0
    return _NEAR["met"]


def edges():
    """the guard-band fixture: name -> int32 pair quads"""
    z = np.load(EDGES)
    return {name: pairs(z[name][:, 0], z[name][:, 1]) for name in sorted(z.files) if name.startswith("edge_")}


def random_classes():
    """every seeded class but small and stream: name -> quads"""
    c = {}
    c.update(magnitude_classes())
    c["octant"] = octant_class()
    c.update(fast_classes())
    c.update(lut_classes())
    c.update(int16_classes())
    return c


def conj(q):
    import oracle
    return oracle.conj_product(q)


def in_int16(q):
    return np.all((q >= -32768) & (q <= 32767), axis=1)


def domain(form, q):
    """the quads of q inside the form's domain (rxb200_fm_disc_device): ROWS |cr| + |cj| < 2^24 (the bound
    test_host_logic.py::test_row_discriminator_operands_fit_fp32 proves for the row front end), STREAM 8-bit-range
    samples, ALE and AM int16 samples; the others take every int32 quad"""
    if form == ROWS:
        cr, cj = conj(q)
        return q[np.abs(cr.astype(np.int64)) + np.abs(cj.astype(np.int64)) < (1 << 24)]
    if form == STREAM:
        return q[np.all((q >= -127) & (q <= 128), axis=1)]
    if form in (ALE, AM):
        return q[in_int16(q)]
    return q
