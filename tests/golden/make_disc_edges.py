"""Makes golden/disc_edges.npz: conjugate-product pairs (cr, cj) whose exact polar_discriminant value
V = atan2(cj, cr) / 3.14159 * 2^14 (src/rtl_fm.c:476-483, 3.14159 being the C double) lies at a chosen distance
d = |V - round(V)| from an integer, on both sides of it.  They sit on the guard bands of the device forms
(csrc/fm_kernels.cu): disc_std_f32 sends d < 1.5e-3 to the fp64 form (operands below 2^24), disc_std_lean sends
d < 1e-5 to libm's atan2.

  edge_f32_in / edge_f32_out      operands < 2^24, d in [1.3e-3, 1.5e-3) / [1.5e-3, 1.7e-3)
  edge_f64_in / edge_f64_out      largest operand >= 2^24, d in [0.8e-5, 1e-5) / [1e-5, 1.2e-5)
  edge_fp64s_in / edge_fp64s_out  operands < 2^24 with the same 1e-5 bands (disc_std_lean through RXB200_DISC_STD_FP64)
  edge_fp64_mid_lo / _hi          d in [1e-8, 1e-7), operands < 2^24 / largest >= 2^24: decided by the fp64 form's own
                                  value (its error is < 4e-9 output units), not by libm
  edge_libm_lo / edge_libm_hi     d < 1e-9 (the libm fallback), operands < 2^24 / largest >= 2^24
Each array is int32 [N][2] of (cr, cj).  A candidate is cr = round(R cos t), cj = round(R sin t) for a random radius R
in the class and t = (k + s delta) * 3.14159 / 2^14 over random k (every octant) and side s; numpy's float64 picks the
candidates whose d is near the band (within 1e-8) and mpmath at 50 digits decides.  The file is written with fixed zip
timestamps, so running this again gives the same bytes:  python tests/golden/make_disc_edges.py
"""
import io
import os
import zipfile

import mpmath
import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "disc_edges.npz")
N = 256
K = 16384.0 / 3.14159
BUCKETS = [  # name, radius bits (lo, hi), d band, operands below 2^24
    ("edge_f32_in", (10, 24), (1.3e-3, 1.5e-3), True),
    ("edge_f32_out", (10, 24), (1.5e-3, 1.7e-3), True),
    ("edge_f64_in", (24, 31), (0.8e-5, 1e-5), False),
    ("edge_f64_out", (24, 31), (1e-5, 1.2e-5), False),
    ("edge_fp64s_in", (14, 24), (0.8e-5, 1e-5), True),
    ("edge_fp64s_out", (14, 24), (1e-5, 1.2e-5), True),
    ("edge_fp64_mid_lo", (14, 24), (1e-8, 1e-7), True),
    ("edge_fp64_mid_hi", (24, 31), (1e-8, 1e-7), False),
    ("edge_libm_lo", (20, 24), (0.0, 1e-9), True),
    ("edge_libm_hi", (24, 31), (0.0, 1e-9), False),
]


def exact_distance(cr, cj):
    """d = |V - round(V)| and V itself, at 50 digits"""
    with mpmath.workdps(50):
        v = mpmath.atan2(int(cj), int(cr)) / mpmath.mpf(3.14159) * 16384
        return abs(v - mpmath.nint(v)), v


def bucket(rng, rbits, band, below):
    lo, hi = band
    got, seen = [], set()
    while len(got) < N:
        m = 1 << 16
        R = np.exp2(rng.uniform(rbits[0], rbits[1], m))
        k = rng.integers(-16384, 16385, m).astype(np.float64)
        s = np.where(rng.random(m) < 0.5, -1.0, 1.0)
        delta = rng.uniform(lo, hi, m)
        t = (k + s * delta) / K
        t = np.where(t > np.pi, t - 2 * np.pi, np.where(t <= -np.pi, t + 2 * np.pi, t))
        cr, cj = np.rint(R * np.cos(t)), np.rint(R * np.sin(t))
        big = np.maximum(np.abs(cr), np.abs(cj))
        ok = (big < (1 << 24)) if below else ((big >= (1 << 24)) & (big < (1 << 31)))
        v = np.arctan2(cj, cr) * K
        d = np.abs(v - np.rint(v))
        ok &= (d >= lo - 1e-8) & (d < hi + 1e-8) & ~((cj == 0) & (cr >= 0))
        for a, b in zip(cr[ok].astype(np.int64), cj[ok].astype(np.int64)):
            if (a, b) in seen:
                continue
            de, _ = exact_distance(a, b)
            if lo <= de < hi:
                seen.add((a, b))
                got.append((a, b))
                if len(got) == N:
                    break
    return np.array(got, dtype=np.int32)


def write_npz(path, arrays):
    with zipfile.ZipFile(path, "w", zipfile.ZIP_STORED) as z:
        for name in sorted(arrays):
            b = io.BytesIO()
            np.lib.format.write_array(b, np.ascontiguousarray(arrays[name]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), b.getvalue())


def main():
    rng = np.random.default_rng(20240601)
    arrays = {name: bucket(rng, rbits, band, below) for name, rbits, band, below in BUCKETS}
    write_npz(OUT, arrays)
    print("wrote", OUT, {k: v.shape for k, v in arrays.items()})


if __name__ == "__main__":
    main()
