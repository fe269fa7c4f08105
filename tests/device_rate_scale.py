"""The launch rule of resample.cu and the group sizes of the capture handles that carry a resampler, restated, so that
a test can say which regime it reaches and assert it, and an exact model of the resampler that evaluates single
outputs, for streams too long for the full numpy model (tests/resample.py).

launch is resample_launch line for line: the call's outputs, the first output's q and phase, the outputs per CTA U and
the term that sets it ("share": two CTAs per SM, "span": RS_SPAN staged samples, "max_u": RS_MAX_U), the staging room,
whether the taps go to shared memory, the shared memory and CTA count, and, over every CTA of the call, the largest v
= pa + u (N mod L) the kernel's multiply-high sees and the most samples a CTA stages.

sparse_outputs evaluates the rule of include/rxb200.h output by output, t = m N, q = floor(t / L), p = t mod L,
A = sum_j h[p + j L] x[q - j], with t, q and p in Python integers and the dot product exact in int64; it shares nothing
with the kernel's CTA split.  check_indices picks which outputs of a call it evaluates.

sdr_host_group is sdr_mix.cu's host_group, power_groups power_mix.cu's pass groups; the raster and two-stage groups
are channelizer_scale.raster_plan and two_stage_plan.
"""
import numpy as np

import resample as rsm

RS_THREADS = 256
RS_SPAN = 8192                   # device samples a CTA stages at most
RS_MAX_U = 512                   # outputs per CTA at most
RS_SMEM_TAPS = 12288             # taps held in shared memory at most
H100_SMEM_OPTIN = 227 * 1024     # the H100's opt-in dynamic shared memory per block
SDR_SCRATCH_BYTES = 64 << 20     # RXB200_SDR_MIX_SCRATCH_BYTES
POWER_SCRATCH_BYTES = 64 << 20   # RXB200_POWER_MIX_SCRATCH_BYTES
RESAMPLE_SCRATCH_BYTES = 64 << 20


def launch(L, N, J, n0, c, n_sm, ctas=True):
    """resample_launch for a call over device samples [n0, n0 + c): a dict of its plan, or None for a call with no
    output.  ctas: also walk every CTA for the worst v and staged count (vectorised; off for very long calls)."""
    m0 = rsm.ceil_div(n0 * L, N)
    n_out = rsm.ceil_div((n0 + c) * L, N) - m0
    if n_out == 0:
        return None
    t0 = m0 * N
    q0, p0 = t0 // L - n0, t0 % L
    nq, nr = N // L, N % L
    span_u = (RS_SPAN - J - 1) * L // N + 1
    bound = min(RS_MAX_U, span_u)
    share = (n_out + 2 * n_sm - 1) // (2 * n_sm)
    U = max(1, min(bound, share))
    which = "share" if share < bound else ("max_u" if RS_MAX_U <= span_u else "span")
    room = (L - 1 + (U - 1) * N) // L + J
    smem_taps = L * J <= RS_SMEM_TAPS
    smem = ((room + 3) & ~3) * 4 + (L * J * 4 if smem_taps else 0)
    out = dict(n_out=n_out, q0=q0, p0=p0, nq=nq, nr=nr, U=U, which=which, room=room, smem_taps=smem_taps, smem=smem,
               ctas=(n_out + U - 1) // U, v_bound=(L - 1) + (U - 1) * nr)
    if ctas:
        i0 = np.arange(out["ctas"], dtype=np.int64) * U
        Ub = np.minimum(U, n_out - i0)
        pa = (p0 + (i0 % L) * nr) % L                  # (p0 + i0 nr) mod L without int64 overflow
        v = pa + (Ub - 1) * nr
        staged = (Ub - 1) * nq + v // L + J
        out["worst_v"] = int(v.max())
        out["worst_staged"] = int(staged.max())
    return out


def umulhi_corrections(v, L):
    """How many +1 steps take __umulhi(v, floor((2^32 - 1) / L)) to floor(v / L) (negative: the estimate is above)."""
    v = np.asarray(v, dtype=np.uint64)
    Lm = np.uint64((2**32 - 1) // L)
    d = (v * Lm) >> np.uint64(32)                       # v < 2^32 and Lm < 2^32: the product fits 64 bits
    return (v // np.uint64(L)).astype(np.int64) - d.astype(np.int64)


def sparse_outputs(ext, H, L, N, taps, S, n0, idx):
    """Outputs idx (indices within the call over device samples [n0, n0 + c)) of the rule, as int16 [len(idx)][2].
    ext: int16 [2(H + c)], the H samples before n0 (zeros from create or reset, else the stream's own), then the call's
    c samples; H >= J - 1."""
    x = np.asarray(ext, dtype=np.int16).reshape(-1, 2).astype(np.int64)
    h = np.asarray(taps, dtype=np.int64).reshape(-1)
    J = h.size // L
    assert H >= J - 1
    m0 = rsm.ceil_div(n0 * L, N)
    jj = np.arange(J, dtype=np.int64)
    out = np.empty((len(idx), 2), np.int64)
    blk = max(1, (1 << 20) // J)
    idx = [int(i) for i in idx]
    for a in range(0, len(idx), blk):
        q, p = [], []
        for i in idx[a:a + blk]:
            t = (m0 + i) * N                                 # Python integers: n0 may be near 2^64
            q.append(t // L - n0 + H)                        # ext index of x[q]
            p.append(t % L)
        q, p = np.array(q, np.int64), np.array(p, np.int64)
        xi = x[q[:, None] - jj[None, :]]
        hp = h[p[:, None] + jj[None, :] * L]
        out[a:a + q.size] = (hp[..., None] * xi).sum(1)
    y = out if S == 0 else (out + (1 << (S - 1))) >> S
    return np.clip(y, -32768, 32767).astype(np.int16)


def check_indices(n_out, U, J, edges=(), seed=0, every=64, lead=0):
    """The outputs of a call to check with the sparse model: every CTA's first and last, every output within J of the
    call's ends and of each edge (output indices where a group or read starts), and a seeded 1/every of the rest.
    lead: outputs the launch makes ahead of the call's first (a launch that starts earlier, for context), so that its
    CTAs start at k U - lead."""
    s = set()
    for b in range(-lead, n_out, U):
        if b + U > 0:
            s.add(max(0, b))
            s.add(min(n_out, b + U) - 1)
    for e in list(edges) + [0, n_out]:
        s.update(range(max(0, e - J), min(n_out, e + J)))
    rng = np.random.default_rng(seed)
    s.update(int(v) for v in rng.integers(0, n_out, size=max(1, n_out // every)))
    return sorted(s)


def sdr_host_group(L, N, M, n_ch, elem_bytes):
    """host_group of sdr_mix.cu with a resampler: (device samples per group, outputs per channel per group bound)."""
    rows = n_ch * elem_bytes
    S = SDR_SCRATCH_BYTES
    g = max(1, S * N * M // (4 * N * M + (4 * M + rows) * L))
    return g, rsm.ceil_div(g * L, N) // M + 1


def host_groups_crossed(c, g):
    """Groups a host call of c device samples runs in."""
    return rsm.ceil_div(c, g)


def power_groups(n_pass, n_hops, buf_len):
    """power_mix_call's pass groups for a call of n_pass passes: (passes per group, groups)."""
    per_pass = n_hops * buf_len * 2
    group = max(1, min(n_pass, POWER_SCRATCH_BYTES // per_pass))
    return group, rsm.ceil_div(n_pass, group)


def in_len_brute(L, N, n0, n_out):
    """The least c with out_count(n0, c) >= n_out, by search."""
    c = 0
    while rsm.out_count(n0, c, L, N) < n_out:
        c += 1
    return c


def periodic(base, start, n):
    """Samples [start, start + n) of the stream that repeats base (int16 [2B]) forever, as int16 [2n]."""
    B = base.size // 2
    k = np.arange(start % B, start % B + n) % B
    return base.reshape(-1, 2)[k].reshape(-1)
