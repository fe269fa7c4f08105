"""The resampler at the edges of its launch rule, for compute-sanitizer (memcheck): J L = 2^22 at U = 512 outputs per CTA
(J = 1 at L = 4 194 301 with v within 2^23 of 2^31, where a wrong multiply-high quotient would index outside the staged
samples, and J = 1024 with the largest staging room), both sides of the shared-memory taps flip and both sides of the
accumulator flip.  Each call is long enough for at least two waves of CTAs at that U, runs through
rxb200_resample_device from a source and into an output that sit exactly in their own allocations, and is compared with
the numpy model (the sparse model for J = 1024) after its regime is asserted.  Exits nonzero when a regime or a result
differs.

    compute-sanitizer --tool memcheck python tests/sanitize_device_rate_scale.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import device_rate_scale as drs  # noqa: E402
import mix_scale as ms  # noqa: E402
import resample as rsm  # noqa: E402
import test_device_rate_scale_gpu as t  # noqa: E402
from rx_tools_b200 import resample as rs  # noqa: E402

n_sm = ms.device_sms()
differs = 0
for name in ("top_J1_N=L-1", "top_J1024", "smem_12288", "gmem_12289", "acc_15_65535", "acc_15_65537"):
    L, N, J, kind, (U, which), smem_taps, wide = t.EDGES[name]
    h, S = t._edge_taps(kind, L, J, np.random.default_rng(5))
    c = t._edge_len(L, N, U, n_sm)
    a = drs.launch(L, N, J, 0, c, n_sm)
    regime = ((a["U"], a["which"]) == (U, which) and a["smem_taps"] == smem_taps and rsm.wide(h, L, S) == wide
              and a["ctas"] >= 4 * n_sm and a["worst_v"] < 1 << 31 and a["worst_staged"] <= a["room"] <= drs.RS_SPAN
              and (not name.startswith("top_J1_") or a["worst_v"] > (1 << 31) - (1 << 23)))
    x = t._stream(c, 7)
    if kind.startswith("acc"):
        x.reshape(-1, 2)[c // 3:] = -32768                             # every sum at its bound
    src = torch.from_numpy(x).cuda()                                   # exactly the call's samples
    n = a["n_out"]
    dst = torch.empty(2 * n, dtype=torch.int16, device="cuda")         # exactly the call's outputs
    rs.resample_device(L, N, h, S, 0, src.data_ptr(), c, dst.data_ptr())
    torch.cuda.synchronize()
    got = dst.cpu().numpy()
    ext = np.concatenate([np.zeros(2 * J, np.int16), x])
    try:
        t._check(got, ext, J, L, N, h, S, 0, a, 0)
        ok = True
    except AssertionError:
        ok = False
    differs += not (ok and regime)
    print(name, "U", a["U"], a["which"], "worst v", a["worst_v"], "outputs", n,
          "ok" if ok and regime else ("REGIME DIFFERS" if not regime else "DIFFERS"))
sys.exit(1 if differs else 0)
