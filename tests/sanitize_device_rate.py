"""Small run of the capture handles with a resampler attached, for compute-sanitizer (memcheck): an rx_sdr handle of each
kind and an rx_fm single-stage handle, at 21/25 (taps in shared memory) and 187/256 (taps through the caches), over two
device calls whose device samples sit exactly in their own allocations, compared with the composition (the resampler's
numpy model, then the same handle without one).  Exits nonzero when a result differs.

    compute-sanitizer --tool memcheck python tests/sanitize_device_rate.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import resample as rsm  # noqa: E402
import test_device_rate_gpu as t  # noqa: E402
from rx_tools_b200 import sdr  # noqa: E402

differs = 0
for plan in ("21/25", "187/256"):
    L, N, taps = t._plan(plan)
    x = t._stream(20_000, 1)
    y = rsm.resample_model(x, L, N, taps, 15)[0]
    cut = (x.size // 2 // 3) * 2 + 2
    for kind in ("single", "raster", "two_stage"):
        ref = t._sdr_mix(kind)
        want = ref.process(y)
        ref.close()
        h = t._sdr_mix(kind)
        h.set_device_rate(L, N, taps, 15)
        parts = []
        for piece in (x[:cut], x[cut:]):
            src = torch.from_numpy(np.ascontiguousarray(piece)).cuda()          # exactly the device samples
            n = h.decimated_len(piece.size)
            out = torch.empty(max(h.n_channels * n * 2, 1), dtype=torch.int16, device="cuda")
            h.process_device(src.data_ptr(), piece.size, sdr.OUT_CS16, out.data_ptr(), h.n_channels * n, n)
            parts.append(out.cpu().numpy()[:h.n_channels * n * 2].reshape(h.n_channels, 2 * n))
        h.close()
        ok = np.array_equal(np.concatenate(parts, axis=1), want[:, :sum(p.shape[1] for p in parts)])
        differs += not ok
        print("sdr", kind, plan, "ok" if ok else "DIFFERS")
    ref, h = t._fm_mix("single"), t._fm_mix("single")
    h.set_device_rate(L, N, taps, 15)
    n_cap = [rsm.out_count(0, cut // 2, L, N), rsm.out_count(cut // 2, x.size // 2 - cut // 2, L, N)]
    want = t._fm_reads(ref, t._split(y, n_cap), False)
    ok = np.array_equal(t._fm_reads(h, [x[:cut], x[cut:]], True), want)
    differs += not ok
    print("fm single", plan, "ok" if ok else "DIFFERS")
    ref.close()
    h.close()
sys.exit(1 if differs else 0)
