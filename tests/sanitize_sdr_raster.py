"""Small run of the rx_sdr raster I/Q handles for compute-sanitizer (memcheck): every format, two device calls whose
captures and output rows sit exactly in their own allocations (rows packed with no gap, the second call not a multiple
of M), compared with the numpy model.  Exits nonzero when a result differs.

    compute-sanitizer --tool memcheck python tests/sanitize_sdr_raster.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import sdr_raster as sr  # noqa: E402
from rx_tools_b200 import sdr  # noqa: E402

differs = 0
for name in ("k3", "k4096_sat", "repeats_k64", "unit_k5"):
    x = sr.case_capture(name)
    want, M = sr.model(name, x)
    h = sr.handle(name)
    for fmt in sr.FORMATS:
        f = sdr.FORMATS[fmt]
        h.reset()
        parts = []
        cut = (x.size // 2 // 3) * 2 + 2
        for piece in (x[:cut], x[cut:]):
            src = torch.from_numpy(np.ascontiguousarray(piece)).cuda()         # exactly the capture
            n = h.decimated_len(piece.size)
            out = torch.empty(max(h.n_channels * n * 2, 1), dtype=torch.from_numpy(np.zeros(1, sdr.DTYPES[f])).dtype,
                              device="cuda")
            h.process_device(src.data_ptr(), piece.size, f, out.data_ptr(), h.n_channels * n, n)
            parts.append(out.cpu().numpy()[:h.n_channels * n * 2].reshape(h.n_channels, 2 * n))
        got = np.concatenate(parts, axis=1)
        ok = got.view(np.uint8).tobytes() == sr.convert(want, fmt).view(np.uint8).tobytes()
        differs += not ok
        print(name, fmt, "ok" if ok else "DIFFERS")
    h.close()
sys.exit(1 if differs else 0)
