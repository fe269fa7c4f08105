"""Small run of the raster kernels for compute-sanitizer (memcheck).  The first window of a call reaches T - 1 samples
before the capture (the history) and the last ends at its last sample, so the capture sits exactly in its own
allocation; a call spans several frame groups (K = 4096, M = 1), and the DFT's last tiles hold frames and channels past
the ends (loads of zero rows, stores skipped).

    compute-sanitizer --tool memcheck python tests/sanitize_raster.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import fm_any_chunk as fac  # noqa: E402
import fm_raster as frs  # noqa: E402
from rx_tools_b200 import fm  # noqa: E402

differs = 0
for K, bins, dd, n in ((4096, [0, 1, 2048, 4095, 1], (1, np.array([3, -1, 2], np.int32), 18), 2101),
                       (3, [0, 1, 2, 2], (7, frs.near_limit(17, 0.05), 36), 1003),
                       (768, [408, 0, 360], (64, frs.fdd.lowpass(257, 12500 / 19.2e6), 30), 64 * 37 + 5)):
    x = np.random.default_rng(K).integers(-32768, 32768, size=2 * n).astype(np.int16)
    src = torch.from_numpy(x).cuda()                                            # exactly the capture
    out = torch.empty(len(bins) * 2 * (n // dd[0]), dtype=torch.int16, device="cuda")
    fm.raster_device(K, bins, (1 << 64) - 5, dd, src.data_ptr(), n, out.data_ptr())
    torch.cuda.synchronize()
    want, _ = frs.raster_model(x, K, bins, dd[1], dd[0], dd[2], phase=((1 << 64) - 5) % K)
    ok = out.cpu().numpy().tobytes() == want.tobytes()
    differs += not ok
    mx = fm.FmMix(fac.with_(fac.RAW, downsample=1, offset_tuning=1), ddc=dd, raster=(K, bins))
    got = np.concatenate([mx.process_read(x[:2 * (n // 2)]), mx.process_read(x[2 * (n // 2):])], axis=1)
    mx.close()
    print("raster K =", K, "M =", dd[0], "T =", dd[1].size, "exact" if ok else "DIFFERS", "handle", got.shape)
sys.exit(1 if differs else 0)
