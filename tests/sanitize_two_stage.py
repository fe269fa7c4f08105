"""Small run of the two-stage kernels for compute-sanitizer (memcheck).  The capture sits exactly in its own
allocation; the first coarse window reaches T1 - 1 samples before it (the history) and the fine stage reads T2 - 1
coarse samples before each group's row; one call spans several coarse groups (K = 4096, thousands of bins), and the
DFT's last tiles hold frames and bins past the ends (loads of zero rows, stores skipped).

    compute-sanitizer --tool memcheck python tests/sanitize_two_stage.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import fm_any_chunk as fac  # noqa: E402
import fm_two_stage as fts  # noqa: E402
from rx_tools_b200 import fm  # noqa: E402

differs = 0
for rate, K, offs, coarse, fine, n in (
        (4_096_000, 4096, [1000 * k - 2_000_000 + 7 for k in range(3000)], (1, np.array([3, -1, 2], np.int32), 18),
         (2, np.array([1, 2, 1], np.int32), 2), 2101),
        (1_008_000, 3, [0, 1, 335_999, -170_001], (3, fts.frs.near_limit(17, 0.05), 36),
         (2, fts.fdd.lowpass(9, 0.2), 15), 1003),
        (19_200_000, 32, [-9_000_001, 123_457, 5_000_000, 5_000_001], fts.C19, fts.F19, 64 * 37 + 5)):
    x = np.random.default_rng(K).integers(-32768, 32768, size=2 * n).astype(np.int16)
    src = torch.from_numpy(x).cuda()                                            # exactly the capture
    M = coarse[0] * fine[0]
    out = torch.empty(len(offs) * 2 * (n // M), dtype=torch.int16, device="cuda")
    fm.two_stage_device(rate, K, offs, (1 << 64) - 5, coarse, fine, src.data_ptr(), n, out.data_ptr())
    torch.cuda.synchronize()
    want = fts.two_stage_model(x, rate, K, offs, coarse, fine, (1 << 64) - 5)
    ok = out.cpu().numpy().tobytes() == want.tobytes()
    differs += not ok
    mx = fm.FmMix(fac.with_(fac.RAW, downsample=1, offset_tuning=1), rate, offs, two_stage=(K, coarse, fine))
    got = np.concatenate([mx.process_read(x[:2 * (n // 2)]), mx.process_read(x[2 * (n // 2):])], axis=1)
    mx.close()
    print("two-stage K =", K, "M =", M, "exact" if ok else "DIFFERS", "handle", got.shape)
sys.exit(1 if differs else 0)
