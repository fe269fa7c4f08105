"""Small run of device-rate bursts, for compute-sanitizer (memcheck): a power mixing handle with a burst device rate
takes one burst per tile through the device entry, each burst exactly in its own allocation, at 15/16 (a 2048-bin plan)
and 10/11 (int64 DDC sums), and is compared with the resampler handle followed by the capture-rate burst of a handle
without one.  Exits nonzero when a result differs.

    compute-sanitizer --tool memcheck python tests/sanitize_power_burst_rate.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import test_power_burst_rate_gpu as t  # noqa: E402

differs = 0
for name in ("fft_3.2M", "rms_wide_acc"):
    plan, win, tl, tiles, offs, dd, res = t._case(name)
    a, b = t._handles(plan, win, tl, offs, dd, res)
    rng = np.random.default_rng(5)
    for hb, he, _ in tiles:
        x = rng.integers(-20000, 20001, size=a.burst_in_len(1), dtype=np.int32).astype(np.int16)
        src = torch.from_numpy(x).cuda()                         # exactly the burst's device samples
        a.accumulate_burst_device(hb, he, src.data_ptr(), x.size, sync=True)
        b.accumulate_burst(hb, he, t._capture_burst(res, x))
    ga, gb = a.read(), b.read()
    ok = np.array_equal(ga[0], gb[0]) and np.array_equal(ga[1], gb[1])
    differs += not ok
    print("power burst", name, "ok" if ok else "DIFFERS")
    a.close()
    b.close()
sys.exit(1 if differs else 0)
