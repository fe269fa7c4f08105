"""Small run of bursts (rxb200_power_mix_accumulate_burst*) for compute-sanitizer (memcheck).  A burst's history is read
from its own lead, so the first staged window starts at the burst's first sample: an off-by-one there reads before the
buffer.  Each burst sits at the very start of its own allocation (and the device one is exactly the burst, so the last
window ends at its last sample), with hops on two grid rows of power_ddc_kernel starting at a hop other than 0, a lead
that is a whole number of M past T - 1 and one that is exactly T - 1.

    compute-sanitizer --tool memcheck python tests/sanitize_power_tiles.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import power_mix as pm  # noqa: E402
import power_paths  # noqa: E402
import power_tiles as ptl  # noqa: E402
from rx_tools_b200 import power  # noqa: E402

plan = power_paths.mkplan(4, 64, n_hops=300)
R = 1_000_000
offs = [(i * 3877) % 999_999 - 499_999 for i in range(plan.n_hops)]
for dd in ((3, power.ddc_lowpass(3, 97, 15), 15), (4, power.ddc_lowpass(4, 9, 15), 15)):
    host, dev = power.PowerMix(plan, R, offs, dd), power.PowerMix(plan, R, offs, dd)
    G = host.lead
    assert G == ptl.lead(dd[0], dd[1].size)
    x = pm.capture(host.burst_int16(2) // 2, R, offs, 5)
    host.accumulate_burst(3, 290, x)
    buf = torch.from_numpy(x).cuda()                                         # exactly the burst
    dev.accumulate_burst_device(3, 290, buf.data_ptr(), x.size, sync=True)
    ok = all(np.array_equal(a, b) for a, b in zip(host.read(), dev.read()))
    print("burst G =", G, "T =", dd[1].size, "exact" if ok else "DIFFERS")
    host.close()
    dev.close()
