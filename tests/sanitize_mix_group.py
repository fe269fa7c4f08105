"""Small run of a mixing group for compute-sanitizer (memcheck): odd-length captures through groups of 2 and 3 members on
ordinal 0 (the second with an empty member), by process_read and by chunk calls, then a reset and the reads again --
each member's staging copies, mixer and chain, and the 2-D copies of its PCM rows into the caller's buffer, are where an
access past a buffer would show.

    compute-sanitizer --tool memcheck python tests/sanitize_mix_group.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import fm_mix as fmx  # noqa: E402
from rx_tools_b200 import fm  # noqa: E402

for name, devices in (("fm5a_lut_d100", [0, 0]), ("fm2b_f9", [0, 0, 0]), ("fm_lut_d42_squelch", [0, 0, 0])):
    p, rate, offs, cap = fmx.case_input(name)
    n16 = 2 * 2003 if not p.downsample_passes else 2 * 2044
    x = cap[:n16]
    g = fm.FmMixGroup(p, rate, offs, devices)
    mx = fm.FmMix(p, rate, offs)
    ok = np.array_equal(g.process_read(x), mx.process_read(x))
    # chunk calls: odd chunks and a short last one without passes, the passes' granule with them
    y, chunk = (cap[:2 * (3 * 1001 + 457)], 2 * 1001) if not p.downsample_passes else (cap[:3 * 2048], 2048)
    ok = ok and np.array_equal(g.full_demod(y, chunk), mx.full_demod(y, chunk))
    g.reset()
    mx.reset()
    ok = ok and np.array_equal(g.process_read(x), mx.process_read(x))
    print(name, "exact" if ok else "DIFFERS")
    g.close()
    mx.close()
