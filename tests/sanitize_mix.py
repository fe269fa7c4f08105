"""Small run of several rx_fm channels of one capture for compute-sanitizer (memcheck): an odd-length capture from a
tensor of exactly its size at a 4-byte offset, through the host and the device entry points of a mixing handle, and the
mixer alone -- the partial last unit of the capture is where a read past it would show.

    compute-sanitizer --tool memcheck python tests/sanitize_mix.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import fm_mix as fmx  # noqa: E402
from rx_tools_b200 import fm  # noqa: E402

for name in ("fm5a_lut_d100", "fm2b_f9", "fm_lut_d42_squelch"):
    p, rate, offs, x = fmx.case_input(name)
    n16 = 2 * 2003 if not p.downsample_passes else 2 * 2044
    x = x[:n16]
    mx = fm.FmMix(p, rate, offs)
    got = mx.process_read(x)
    mx.reset()
    buf = torch.from_numpy(np.concatenate([np.zeros(2, np.int16), x])).cuda()   # exactly the capture after 4 bytes
    cap = got.shape[1] + 8
    out = torch.zeros(len(offs) * cap, dtype=torch.int16, device="cuda")
    k = mx.process_read_device(buf.data_ptr() + 4, n16, out.data_ptr(), cap, sync=True)
    ok = np.array_equal(out.view(len(offs), cap)[:, :k].cpu().numpy(), got)
    dst = torch.zeros(n16, dtype=torch.int16, device="cuda")
    fm.mix_device(rate, offs[-1], 5, buf.data_ptr() + 4, n16 // 2, dst.data_ptr())
    torch.cuda.synchronize()
    ok = ok and np.array_equal(dst.cpu().numpy(), fmx.mix_model(x, fm.mix_table(rate, offs[-1]), 5))
    print(name, "exact" if ok else "DIFFERS")
    mx.close()
