"""Small any-length rx_fm run for compute-sanitizer (memcheck): several channels of an odd length, one call through the
host entry point and one through the device entry point from a tensor of exactly the input's size -- the partial
last block of the last channel is where a read past the input would show.

    compute-sanitizer --tool memcheck python tests/sanitize_any_chunk.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import fm_any_chunk as fac  # noqa: E402
import oracle  # noqa: E402
from rx_tools_b200 import fm  # noqa: E402

port = oracle.port()
n_ch, n, c = 3, 2 * 1001 + 5, 1001
for name in ("fm_lut_d100", "fm_fast_d1_deemph181", "fm_lut_d42_squelch", "raw"):
    p = fac.shapes()[name]
    x = np.stack([fac.signal(n, 30 + k) for k in range(n_ch)])
    d = fm.FmDemod(p, n_channels=n_ch)
    got = d.full_demod(x, 2 * c)
    ok = all(np.array_equal(got[k], port.fm_run(p, x[k], 2 * c)) for k in range(n_ch))
    d.reset()
    buf = torch.from_numpy(x.reshape(-1)).cuda()            # a tensor of exactly the input's size
    cap = d.max_output(2 * n, 2 * c) + 8
    out = torch.zeros(n_ch * cap, dtype=torch.int16, device="cuda")
    k = d.process_device(buf.data_ptr(), 2 * n, 2 * c, out.data_ptr(), cap, sync=True)
    ok = ok and np.array_equal(out.view(n_ch, cap)[:, :k].cpu().numpy(), got)
    print(name, "exact" if ok else "DIFFERS")
    d.close()
