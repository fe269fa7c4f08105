"""Small rx_power run for compute-sanitizer (memcheck): one draw each of power_fft8_kernel<12, 512>, the generic kernel
with NB 0 and its sine and window tables in global memory, and power_big_decim with the global-memory FFT steps.  The
hop buffers come from device tensors of exactly the input's size, so a read past the last hop buffer would show.

    compute-sanitizer --tool memcheck python tests/sanitize_power.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import oracle  # noqa: E402
import power_paths as pp  # noqa: E402
from rx_tools_b200 import power  # noqa: E402

port = oracle.port()
rng = np.random.default_rng(1)
shapes = {
    "fft8<12,512>": pp.mkplan(12, 16384, n_hops=2),
    "generic<0> global tables": pp.mkplan(15, 65536, n_hops=1),
    "big_decim": pp.mkplan(10, 131072, ds=8, passes=3, fir=9, boxcar=0, n_hops=1),
}
for name, plan in shapes.items():
    x = pp.hop_input(rng, "noise", (2, plan.n_hops, plan.buf_len), False)
    win = power.window_table("hamming", 1 << plan.bin_e)
    want, want_smp = port.power_scan(pp.oracle_params(plan), win, x, 2, plan.n_hops)
    sc = power.PowerScanner(plan, win)
    buf = torch.from_numpy(x.reshape(-1)).cuda()            # a tensor of exactly the input's size
    torch.cuda.synchronize()
    sc.scanner_device(buf.data_ptr(), 2, sync=True)
    avg, smp = sc.read()
    path = sc.last_path()
    ok = np.array_equal(avg, want) and np.array_equal(smp, want_smp) and \
        path == pp.expected_path(plan, {}, 2, plan.n_hops, torch.cuda.get_device_properties(0).multi_processor_count)
    print(name, path["kernel"], "exact" if ok else "DIFFERS")
    sc.close()
