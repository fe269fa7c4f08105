"""Small run of rx_power hops of one capture for compute-sanitizer (memcheck): a power mixing handle with hops on two
grid rows of power_ddc_kernel, fed from a tensor of exactly one pass at a 4-byte offset (the last staged window ends at
its last sample) and from the host; then the stateless entry with n < M and an odd sample count.

    compute-sanitizer --tool memcheck python tests/sanitize_power_mix.py
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
from rx_tools_b200 import power  # noqa: E402

plan = power_paths.mkplan(4, 64, n_hops=258)
R = 1_000_000
offs = [(i * 3877) % 999_999 - 499_999 for i in range(plan.n_hops)]
dd = (3, power.ddc_lowpass(3, 97, 15), 15)
pas = dd[0] * plan.buf_len
x = pm.capture(2 * pas // 2, R, offs, 5)
host, dev = power.PowerMix(plan, R, offs, dd), power.PowerMix(plan, R, offs, dd)
host.accumulate(x)
buf = torch.from_numpy(np.concatenate([np.zeros(2, np.int16), x])).cuda()     # exactly the capture after 4 bytes
dev.accumulate_device(buf.data_ptr() + 4, pas, sync=False)
dev.accumulate_device(buf.data_ptr() + 4 + 2 * pas, pas, sync=True)
ok = all(np.array_equal(a, b) for a, b in zip(host.read(), dev.read()))
print("power mix", "exact" if ok else "DIFFERS")
host.close()
dev.close()

src = torch.from_numpy(x[:2 * 101]).cuda()
dst = torch.zeros(2 * 40, dtype=torch.int16, device="cuda")
for n in (2, 101):
    power.power_ddc_device(R, offs[7], 9, dd, src.data_ptr(), n, dst.data_ptr())
    torch.cuda.synchronize()
    want, _ = pm.ddc(x[:2 * n], R, offs[7], dd, 9)
    ok = np.array_equal(dst[:want.size].cpu().numpy(), want)
    print("power ddc n =", n, "exact" if ok else "DIFFERS")
