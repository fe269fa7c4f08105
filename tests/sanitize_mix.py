"""Small run of several rx_fm channels of one capture for compute-sanitizer (memcheck): an odd-length capture from a
tensor of exactly its size at a 4-byte offset, through the host and the device entry points of a mixing handle, and the
mixer alone -- the partial last unit of the capture is where a read past it would show.  Then a decimating handle on
the same kind of capture: fm_ddc_kernel's staged windows and its reads of the history, and the history carry, with a
read shorter than M (no output) and one shorter than T - 1 (the carry keeps part of the old history).

    compute-sanitizer --tool memcheck python tests/sanitize_mix.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import fm_ddc as fdd  # noqa: E402
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

p, rate, offs, ddc, cap, _ = fdd.case_input("am_m100")
M, T = ddc[0], ddc[1].size
lens = [2 * 2003, 2 * 37, 2 * 251]                    # odd complex counts; 37 < M, and 37, 251 < T - 1
assert 37 < M and 251 < T - 1
x = cap[:sum(lens)]
host, dev = fm.FmMix(p, rate, offs, ddc=ddc), fm.FmMix(p, rate, offs, ddc=ddc)
buf = torch.from_numpy(np.concatenate([np.zeros(2, np.int16), x])).cuda()   # exactly the capture after 4 bytes
stride = 2 * sum(lens) // (2 * M) + 8
out = torch.zeros(len(offs) * stride, dtype=torch.int16, device="cuda")
ok, pos = True, 0
for n16 in lens:
    want = host.process_read(x[pos:pos + n16])
    k = dev.process_read_device(buf.data_ptr() + 4 + 2 * pos, n16, out.data_ptr(), stride, sync=True)
    ok = ok and np.array_equal(out.view(len(offs), stride)[:, :k].cpu().numpy(), want)
    pos += n16
host.reset()
dev.reset()
chunk = 2 * M * 4                                     # the last chunk of the first read is 3 samples
want = host.full_demod(x[:lens[0]], chunk)
k = dev.process_device(buf.data_ptr() + 4, lens[0], chunk, out.data_ptr(), stride, sync=True)
ok = ok and np.array_equal(out.view(len(offs), stride)[:, :k].cpu().numpy(), want)
print("am_m100 ddc", "exact" if ok else "DIFFERS")
host.close()
dev.close()
