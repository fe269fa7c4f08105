"""Small run of every capture handle kind in each narrow input format, for compute-sanitizer (memcheck): rx_fm single
stage, raster and two stages, rx_sdr single stage, rx_power stream calls and bursts, each fed CS8, CU8 and CS12 through
the device entry from a buffer exactly the call's bytes long at an odd address, and compared with the same handle on
the widened CS16 stream.  Exits nonzero when a result differs.

    compute-sanitizer --tool memcheck python tests/sanitize_device_format.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

from rx_tools_b200 import power  # noqa: E402
import device_format as df  # noqa: E402
import power_mix as pm  # noqa: E402
import test_device_format_gpu as t  # noqa: E402


def exact(b, off=1):
    """b's bytes on the device at byte offset off of an allocation that ends where they end."""
    d = torch.zeros(b.size + off, dtype=torch.uint8, device="cuda")
    d[off:] = torch.from_numpy(np.ascontiguousarray(b)).cuda()
    return d, d.data_ptr() + off


differs = 0
for fmt in df.FORMATS:
    b = df.narrow_stream(9_001, fmt, 1)
    for kind in ("single", "raster", "two_stage"):
        a, ref = t._fm_mix(kind), t._fm_mix(kind)
        a.set_input_format(fmt)
        cap = a.max_output(2 * 9_001, 2 * 9_001) + 8
        d, p = exact(b)
        d_out = torch.zeros((a.n_channels, cap), dtype=torch.int16, device="cuda")
        n = a.process_read_device(p, 2 * 9_001, d_out.data_ptr(), cap, sync=True)
        ok = np.array_equal(d_out[:, :n].cpu().numpy(), ref.process_read(df.widen(b, fmt)))
        differs += not ok
        print("fm_mix", kind, fmt, "ok" if ok else "DIFFERS")
        a.close()
        ref.close()
    a, ref = t._sdr_mix("single"), t._sdr_mix("single")
    a.set_input_format(fmt)
    d, p = exact(b)
    nd = a.decimated_len(2 * 9_001)
    d_out = torch.zeros(a.n_channels * nd * 4, dtype=torch.uint8, device="cuda")
    a.process_device(p, 2 * 9_001, 4, d_out.data_ptr(), a.n_channels * nd, nd)
    got = d_out.cpu().numpy().view(np.int16).reshape(a.n_channels, -1)
    ok = np.array_equal(got, ref.process(df.widen(b, fmt)))
    differs += not ok
    print("sdr_mix", fmt, "ok" if ok else "DIFFERS")
    a.close()
    ref.close()
    pl, win, Rp, offs, dd = pm.shape("fm_band")
    a, ref = power.PowerMix(pl, Rp, offs, dd, win), power.PowerMix(pl, Rp, offs, dd, win)
    a.set_input_format(fmt)
    x = df.narrow_stream(dd[0] * pl.buf_len // 2, fmt, 2)
    d, p = exact(x)
    a.accumulate_device(p, dd[0] * pl.buf_len, sync=True)
    ref.accumulate(df.widen(x, fmt))
    bb = df.narrow_stream(a.burst_int16(1) // 2, fmt, 3)
    d, p = exact(bb)
    a.accumulate_burst_device(0, 2, p, a.burst_int16(1), sync=True)
    ref.accumulate_burst(0, 2, df.widen(bb, fmt))
    ga, gb = a.read(), ref.read()
    ok = all(np.array_equal(u, v) for u, v in zip(ga, gb))
    differs += not ok
    print("power_mix", fmt, "ok" if ok else "DIFFERS")
    a.close()
    ref.close()
sys.exit(1 if differs else 0)
