"""Times rx_power hops of one capture (rxb200_power_mix_*) on one second of capture for two sweeps, each planned the way
the rx_power shell plans capture mode:
* 88-108 MHz at 10 kHz bins: 8 hops, R = 20 Msps, M = 8, 257 taps;
* 24-60 MHz at 10 kHz bins cropped 28.5 %: 18 hops, R = 39 160 828 Hz, M = 14, 449 taps.

For each: power_ddc_kernel's device time (CUDA events, PowerMix.kernel_ms, summed over the call's groups of passes), the
member's last accumulate kernel (PowerMix.accumulate_ms), the whole device call on a device-resident capture (CUDA events
around accumulate_device), and the host call from a pinned capture buffer (host clock around the synchronised call).
The second of capture is cut to whole passes.  Prints the GPU's name and power limit, then one JSON line per sweep.

    python tools/power_mix_time.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import power_mix as pm  # noqa: E402
from rx_tools_b200 import power  # noqa: E402

SWEEPS = {"88-108M_10k": ("88M:108M:10k", 0.0), "24-60M_10k_crop28.5": ("24M:60M:10k", 0.285)}


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def run(name, reps):
    freq, crop = SWEEPS[name]
    plan = power.plan_range(freq, crop)
    _, offs, M, R, dd = pm.capture_plan(plan)
    pass16 = M * plan.buf_len
    n_pass = R * 2 // pass16                                  # one second of capture, whole passes
    x = pm.capture(n_pass * pass16 // 2, R, offs, 1, noise=1500)
    pin = torch.from_numpy(x).pin_memory()
    d_x = torch.from_numpy(x).cuda()
    mx = power.PowerMix(plan, R, offs, dd, "hamming")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    stream = torch.cuda.ExternalStream(mx.stream)
    dev_ms, ddc_ms, acc_ms, host_ms = [], [], [], []
    for r in range(reps + 1):
        mx.reset()
        e0.record(stream)
        mx.accumulate_device(d_x.data_ptr(), x.size, sync=False)
        e1.record(stream)
        e1.synchronize()
        if r:
            dev_ms.append(e0.elapsed_time(e1))
            ddc_ms.append(mx.kernel_ms())
            acc_ms.append(mx.accumulate_ms())
    want = mx.read()
    for r in range(reps + 1):
        mx.reset()
        t0 = time.perf_counter()
        power._lib.check(power._lib.lib().rxb200_power_mix_accumulate(mx._m, pin.data_ptr(), x.size))
        if r:
            host_ms.append((time.perf_counter() - t0) * 1e3)
    same = all(np.array_equal(a, b) for a, b in zip(mx.read(), want))
    mx.close()
    return dict(sweep=name, hops=plan.n_hops, capture_rate=R, decim=M, taps=int(dd[1].size), bin_e=plan.bin_e,
                passes=n_pass, capture_s=n_pass * pass16 / 2 / R, ddc_kernel_ms=min(ddc_ms),
                last_accumulate_kernel_ms=min(acc_ms), device_call_ms=min(dev_ms), host_call_ms=min(host_ms),
                host_equals_device=same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print("gpu:", gpu_info())
    for name in SWEEPS:
        print(json.dumps(run(name, a.reps)))


if __name__ == "__main__":
    main()
