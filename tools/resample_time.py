"""Time one second of device-resident capture through the rational resampler (rxb200_resample_*) for each named plan:
the device's stream at R_dev to the capture plan's rate R, with rxb200_plan_resample's L/N and J and the
rxb200_resample_lowpass prototype.  Per plan it reports, as the median over --repeats after a warm-up call:
  - kernel_ms: the handle's kernel time (CUDA events around resample_kernel) for one device call of the whole second;
  - device_ms: that device call, host clock around the call and a synchronise;
  - host_ms: the host call (rxb200_resample_process) from and to pinned host buffers, which stages in groups.
The card's name, power limit and maximum SM clock are printed first, then one JSON line per plan.

    python tools/resample_time.py [--repeats 5]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def board():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                     # the timing itself needs no nvidia-smi
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch
    import resample as rm
    from rx_tools_b200 import _lib, resample
    print("board:", board(), flush=True)
    for name, R_dev, R, span, _, _ in rm.NAMED:
        p = resample.plan_resample(R_dev, R, span)
        h = resample.lowpass(p.up, p.down, p.taps_per_phase)
        r = resample.Resampler(p.up, p.down, h, p.shift)
        x = torch.randint(-32768, 32768, (2 * R_dev,), dtype=torch.int16)
        d_x = x.cuda()
        n = r.out_len(2 * R_dev)
        d_y = torch.empty(2 * n, dtype=torch.int16, device="cuda")
        h_x = x.pin_memory()
        h_y = torch.empty(2 * n, dtype=torch.int16).pin_memory()
        kern, dev, host = [], [], []
        for k in range(args.repeats + 1):
            r.reset()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r.process_device(d_x.data_ptr(), 2 * R_dev, d_y.data_ptr(), n, sync=1)
            t1 = time.perf_counter()
            km = r.kernel_ms()
            r.reset()
            got = C.c_size_t(0)
            t2 = time.perf_counter()
            _lib.check(_lib.lib().rxb200_resample_process(r._h, h_x.data_ptr(), 2 * R_dev, h_y.data_ptr(), n,
                                                          C.byref(got)))
            t3 = time.perf_counter()
            if k:
                kern.append(km)
                dev.append(1e3 * (t1 - t0))
                host.append(1e3 * (t3 - t2))
        same = bool(torch.equal(d_y.cpu(), h_y))
        macs = 2.0 * n * p.taps_per_phase
        km = float(np.median(kern))
        print(json.dumps({"plan": name, "R_dev": R_dev, "R": R, "L": p.up, "N": p.down, "J": p.taps_per_phase,
                          "taps": p.up * p.taps_per_phase, "outputs": n, "kernel_ms": round(km, 3),
                          "device_ms": round(float(np.median(dev)), 3), "host_ms": round(float(np.median(host)), 3),
                          "gmac_per_s": round(macs / km / 1e6, 1), "host_equals_device": same}), flush=True)
        r.close()


if __name__ == "__main__":
    main()
