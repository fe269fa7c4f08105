"""Times wide rx_power sweeps in tiles (rxb200_power_plan_tiles + rxb200_power_mix_accumulate_burst_device) for two
plans, each tiled the way the rx_power shell's tile mode tiles it:
* 24 MHz - 1.766 GHz at 100 kHz bins, captures of at most 61.44 Msps;
* 400-500 MHz at 10 kHz bins, captures of at most 20 Msps.

For each: the tiles against the hops (retunes per sweep in tile mode against hop mode), and the device time of one
sweep's bursts (one burst per tile of the lead plus one pass, device-resident): power_ddc_kernel's time
(PowerMix.kernel_ms) and the member's accumulate kernel (PowerMix.accumulate_ms), each summed over the tiles, and the
whole sweep's bursts between two CUDA events with no synchronisation in between.  Retune and settling time belong to
the radio and are not measured.  Prints the GPU's name, power limit and SM clock, then one JSON line per plan.

    python tools/power_tiles_time.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import power_mix as pm  # noqa: E402
from rx_tools_b200 import power  # noqa: E402

PLANS = {"24M-1766M_100k_61.44M": ("24M:1766M:100k", 61_440_000), "400-500M_10k_20M": ("400M:500M:10k", 20_000_000)}


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def run(name, reps):
    freq, cap = PLANS[name]
    plan = power.plan_range(freq)
    tl, tiles, offs = power.plan_tiles(plan, cap)
    dd = (tl.decim, power.ddc_lowpass(tl.decim, tl.n_taps, 15), 15)
    mx = power.PowerMix(plan, tl.capture_rate, offs, dd, "hamming")
    n16, G = mx.burst_int16(1), mx.lead
    xs = [pm.capture(n16 // 2, tl.capture_rate, offs[b:e], 10 + t, noise=1500) for t, (b, e, _) in enumerate(tiles)]
    d_x = [torch.from_numpy(x).cuda() for x in xs]
    stream = torch.cuda.ExternalStream(mx.stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sweep_ms, ddc_ms, acc_ms, same = [], [], [], True
    for r in range(reps + 1):
        mx.reset()
        e0.record(stream)
        for (b, e, _), d in zip(tiles, d_x):
            mx.accumulate_burst_device(b, e, d.data_ptr(), n16, sync=False)
        e1.record(stream)
        e1.synchronize()
        want = mx.read()
        mx.reset()
        ddc, acc = 0.0, 0.0
        for (b, e, _), d in zip(tiles, d_x):
            mx.accumulate_burst_device(b, e, d.data_ptr(), n16, sync=True)
            ddc += mx.kernel_ms()
            acc += mx.accumulate_ms()
        same &= all(np.array_equal(u, v) for u, v in zip(mx.read(), want))
        if r:
            sweep_ms.append(e0.elapsed_time(e1))
            ddc_ms.append(ddc)
            acc_ms.append(acc)
    mx.close()
    return dict(plan=name, hops=plan.n_hops, tiles=tl.n_tiles, hops_per_tile=tl.hops_per_tile,
                capture_rate=tl.capture_rate, decim=tl.decim, taps=tl.n_taps, lead=G,
                burst_complex=n16 // 2, burst_ms=n16 / 2 / tl.capture_rate * 1e3, ddc_kernel_ms=min(ddc_ms),
                accumulate_kernel_ms=min(acc_ms), sweep_device_ms=min(sweep_ms), synced_equals_async=same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print("gpu:", gpu_info())
    for name in PLANS:
        print(json.dumps(run(name, a.reps)))


if __name__ == "__main__":
    main()
