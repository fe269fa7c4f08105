#!/usr/bin/env python
"""Time rx_power -F on hop buffers beyond shared memory (power_big_decim + the global-memory FFT path).

For each planner shape: device time per hop buffer (rxb200_power_kernel_ms over a batch of passes after a warm-up),
its split into power_big_decim and the rest of the big path (torch.profiler, a separate run), the front kernel's
achieved bytes/s against the buf_len * 2 bytes it has to read, its level-0 read amplification, and the port oracle
on one host core for the same buffers.  The boxcar big path (power_big_load) is timed the same way for comparison.
Needs a CUDA device; prints one JSON line per shape and writes them all to --out.

    python tools/power_decim_big_time.py [--out power_decim_big_time.json] [--mib 128] [--only 102.8M ...]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (-f argument, boxcar, -F argument, window)
SHAPES = [
    ("100M:100.5M:50", 0, 0, "hamming"),
    ("100M:100.1M:40", 0, 9, "hamming"),
    ("100M:100.1M:10", 0, 9, "blackman"),
    ("100M:100.01M:1", 0, 9, "hamming"),
    ("100M:102.8M:40", 1, 0, "blackman"),       # boxcar: power_big_load, for comparison
]


def decim_tiles(n_final, P, fir_on, n_sm):
    """power_big_decim's tiles as rxb200_power_accumulate_device plans them (decim_plan / decim_window in
    csrc/power_kernels.cu): returns (tile, level-0 complex samples staged over all tiles)."""
    def window0(m0, m1):
        lo, hi = max(m0 - 9 * fir_on, 0), m1 - 1
        for _ in range(P):
            lo, hi = max(2 * lo - 5, 0), (2 * hi if hi >= 5 else 8)
        return lo & ~3, hi | 3

    def span_max(t):
        return max(h - l + 1 for l, h in (window0(m0, min(m0 + t, n_final)) for m0 in range(0, n_final, t)))

    cap = (227 * 1024 - 256) // 4
    t = max(-(-n_final // (4 * n_sm)), 4 * (5 + 9 * fir_on))
    t = min(t, (cap - 7 - 5 * ((1 << P) - 1)) // (1 << P) + 1 - 9 * fir_on, n_final)
    while t > 1 and span_max(t) > cap:
        t -= 1
    staged = sum(h - l + 1 for l, h in (window0(m0, min(m0 + t, n_final)) for m0 in range(0, n_final, t)))
    return t, staged


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--mib", type=int, default=128, help="hop buffers per timed batch, MiB")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--only", nargs="*", default=None, help="time only the shapes whose -f argument contains one of these")
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import oracle
    from rx_tools_b200 import _lib, power
    port = oracle.port()
    dev = torch.device("cuda", 0)
    n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
    card = gpu_info()
    shapes = [s for s in SHAPES if not args.only or any(o in s[0] for o in args.only)]

    def setup(freq, boxcar, fir, wname):
        plan = power.plan_range(freq, 0.0, boxcar=boxcar, comp_fir_size=fir)
        n_pass = max(4, (args.mib << 20) // (plan.buf_len * 2 * plan.n_hops))
        rng = np.random.default_rng(7)
        base = rng.integers(-3000, 3001, size=(2, plan.n_hops, plan.buf_len), dtype=np.int32).astype(np.int16)
        d_in = torch.from_numpy(base).to(dev).repeat(-(-n_pass // 2), 1, 1)[:n_pass].contiguous()
        win = power.window_table(wname, 1 << plan.bin_e)
        return plan, n_pass, base, d_in, win, power.PowerScanner(plan, win)

    # phase 1: device time per hop buffer, CUDA events only (no profiler attached yet in this process)
    rows = []
    for freq, boxcar, fir, wname in shapes:
        try:
            plan, n_pass, base, d_in, win, sc = setup(freq, boxcar, fir, wname)
        except _lib.Rxb200Error as e:          # a library without the shape (RXB200_LIB pointing at an older build)
            print(json.dumps({"shape": f"-f {freq}", "card": card, "error": str(e)}), flush=True)
            continue
        n_buf = n_pass * plan.n_hops
        sc.scanner_device(d_in.data_ptr(), n_pass, sync=True)          # warm-up: allocations, modules
        ms = []
        for _ in range(args.repeats):
            sc.scanner_device(d_in.data_ptr(), n_pass, sync=True)
            ms.append(sc.kernel_ms())
        sc.close()
        pp = oracle.PowerParams(bin_e=plan.bin_e, buf_len=plan.buf_len, downsample=plan.downsample,
                                downsample_passes=plan.downsample_passes, comp_fir_size=plan.comp_fir_size,
                                boxcar=plan.boxcar)
        port_s = port.power_time(pp, win, base, 2, plan.n_hops, 1) / (2 * plan.n_hops)
        row = {"shape": f"-f {freq}" + ("" if boxcar else f" -F {fir}"), "card": card, "bin_e": plan.bin_e,
               "passes_P": plan.downsample_passes, "downsample": plan.downsample, "buf_len_int16": plan.buf_len,
               "hop_buffers_per_batch": n_buf, "device_ms_per_hop_buffer": float(np.median(ms)) / n_buf,
               "device_ms_per_hop_buffer_all": [m / n_buf for m in ms],
               "port_one_core_ms_per_hop_buffer": port_s * 1e3}
        if not boxcar:
            n_final = plan.buf_len >> (plan.downsample_passes + 1)
            tile, staged = decim_tiles(n_final, plan.downsample_passes, 1 if fir == 9 else 0, n_sm)
            row.update({"tile_final_samples": tile, "ctas": -(-n_final // tile),
                        "read_amplification": staged * 4 / (plan.buf_len * 2)})
        rows.append((row, (freq, boxcar, fir, wname)))
        del d_in
        torch.cuda.empty_cache()
    # phase 2: the front kernel against the rest of the big path, from a torch.profiler trace of one batch
    for row, spec in rows:
        plan, n_pass, base, d_in, win, sc = setup(*spec)
        n_buf = n_pass * plan.n_hops
        sc.scanner_device(d_in.data_ptr(), n_pass, sync=True)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            sc.scanner_device(d_in.data_ptr(), n_pass, sync=True)
        sc.close()
        front_name = "power_big_load" if spec[1] else "power_big_decim"
        front_us = rest_us = 0.0
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            t = ev.cuda_time_total if t is None else t
            if front_name in ev.key:
                front_us += t
            elif "power_big_" in ev.key:
                rest_us += t
        front_us /= n_buf
        rest_us /= n_buf
        row.update({"front_kernel": front_name, "front_us_per_hop_buffer": front_us, "rest_us_per_hop_buffer": rest_us,
                    "front_GBps_vs_buf_len_x2": plan.buf_len * 2 / (front_us * 1e-6) / 1e9 if front_us else None})
        print(json.dumps(row), flush=True)
        del d_in
        torch.cuda.empty_cache()
    rows = [r for r, _ in rows]
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
