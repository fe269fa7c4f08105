#!/usr/bin/env python
"""Time rx_fm calls whose chunks are not a multiple of 8 complex samples (the any-length kernel) against the same
calls at the usual 131072-sample chunk.

For the fm1, fm5a and fm2a shapes of bench.py, at bench.py's sizes, device-resident calls (rxb200_fm_process_device)
with chunks of 131071 complex samples and of 131072: the device time of a call (rxb200_fm_kernel_ms, median of the
repeats after a warm-up call), the kernel kind each call took, and the card's name, power limit and maximum SM clock
read in the same run.  Needs a CUDA device; prints one JSON line per shape and chunk and writes them all to --out.

    python tools/any_chunk_time.py [--out any_chunk_time.json] [--repeats 5] [--only fm1 fm5a fm2a]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CHUNKS = (131072, 131071)          # complex samples
FM5A_CHANNELS, FM5A_PER = 256, 2_400_000 - (2_400_000 % 8)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def shape(name):
    """(params, channels, complex samples per channel, one period of input) as bench.py builds them."""
    from rx_tools_b200 import fm, synth
    if name == "fm5a":
        p = fm.FmParams(downsample=100, custom_atan=fm.ATAN_LUT, rate_out=24000)
        return p, FM5A_CHANNELS, FM5A_PER, synth.cfg5_iq(FM5A_PER, 0)
    if name == "fm1":
        p = fm.derive_params(rate_s=1024000, rate_r=24000).params
        return p, 1, (256 << 20) // 4, synth.cfg1_iq(1 << 24)
    p = fm.derive_params(wbfm=1, rate_s=2400000, rate_r=48000).params
    return p, 1, (1024 << 20) // 4, synth.cfg2_iq(1 << 24)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--only", nargs="*", default=["fm1", "fm5a", "fm2a"])
    args = ap.parse_args()
    import torch
    from rx_tools_b200 import fm
    dev = torch.device("cuda", 0)
    card = gpu_info()
    rows = []
    for name in args.only:
        p, n_ch, n, period = shape(name)
        # the period tiled over the call and the channels, as bench.py does
        d_in = torch.from_numpy(period).to(dev).repeat(n_ch * (n // (period.size // 2))).contiguous()
        for chunk in CHUNKS:
            d = fm.FmDemod(p, n_channels=n_ch)
            cap = d.max_output(2 * n, 2 * chunk) + 8
            d_out = torch.empty(n_ch * cap, dtype=torch.int16, device=dev)
            d.process_device(d_in.data_ptr(), 2 * n, 2 * chunk, d_out.data_ptr(), cap, sync=True)     # warm-up
            ms = []
            for _ in range(args.repeats):
                d.process_device(d_in.data_ptr(), 2 * n, 2 * chunk, d_out.data_ptr(), cap, sync=True)
                ms.append(d.kernel_ms())
            st = d.stats()
            row = {"shape": name, "card": card, "chunk_complex": chunk, "channels": n_ch, "complex_per_channel": n,
                   "kernel_kind": st["kernel_kind"], "launches": st["launches"], "device_ms": float(np.median(ms)),
                   "device_ms_all": ms, "Msamples_per_s": n_ch * n / (float(np.median(ms)) * 1e-3) / 1e6}
            print(json.dumps(row), flush=True)
            rows.append(row)
            d.close()
            del d_out
        del d_in
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
