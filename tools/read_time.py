#!/usr/bin/env python
"""Time one device read per call (rxb200_fm_process_read_device) for the fm2b shape (-M wbfm -s 300k -F 9 -r 48k),
off the passes' granule, against the aligned rxb200_fm_process_device call at the nearest granule multiple.

For reads of 2044, 8188 and 131071 complex samples (and 2048, 8192, 131072 aligned): the device time of a call
(rxb200_fm_kernel_ms) and the host wall time of a synchronous call (entry to return, sync on), medians over --repeats
calls on one handle after warm-up calls, the kernel kind each took, and the card's name, power limit and maximum SM clock
read in the same run.  Needs a CUDA device; prints one JSON line per read length and writes them all to --out.

    python tools/read_time.py [--out read_time.json] [--repeats 200]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from any_chunk_time import gpu_info  # noqa: E402

READS = ((2044, 2048), (8188, 8192), (131071, 131072))      # (off the granule, aligned) complex samples


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--repeats", type=int, default=200)
    args = ap.parse_args()
    import torch
    from rx_tools_b200 import fm, synth
    dev = torch.device("cuda", 0)
    card = gpu_info()
    p = fm.derive_params(wbfm=1, rate_s=300000, rate_r=48000, use_F=1, comp_fir_size=9).params
    x = torch.from_numpy(synth.cfg2_iq(1 << 18)).to(dev)
    rows = []
    for pair in READS:
        for n, read in zip(pair, (True, False)):
            d = fm.FmDemod(p)
            cap = d.max_output(2 * n, 2 * n) + 8
            d_out = torch.empty(cap, dtype=torch.int16, device=dev)

            def call():
                if read:
                    return d.process_read_device(x.data_ptr(), 2 * n, d_out.data_ptr(), cap, sync=True)
                return d.process_device(x.data_ptr(), 2 * n, 2 * n, d_out.data_ptr(), cap, sync=True)

            for _ in range(10):
                call()
            ms, wall = [], []
            for _ in range(args.repeats):
                t0 = time.perf_counter()
                call()
                wall.append((time.perf_counter() - t0) * 1e3)
                ms.append(d.kernel_ms())
            st = d.stats()
            row = {"shape": "fm2b", "card": card, "entry": "process_read_device" if read else "process_device",
                   "complex": n, "kernel_kind": st["kernel_kind"], "launches": st["launches"],
                   "device_ms": float(np.median(ms)), "host_ms": float(np.median(wall)),
                   "host_ms_p90": float(np.percentile(wall, 90)), "signal_ms_at_2400ksps": n / 2400.0}
            print(json.dumps(row), flush=True)
            rows.append(row)
            d.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
