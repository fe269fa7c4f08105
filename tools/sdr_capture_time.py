"""Time one second of a 20 Msps device-resident capture through the rx_sdr I/Q down-converter handles
(rxb200_sdr_mix_*) for 8, 64 and 256 channels at arbitrary offsets: the single stage (M = 80, T = 2561, the capture
plan's filter for 250 kHz channels) against the two stages (fm_two_stage's plan for M' = 80: K = 40, M1 = 20,
T1 = 481, M2 = 4, T2 = 129), each writing CS16 and CF32.  Each figure is the median over repeats of the handle's
kernel time (CUDA events around its down-converter launches) for one device call of the whole second, after a
warm-up call.  Prints one JSON line per case, and first the board, its power limit and its maximum SM clock.

    python tools/sdr_capture_time.py [--repeats 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

RATE, S = 20_000_000, 250_000


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
    import fm_two_stage as fts
    from rx_tools_b200 import power, sdr
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    print(json.dumps({"board": board()}), flush=True)
    M = RATE // S
    single = (M, power.ddc_lowpass(M, min(8191, 32 * M + 1), 15), 15)
    two = fts.plan_stages(M)
    rng = np.random.default_rng(1)
    x = torch.from_numpy(rng.integers(-3000, 3001, size=2 * RATE, dtype=np.int32).astype(np.int16)).cuda()
    for n_ch in (8, 64, 256):
        offs = [int(v) for v in rng.choice(np.arange(-RATE // 2 + S, RATE // 2 - S), size=n_ch, replace=False)]
        for kind in ("single", "two"):
            h = sdr.SdrMix(RATE, offs, ddc=single) if kind == "single" else sdr.SdrMix(RATE, offs, two_stage=two)
            n = h.decimated_len(x.numel())
            for fmt in ("CS16", "CF32"):
                out = torch.empty(n_ch * n * sdr.ELEM_BYTES[sdr.FORMATS[fmt]], dtype=torch.uint8, device="cuda")
                ms = []
                for r in range(args.repeats + 1):
                    h.reset()
                    h.process_device(x.data_ptr(), x.numel(), fmt, out.data_ptr(), n_ch * n, n)
                    if r:
                        ms.append(h.kernel_ms())
                print(json.dumps({"channels": n_ch, "stages": 1 if kind == "single" else 2, "format": fmt,
                                  "outputs_per_channel": n, "kernel_ms_median": round(float(np.median(ms)), 3),
                                  "kernel_ms_min": round(float(min(ms)), 3), "capture_s": 1.0}), flush=True)
            h.close()


if __name__ == "__main__":
    main()
