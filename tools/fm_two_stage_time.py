"""Times two-stage mixing handles (rxb200_fm_mix_create_two_stage) against decimating handles (rxb200_fm_mix_create_ddc)
and, for channels on the 768-bin raster, raster handles (rxb200_fm_mix_create_raster), on one second of a 19.2 Msps
capture into a D = 12 lut NBFM chain (300 kHz -> 25 kHz).  The two-stage handle uses the rx_fm shell's plan at M' = 64:
K = 32 bins, a 385-tap coarse filter at M1 = 16, then a 129-tap fine filter at M2 = 4.  The decimating handle runs
rxb200_ddc_lowpass(64, T, 15) with T = 257 and 2049 taps, on the same offsets rounded to 25 kHz (its table mixer refuses
most arbitrary offsets); the raster handle the 2049-tap one, on random bins of the 768-bin raster.  The two-stage
channels sit at arbitrary offsets.

For each configuration: the front stage's device time (CUDA events around its kernels, FmMix.mix_ms) of one device call
over the whole second, best of --reps after a warm-up call.  The first line names the card and its power limit.
Prints one JSON line per configuration.

    python tools/fm_two_stage_time.py [--reps 3] [--c 8,64,256,768]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from rx_tools_b200 import fm, power  # noqa: E402

RATE, M = 19_200_000, 64
CHUNK = 2 * M * 2048
NBFM12 = dict(mode=0, downsample=12, custom_atan=2, rate_out=25000, offset_tuning=1)


def front_ms(mx, d_x, n16, reps):
    cap = mx.max_output(n16, CHUNK)
    d_out = torch.empty((mx.n_channels, cap), dtype=torch.int16, device="cuda")
    best = None
    for r in range(reps + 1):
        mx.reset()
        mx.process_device(d_x.data_ptr(), n16, CHUNK, d_out.data_ptr(), cap, sync=True)
        if r:
            best = mx.mix_ms() if best is None else min(best, mx.mix_ms())
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--c", default="8,64,256,768")
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"card": q.stdout.strip()}))
    n = RATE - RATE % (CHUNK // 2)
    rng = np.random.default_rng(1)
    x = rng.integers(-3000, 3001, size=2 * n).astype(np.int16)
    d_x = torch.from_numpy(x).cuda()
    p = fm.FmParams(**{k: v for k, v in NBFM12.items()})
    K1, M1 = 32, 16
    coarse = (M1, power.ddc_lowpass(M1, 24 * M1 + 1, 15), 30)
    fine = (4, power.ddc_lowpass(4, 129, 15), 15)
    for C in (int(v) for v in a.c.split(",")):
        offs = [int(v) for v in rng.integers(-RATE // 2 + 150_000, RATE // 2 - 150_000, size=C)]
        bins = [int(v) for v in rng.choice(768, size=C, replace=False)] if C <= 768 else None
        rows = []
        mx = fm.FmMix(p, RATE, offs, two_stage=(K1, coarse, fine))
        rows.append(("two_stage", f"K{K1} M1 {M1} T1 {coarse[1].size} M2 4 T2 129", front_ms(mx, d_x, 2 * n, a.reps)))
        mx.close()
        # the table mixer refuses most arbitrary offsets (period above 2^20): the DDC handle's channels are the same
        # offsets rounded to 25 kHz, which costs it the same work
        grid = [25_000 * round(f / 25_000) for f in offs]
        for T in (257, 2049):
            mx = fm.FmMix(p, RATE, grid, ddc=(M, power.ddc_lowpass(M, T, 15), 15))
            rows.append(("ddc", f"T {T}", front_ms(mx, d_x, 2 * n, a.reps)))
            mx.close()
        if bins is not None:
            mx = fm.FmMix(p, ddc=(M, power.ddc_lowpass(M, 2049, 15), 30), raster=(768, bins))
            rows.append(("raster", "K768 T 2049", front_ms(mx, d_x, 2 * n, a.reps)))
            mx.close()
        for kind, shape, ms in rows:
            print(json.dumps({"channels": C, "kind": kind, "shape": shape, "front_ms_per_s": round(ms * RATE / n, 3)}))


if __name__ == "__main__":
    main()
