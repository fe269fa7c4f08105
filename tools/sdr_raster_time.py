"""Time one second of device-resident capture through the rx_sdr I/Q handles (rxb200_sdr_mix_*) on a channel raster:
the raster kind (rxb200_sdr_mix_create_raster), the single stage on the same offsets (rxb200_sdr_mix_create) and the
two stages on rxb200_fm_plan_capture_two_stage's plan for the same -f set (rxb200_sdr_mix_create_two_stage), each
writing CS16 and CF32.  Two rasters:
  - the FM broadcast band, one -f per station 88.1-107.9 MHz at -s 250k: rxb200_fm_plan_capture_raster gives
    R = 20.25 Msps, K = 405, M = 81, T = 2593 for 100 channels;
  - tools/fm_raster_time.py's 768-bin 19.2 Msps raster (25 kHz bins), M = 64, T = 2049, at 8, 64, 256 and 768
    channels spread over the bins (the single stage mixes the Nyquist bin's channel by 0 instead, the same work).
Each kind runs one second at its own capture rate (the two-stage plan rounds M up to a multiple of 4).  Each figure is
the median over --repeats of the handle's kernel time (CUDA events around its down-converter launches) for one device
call of the whole second, after a warm-up call.  Prints the card's name, power limit and maximum SM clock first, then
one JSON line per case.

    python tools/sdr_raster_time.py [--repeats 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def board():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                     # the timing itself needs no nvidia-smi
        return f"unknown ({e})"


def time_handle(h, x, n_samples, fmt, repeats):
    import torch
    from rx_tools_b200 import sdr
    n = h.decimated_len(2 * n_samples)
    out = torch.empty(h.n_channels * n * sdr.ELEM_BYTES[sdr.FORMATS[fmt]], dtype=torch.uint8, device="cuda")
    ms = []
    for r in range(repeats + 1):
        h.reset()
        h.process_device(x.data_ptr(), 2 * n_samples, fmt, out.data_ptr(), h.n_channels * n, n)
        if r:
            ms.append(h.kernel_ms())
    return n, ms


def cases(tuned, chain_rate, K, bins, M, T):
    """(kind, capture rate, constructor) of the three kinds for one -f set whose raster plan is (K, bins, M, T)."""
    from rx_tools_b200 import fm, power, sdr
    R = M * chain_rate
    taps = power.ddc_lowpass(M, T, 15)
    offs = [(b if 2 * b < K else b - K) * (R // K) for b in bins]
    offs = [o if 2 * abs(o) < R else 0 for o in offs]
    tp, toffs = fm.plan_capture_two_stage(tuned, chain_rate, 1 << 40)
    coarse = (tp.coarse_decim, power.ddc_lowpass(tp.coarse_decim, tp.coarse_taps, 15), tp.coarse_shift)
    fine = (tp.fine_decim, power.ddc_lowpass(tp.fine_decim, tp.fine_taps, 15), tp.fine_shift)
    return [("raster", R, lambda: sdr.SdrMix(ddc=(M, taps, 30), raster=(K, bins))),
            ("single", R, lambda: sdr.SdrMix(R, offs, ddc=(M, taps, 15))),
            ("two_stage", tp.capture_rate, lambda: sdr.SdrMix(tp.capture_rate, toffs, two_stage=(tp.n_bins, coarse, fine)))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch
    from rx_tools_b200 import fm
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    print(json.dumps({"board": board()}), flush=True)
    rng = np.random.default_rng(1)
    x = torch.from_numpy(rng.integers(-3000, 3001, size=2 * 21_500_000, dtype=np.int32).astype(np.int16)).cuda()
    sets = []
    tuned = [88_100_000 + 200_000 * k for k in range(100)]
    plan, bins = fm.plan_capture_raster(tuned, 250_000, 25_000_000)
    assert (plan.n_bins, plan.decim, plan.n_taps, plan.capture_rate) == (405, 81, 2593, 20_250_000)
    sets.append(("fm_broadcast", tuned, 250_000, plan.n_bins, bins, plan.decim, plan.n_taps))
    for C in (8, 64, 256, 768):
        bins = [k * 768 // C for k in range(C)]
        tuned = [1_000_000_000 + 25_000 * (b if 2 * b < 768 else b - 768) for b in bins]
        sets.append((f"k768_c{C}", tuned, 300_000, 768, bins, 64, 2049))
    for name, tuned, c, K, bins, M, T in sets:
        for kind, R, make in cases(tuned, c, K, bins, M, T):
            h = make()
            for fmt in ("CS16", "CF32"):
                n, ms = time_handle(h, x, R, fmt, args.repeats)
                print(json.dumps({"set": name, "kind": kind, "channels": len(bins), "capture_rate": R, "format": fmt,
                                  "outputs_per_channel": n, "kernel_ms_median": round(float(np.median(ms)), 3),
                                  "kernel_ms_min": round(float(min(ms)), 3), "capture_s": 1.0}), flush=True)
            h.close()


if __name__ == "__main__":
    main()
