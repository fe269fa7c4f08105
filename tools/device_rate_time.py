"""Time one second of device-rate capture through each capture-handle kind with a resampler attached, against the same
handle on the pre-resampled capture, for each named plan of tests/resample.py.  The kinds are an rx_fm single-stage
handle (4 channels, decimation 8, chunks of 131072 decimated samples), an rx_sdr single-stage handle (4 channels, decimation 8, CS16) and
an rx_power handle (the "fm_band" sweep's hops, whole passes).  Per plan and kind it reports, as the median over
--repeats after a warm-up call:
  - dev_ms / dev_ms_pre: one device call of the second (host clock around the call and a synchronise), with the
    resampler attached on R_dev device samples / without it on the R capture samples they resample to;
  - host_ms / host_ms_pre: the same through the host entry, from pinned host buffers;
  - extra_ms: dev_ms - dev_ms_pre, the GPU time the resampler adds to a second of capture.
The card's name, power limit and maximum SM clock are printed first, then one JSON line per plan and kind.

    python tools/device_rate_time.py [--repeats 5]
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


def median_ms(fn, repeats, reset):
    out = []
    for k in range(repeats + 1):
        reset()
        t0 = time.perf_counter()
        fn()
        t1 = time.perf_counter()
        if k:
            out.append(1e3 * (t1 - t0))
    return round(float(np.median(out)), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch
    import power_mix as pm
    import resample as rm
    from rx_tools_b200 import _lib, fm, power, sdr
    from rx_tools_b200 import resample
    print("board:", board(), flush=True)
    P = fm.derive_params(rate_s=170_000).params
    for name, R_dev, R, span, _, _ in rm.NAMED:
        p = resample.plan_resample(R_dev, R, span)
        taps = resample.lowpass(p.up, p.down, p.taps_per_phase)
        offs = [-(R // 8), 0, R // 8, R // 4]
        dd = (8, power.ddc_lowpass(8, 257, 15), 15)
        pl, win, _, _, pdd = pm.shape("fm_band")
        pas = pdd[0] * pl.buf_len // 2
        kinds = {
            "fm_mix": lambda: fm.FmMix(P, R, offs, ddc=dd),
            "sdr_mix": lambda: sdr.SdrMix(R, offs, ddc=dd),
            "power_mix": lambda: power.PowerMix(pl, R, [0] * pl.n_hops, pdd, win),
        }
        for kind, make in kinds.items():
            if kind == "power_mix":                       # device samples that resample to whole passes
                n_pass = max(1, R // pas)
                n_dev = resample.in_len(p.up, p.down, 0, n_pass * pas)
            else:
                n_dev = R_dev
            x = torch.randint(-8000, 8000, (2 * n_dev,), dtype=torch.int16)
            r = resample.Resampler(p.up, p.down, taps, p.shift)
            y = torch.from_numpy(r.process(x.numpy()))
            r.close()
            res = {"plan": name, "kind": kind, "R_dev": R_dev, "R": R, "L": p.up, "N": p.down, "J": p.taps_per_phase,
                   "device_samples": n_dev, "capture_samples": y.numel() // 2}
            for tag, src in (("", x), ("_pre", y)):
                h = make()
                if not tag:
                    h.set_device_rate(p.up, p.down, taps, p.shift)
                d_src, h_src = src.cuda(), src.pin_memory()
                n16 = src.numel()
                if kind == "fm_mix":
                    chunk = 2 * 8 * 131072                # capture int16 per chain chunk: 131072 decimated samples
                    cap = h.max_output(n16, chunk) + 8
                    d_out = torch.empty((4, cap), dtype=torch.int16, device="cuda")
                    h_out = torch.empty((4, cap), dtype=torch.int16).pin_memory()
                    n = C.c_size_t(0)

                    def dev():
                        h.process_device(d_src.data_ptr(), n16, chunk, d_out.data_ptr(), cap, sync=True)

                    def host():
                        _lib.check(_lib.lib().rxb200_fm_mix_process(h._h, h_src.data_ptr(), n16, chunk,
                                                                    h_out.data_ptr(), cap, C.byref(n), None))
                elif kind == "sdr_mix":
                    nd = h.decimated_len(n16) + 1
                    d_out = torch.empty((4, 2 * nd), dtype=torch.int16, device="cuda")
                    h_out = torch.empty((4, 2 * nd), dtype=torch.int16).pin_memory()
                    n = C.c_size_t(0)

                    def dev():
                        h.process_device(d_src.data_ptr(), n16, sdr.OUT_CS16, d_out.data_ptr(), 4 * nd, nd)

                    def host():
                        _lib.check(_lib.lib().rxb200_sdr_mix_process(h._h, h_src.data_ptr(), n16, sdr.OUT_CS16,
                                                                     h_out.data_ptr(), 4 * nd, nd, C.byref(n)))
                else:
                    def dev():
                        h.accumulate_device(d_src.data_ptr(), n16, sync=True)

                    def host():
                        _lib.check(_lib.lib().rxb200_power_mix_accumulate(h._m, h_src.data_ptr(), n16))

                def reset():
                    h.reset()
                    torch.cuda.synchronize()

                res["dev_ms" + tag] = median_ms(dev, args.repeats, reset)
                res["host_ms" + tag] = median_ms(host, args.repeats, reset)
                h.close()
            res["extra_ms"] = round(res["dev_ms"] - res["dev_ms_pre"], 3)
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
