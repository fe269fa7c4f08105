"""Time the capture handles' input stage (include/rxb200.h, "capture handles in a device's own format"; DESIGN.md
section 4.8) in one session on one GPU.

1. The widening kernel (sdr_convert_kernel's CS8, CU8 and CS12 kinds, RXB200_CVT_*_CS16) on 10^8 device-resident
   elements from and to 16-byte aligned buffers: the median kernel time over --repeats (CUDA events), and the bytes
   moved per second, counting the element's bytes in and its 4 bytes out, against the H100 SXM's 3.35 TB/s.
2. One second of capture through three plans, CS16 against CU8 and CS12: the rx_power 88-108 MHz capture plan (8 hops,
   R = 20 Msps, M = 8), tools/sdr_capture_time.py's 64 channels at 20 Msps (single stage, M = 80, T = 2561, CS16 out)
   and 64 channels of tools/fm_raster_time.py's 768-bin rx_fm raster at 19.2 Msps (M = 64, T = 257).  For each it
   reports the host call (pinned host capture, host clock around the call, median) and the device call (device-resident
   capture, host clock around the call and a synchronise), and the stage's share of the device call: the widening
   kernel's time on the second's elements over the device call in that format.
The card's name, power limit and maximum SM clock are printed first, then one JSON line per case.

    python tools/device_format_time.py [--repeats 5]
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

KINDS = {"CS8": 5, "CU8": 6, "CS12": 3}           # RXB200_CVT_CS8_CS16, _CU8_CS16, _CS12_CS16
ELEM = {"CS16": 4, "CS8": 2, "CU8": 2, "CS12": 3}
HBM = 3.35e12


def board():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                     # the timing itself needs no nvidia-smi
        return f"unknown ({e})"


def median_ms(fn, repeats, before=None):
    out = []
    for k in range(repeats + 1):
        if before:
            before()
        t0 = time.perf_counter()
        fn()
        t1 = time.perf_counter()
        if k:
            out.append(1e3 * (t1 - t0))
    return float(np.median(out))


def widen_ms(torch, lib, fmt, d_src, n, d_dst, repeats):
    """Median kernel time of one widening of n elements (CUDA events)."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for k in range(repeats + 1):
        a.record()
        rc = lib.rxb200_sdr_convert_device(KINDS[fmt], d_src.data_ptr(), n, d_dst.data_ptr(), None)
        b.record()
        assert rc == 0
        torch.cuda.synchronize()
        if k:
            out.append(a.elapsed_time(b))
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch
    from rx_tools_b200 import _lib, fm, power, sdr
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to time")
    lib = _lib.lib()
    print(json.dumps({"board": board(), "gpu": torch.cuda.get_device_name(0)}), flush=True)
    rng = np.random.default_rng(1)

    # ---- 1. the kernel
    n = 10**8
    d_dst = torch.empty(n, dtype=torch.int32, device="cuda")
    for fmt in KINDS:
        d_src = torch.randint(0, 256, (ELEM[fmt] * n,), dtype=torch.uint8, device="cuda")
        ms = widen_ms(torch, lib, fmt, d_src, n, d_dst, args.repeats)
        bps = (ELEM[fmt] + 4) * n / (ms * 1e-3)
        print(json.dumps({"case": "kernel", "format": fmt, "elements": n, "ms": round(ms, 3),
                          "bytes_per_s": f"{bps:.3e}", "of_hbm": round(bps / HBM, 3)}), flush=True)
        del d_src

    # ---- 2. the plans
    def power_plan():
        plan = power.plan_range("88M:108M:10k")
        cp, offs = power.plan_capture(plan, 20_000_000)
        win = power.window_table("hamming", 1 << plan.bin_e)
        dd = (cp.decim, power.ddc_lowpass(cp.decim, cp.n_taps, 15), 15)
        pas = cp.decim * plan.buf_len // 2
        n_c = (cp.capture_rate // pas) * pas                  # one second, cut to whole passes
        return (lambda: power.PowerMix(plan, cp.capture_rate, offs, dd, win)), n_c, "power"

    def sdr_plan():
        R, S, M = 20_000_000, 250_000, 80
        offs = [int(v) for v in rng.choice(np.arange(-R // 2 + S, R // 2 - S), size=64, replace=False)]
        dd = (M, power.ddc_lowpass(M, min(8191, 32 * M + 1), 15), 15)
        return (lambda: sdr.SdrMix(R, offs, ddc=dd)), R, "sdr"

    def raster_plan():
        R, K, M, D, c = 19_200_000, 768, 64, 12, 64
        bins = [(j - c // 2) % K for j in range(c)]
        nbfm = fm.FmParams(mode=fm.MODE_FM, downsample=D, custom_atan=fm.ATAN_LUT, rate_out=25000, offset_tuning=1)
        j = np.arange(257) - 128.0
        h = np.sinc(2.0 * 12500 / R * j) * np.hamming(257)
        taps = np.round(h / h.sum() * 32768.0).astype(np.int32)   # fm_raster_time.py's 257-tap filter
        return (lambda: fm.FmMix(nbfm, ddc=(M, taps, 30), raster=(K, bins))), R, "fm_raster"

    for make_plan in (power_plan, sdr_plan, raster_plan):
        make, n_c, kind = make_plan()
        res = {"case": "plan", "plan": kind, "samples": n_c}
        base = rng.integers(0, 256, size=3 * n_c, dtype=np.uint8)
        for fmt in ("CS16", "CU8", "CS12"):
            if fmt == "CS16":
                src = torch.from_numpy(rng.integers(-3000, 3001, size=2 * n_c, dtype=np.int32).astype(np.int16))
            else:
                src = torch.from_numpy(base[:ELEM[fmt] * n_c].copy())
            h = make()
            if fmt != "CS16":
                h.set_input_format(fmt)
            d_src, h_src = src.cuda(), src.pin_memory()
            n16 = 2 * n_c
            if kind == "power":
                def dev():
                    h.accumulate_device(d_src.data_ptr(), n16, sync=True)

                def host():
                    _lib.check(lib.rxb200_power_mix_accumulate(h._m, h_src.data_ptr(), n16))
            elif kind == "sdr":
                nd = h.decimated_len(n16) + 1
                d_out = torch.empty((64, 2 * nd), dtype=torch.int16, device="cuda")
                h_out = torch.empty((64, 2 * nd), dtype=torch.int16).pin_memory()
                got = C.c_size_t(0)

                def dev():
                    h.process_device(d_src.data_ptr(), n16, sdr.OUT_CS16, d_out.data_ptr(), 64 * nd, nd)

                def host():
                    _lib.check(lib.rxb200_sdr_mix_process(h._h, h_src.data_ptr(), n16, sdr.OUT_CS16, h_out.data_ptr(),
                                                          64 * nd, nd, C.byref(got)))
            else:
                chunk = 2 * 64 * 2048
                cap = h.max_output(n16, chunk) + 8
                d_out = torch.empty((64, cap), dtype=torch.int16, device="cuda")
                h_out = torch.empty((64, cap), dtype=torch.int16).pin_memory()
                got = C.c_size_t(0)

                def dev():
                    h.process_device(d_src.data_ptr(), n16, chunk, d_out.data_ptr(), cap, sync=True)

                def host():
                    _lib.check(lib.rxb200_fm_mix_process(h._h, h_src.data_ptr(), n16, chunk, h_out.data_ptr(), cap,
                                                         C.byref(got), None))

            def reset():
                h.reset()
                torch.cuda.synchronize()

            res[f"dev_ms_{fmt}"] = round(median_ms(dev, args.repeats, reset), 3)
            res[f"host_ms_{fmt}"] = round(median_ms(host, args.repeats, reset), 3)
            if fmt != "CS16":
                dd = torch.empty(n_c, dtype=torch.int32, device="cuda")
                st = widen_ms(torch, lib, fmt, d_src, n_c, dd, args.repeats)
                res[f"stage_ms_{fmt}"] = round(st, 3)
                res[f"stage_share_{fmt}"] = round(st / res[f"dev_ms_{fmt}"], 4)
                del dd
            h.close()
            del d_src, h_src
            torch.cuda.empty_cache()
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
