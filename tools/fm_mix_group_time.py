#!/usr/bin/env python
"""End-to-end throughput of the channels of ONE capture spread over several GPUs (rxb200_fm_mix_group_process) against one
mixing handle (rxb200_fm_mix_process), both from pinned host buffers.

One 2.4 Msps capture (synth.cfg5_iq's channel 0, 2.4 M complex samples, one second) and K NBFM channels around its
centre, each demodulated with fm5a's shape (boxcar D = 100, -A lut, 24 kHz out) and offset_tuning on, in chunks of
131072 complex samples.  K = 64 sits on a 12.5 kHz raster.  K = 256 does not fit a 12.5 kHz raster inside the
capture's 2.4 MHz (|f| < 1.2 MHz takes at most 191 channels), so it sits on a 6.25 kHz raster.
Configurations: one mixing handle on GPU 0, a group of 1 member, and groups of 2, 4 and 8 members on distinct GPUs, as
many as are visible; a larger group is reported as not measured.  Every configuration runs one call on a fresh handle
and compares its PCM with the single handle's, then times --repeats calls after a warm-up call with the host clock
(each call returns synchronised).  Msamples/s counts capture samples times channels.  Prints one JSON line per
configuration, with every visible card's name and power limit read in the same run.

    python tools/fm_mix_group_time.py [--repeats 5] [--out fm_mix_group_time.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RATE, N = 2_400_000, 2_400_000
CHUNK = 262144                     # int16 per chunk = 131072 complex
RASTERS = {64: 12500, 256: 6250}   # K -> channel spacing in Hz
MEMBERS = (1, 2, 4, 8)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines() if q.returncode == 0 and q.stdout.strip() else ["unknown"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from rx_tools_b200 import _lib, fm, synth
    L = _lib.lib()
    n_gpus = int(L.rxb200_device_count())
    if n_gpus < 1:
        sys.exit("no CUDA device")
    cards = gpu_info()
    p = fm.FmParams(downsample=100, custom_atan=fm.ATAN_LUT, rate_out=24000, offset_tuning=1)
    n_int16 = 2 * N
    h_cap = torch.from_numpy(synth.cfg5_iq(N, 0)).pin_memory()
    rows = []

    def timed(call, reset, K):
        reset()
        call()                                    # warm-up
        t0 = time.perf_counter()
        for _ in range(args.repeats):
            call()
        dt = (time.perf_counter() - t0) / args.repeats
        return dt * 1e3, N * K / dt / 1e6

    for K, raster in RASTERS.items():
        offs = [raster * (k - K // 2) for k in range(K)]
        mx = fm.FmMix(p, RATE, offs)
        cap = mx.max_output(n_int16, CHUNK) + 8
        h_out = torch.zeros((K, cap), dtype=torch.int16, pin_memory=True)
        n_pcm = C.c_size_t(0)

        def emit(row):
            row.update({"cards": cards, "channels": K, "raster_hz": raster, "capture_rate": RATE, "complex": N,
                        "chunk_complex": CHUNK // 2, "shape": "D=100 lut offset_tuning", "repeats": args.repeats})
            print(json.dumps(row), flush=True)
            rows.append(row)

        def single_call():
            _lib.check(L.rxb200_fm_mix_process(mx._h, h_cap.data_ptr(), n_int16, CHUNK, h_out.data_ptr(), cap,
                                               C.byref(n_pcm), None))
        single_call()
        want = h_out.numpy()[:, :n_pcm.value].copy()
        ms, rate = timed(single_call, mx.reset, K)
        emit({"config": "one mixing handle", "devices": [0], "ms_per_call": ms, "Msamples_per_s": rate})
        for m in MEMBERS:
            if m > n_gpus:
                emit({"config": f"group of {m}", "devices": None, "Msamples_per_s": "not measured",
                      "reason": f"{n_gpus} GPU(s) visible"})
                continue
            g = fm.FmMixGroup(p, RATE, offs, list(range(m)))
            h_out.zero_()

            def group_call():
                _lib.check(L.rxb200_fm_mix_group_process(g._h, h_cap.data_ptr(), n_int16, CHUNK, h_out.data_ptr(), cap,
                                                         C.byref(n_pcm), None))
            group_call()
            equal = n_pcm.value == want.shape[1] and h_out.numpy()[:, :n_pcm.value].tobytes() == want.tobytes()
            ms, rate = timed(group_call, g.reset, K)
            emit({"config": f"group of {m}", "devices": list(range(m)), "ms_per_call": ms, "Msamples_per_s": rate,
                  "equal_to_one_handle": bool(equal)})
            g.close()
            if not equal:
                sys.exit(f"K={K}, group of {m}: PCM differs from the single mixing handle's")
        ms, rate = timed(single_call, mx.reset, K)
        emit({"config": "one mixing handle, again", "devices": [0], "ms_per_call": ms, "Msamples_per_s": rate})
        mx.close()
        del h_out
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
