#!/usr/bin/env python
"""End-to-end rx_fm throughput of a channel group over several GPUs (rxb200_fm_group_process) against one plain handle
(rxb200_fm_process), both from pinned host buffers.

The fm5a shape of bench.py: 256 NBFM channels of 2.4 M complex samples, chunk 131072 complex, boxcar D = 100, lut.
Channel c is bench.py's input period rotated by c * 997 samples, so that a channel put in the wrong row shows.  Every
configuration runs one call on a fresh handle and compares its PCM with the plain handle's, then times --repeats calls
after a warm-up call with the host clock (each call returns synchronised): Msamples/s = channels * samples / time.
Groups of 1, 2, 4 and 8 members on distinct GPUs, as many as are visible; a larger group is reported as not measured.
Prints one JSON line per configuration, with every visible card's name and power limit read in the same run.

    python tools/fm_group_time.py [--repeats 5] [--out fm_group_time.json]
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

CHANNELS, PER = 256, 2_400_000 - (2_400_000 % 8)
CHUNK = 262144                     # int16 per chunk = 131072 complex
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
    p = fm.FmParams(downsample=100, custom_atan=fm.ATAN_LUT, rate_out=24000)
    n_int16 = 2 * PER
    period = synth.cfg5_iq(PER, 0)
    h_in = torch.empty((CHANNELS, n_int16), dtype=torch.int16, pin_memory=True)
    x = h_in.numpy()
    for c in range(CHANNELS):
        x[c] = np.roll(period, 2 * 997 * c)
    plain = fm.FmDemod(p, device=0, n_channels=CHANNELS)
    cap = plain.max_output(n_int16, CHUNK) + 8
    h_out = torch.zeros((CHANNELS, cap), dtype=torch.int16, pin_memory=True)
    n_pcm = C.c_size_t(0)

    def plain_call():
        _lib.check(L.rxb200_fm_process(plain._h, h_in.data_ptr(), n_int16, CHUNK, h_out.data_ptr(), cap, C.byref(n_pcm),
                                       None))

    def timed(call):
        call()                                    # warm-up
        t0 = time.perf_counter()
        for _ in range(args.repeats):
            call()
        dt = (time.perf_counter() - t0) / args.repeats
        return dt * 1e3, CHANNELS * PER / dt / 1e6

    plain_call()
    want = h_out.numpy()[:, :n_pcm.value].copy()
    rows = []

    def emit(row):
        row.update({"cards": cards, "shape": "fm5a", "channels": CHANNELS, "complex_per_channel": PER,
                    "chunk_complex": CHUNK // 2, "repeats": args.repeats})
        print(json.dumps(row), flush=True)
        rows.append(row)

    ms, rate = timed(plain_call)
    emit({"config": "plain handle", "devices": [0], "ms_per_call": ms, "Msamples_per_s": rate})
    for m in MEMBERS:
        if m > n_gpus:
            emit({"config": f"group of {m}", "devices": None, "Msamples_per_s": "not measured",
                  "reason": f"{n_gpus} GPU(s) visible"})
            continue
        g = fm.FmGroup(p, CHANNELS, list(range(m)))
        h_out.zero_()

        def group_call():
            _lib.check(L.rxb200_fm_group_process(g._h, h_in.data_ptr(), n_int16, CHUNK, h_out.data_ptr(), cap,
                                                 C.byref(n_pcm), None))
        group_call()
        equal = n_pcm.value == want.shape[1] and h_out.numpy()[:, :n_pcm.value].tobytes() == want.tobytes()
        ms, rate = timed(group_call)
        emit({"config": f"group of {m}", "devices": list(range(m)), "ms_per_call": ms, "Msamples_per_s": rate,
              "equal_to_plain": bool(equal)})
        g.close()
        if not equal:
            sys.exit(f"group of {m}: PCM differs from the plain handle's")
    ms, rate = timed(plain_call)
    emit({"config": "plain handle, again", "devices": [0], "ms_per_call": ms, "Msamples_per_s": rate})
    plain.close()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
