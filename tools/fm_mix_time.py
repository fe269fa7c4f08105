#!/usr/bin/env python
"""Throughput of several NBFM channels demodulated from ONE capture (rxb200_fm_mix_*), against K separate streams.

One 2.4 Msps capture (synth.cfg5_iq's channel 0, 2.4 M complex samples, one second), K in {1, 8, 32, 64} channels on a
12.5 kHz raster around its centre, each demodulated with fm5a's shape (boxcar D = 100, -A lut, 24 kHz out) and
offset_tuning on, in chunks of 131072 complex samples.  For each K:
- device-resident: rxb200_fm_mix_process_device from a capture already in HBM.  CUDA events on the handle's stream
  around --repeats calls after a warm-up call give the whole call's time; rxb200_fm_mix_kernel_ms gives the last call's
  fm_mix_kernel alone.
- from the host: rxb200_fm_mix_process from a pinned capture into pinned PCM, against the same K channels fed as K
  separate pre-mixed streams (made on the GPU by rxb200_mix_device, copied to a pinned [K][n] buffer) through
  rxb200_fm_process on a plain K-channel handle.  Host clock around --repeats synchronised calls after a warm-up;
  the two PCM outputs must be equal.
Prints one JSON line per K with the card's name and power limit read in the same run.

    python tools/fm_mix_time.py [--repeats 5] [--out fm_mix_time.json]
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
KS = (1, 8, 32, 64)


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
    if int(L.rxb200_device_count()) < 1:
        sys.exit("no CUDA device")
    cards = gpu_info()
    p = fm.FmParams(downsample=100, custom_atan=fm.ATAN_LUT, rate_out=24000, offset_tuning=1)
    n_int16 = 2 * N
    h_cap = torch.from_numpy(synth.cfg5_iq(N, 0)).pin_memory()
    d_cap = h_cap.cuda()
    rows = []
    for K in KS:
        offs = [12500 * (k - K // 2) for k in range(K)]
        mx = fm.FmMix(p, RATE, offs)
        cap = mx.max_output(n_int16, CHUNK) + 8
        d_out = torch.zeros((K, cap), dtype=torch.int16, device="cuda")
        # device-resident
        stream = torch.cuda.ExternalStream(mx.stream)
        mx.process_device(d_cap.data_ptr(), n_int16, CHUNK, d_out.data_ptr(), cap, sync=True)
        mx.reset()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.repeats):
            mx.process_device(d_cap.data_ptr(), n_int16, CHUNK, d_out.data_ptr(), cap)
        e1.record(stream)
        e1.synchronize()
        dev_ms = e0.elapsed_time(e1) / args.repeats
        mix_ms = mx.mix_ms()
        chain_ms = mx.kernel_ms()
        # from the host: one pinned capture against K pinned pre-mixed streams
        h_out = torch.zeros((K, cap), dtype=torch.int16, pin_memory=True)
        n_pcm = C.c_size_t(0)

        def mix_call():
            _lib.check(L.rxb200_fm_mix_process(mx._h, h_cap.data_ptr(), n_int16, CHUNK, h_out.data_ptr(), cap,
                                               C.byref(n_pcm), None))
        mx.reset()
        mix_call()
        got = h_out.numpy()[:, :n_pcm.value].copy()
        d_sep = torch.empty((K, n_int16), dtype=torch.int16, device="cuda")
        for k, f in enumerate(offs):
            fm.mix_device(RATE, f, 0, d_cap.data_ptr(), N, d_sep[k].data_ptr())
        torch.cuda.synchronize()
        h_sep = d_sep.cpu().pin_memory()
        del d_sep
        plain = fm.FmDemod(p, n_channels=K)

        def plain_call():
            _lib.check(L.rxb200_fm_process(plain._h, h_sep.data_ptr(), n_int16, CHUNK, h_out.data_ptr(), cap,
                                           C.byref(n_pcm), None))
        plain_call()
        equal = n_pcm.value == got.shape[1] and h_out.numpy()[:, :n_pcm.value].tobytes() == got.tobytes()

        def timed(call, reset):
            reset()
            call()                                    # warm-up
            t0 = time.perf_counter()
            for _ in range(args.repeats):
                call()
            return (time.perf_counter() - t0) / args.repeats * 1e3
        host_mix_ms = timed(mix_call, mx.reset)
        host_sep_ms = timed(plain_call, plain.reset)
        row = {"cards": cards, "channels": K, "capture_rate": RATE, "complex": N, "chunk_complex": CHUNK // 2,
               "shape": "D=100 lut offset_tuning", "repeats": args.repeats,
               "device_call_ms": dev_ms, "mix_kernel_ms": mix_ms, "chain_kernel_ms": chain_ms,
               "device_Msamples_per_s_of_capture": N / dev_ms / 1e3,
               "host_mix_call_ms": host_mix_ms, "host_separate_streams_ms": host_sep_ms,
               "equal_to_separate_streams": bool(equal)}
        print(json.dumps(row), flush=True)
        rows.append(row)
        plain.close()
        mx.close()
        if not equal:
            sys.exit(f"K={K}: the mixing handle's PCM differs from the separate streams'")
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
