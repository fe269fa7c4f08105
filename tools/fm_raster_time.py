"""Times raster mixing handles (rxb200_fm_mix_create_raster) against decimating ones (rxb200_fm_mix_create_ddc) on one
second of a 19.2 Msps capture: C = 8, 64, 256 and 768 NBFM channels of the 768-bin (25 kHz) raster, M = 64, with the
257-tap Q15 low-pass of tools/fm_ddc_time.py and with the rx_power shell's channel filter (rxb200_ddc_lowpass, 2049
taps), into a D = 12 lut chain (300 kHz -> 25 kHz).  A decimating handle cannot mix by R/2, so at C = 768 its Nyquist-bin
channel is mixed by 0 instead (the same work).

For each handle: the front stage's kernels (torch.profiler over one device call: raster_branch_kernel and
raster_dft_kernel summed per kernel, or fm_ddc_kernel), the front stage's device time (CUDA events, FmMix.mix_ms), the
whole device call on a device-resident capture and the host call from a pinned capture into pinned PCM (host clock
around synchronised calls, best of --reps), and the DFT's achieved FP64 rate (2 x frames x 2K x 2C useful flops).  The
first line names the card and its power limit.  Prints one JSON line per configuration.

    python tools/fm_raster_time.py [--reps 3] [--c 8,64,256,768] [--taps 257,2049] [--kinds raster,ddc]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from rx_tools_b200 import _lib, fm, power, synth  # noqa: E402

RATE, K, M, D = 19_200_000, 768, 64, 12
CHUNK = 2 * M * 2048


def lowpass(n_taps, cutoff):
    j = np.arange(n_taps) - (n_taps - 1) / 2.0
    h = np.sinc(2.0 * cutoff * j) * np.hamming(n_taps)
    return np.round(h / h.sum() * 32768.0).astype(np.int32)


def taps_for(n_taps):
    return lowpass(n_taps, 12500 / RATE) if n_taps == 257 else power.ddc_lowpass(M, n_taps, 15)


def capture(n_complex):
    x = np.zeros(2 * n_complex, np.int64)
    for k in range(8):                                        # a few live channels; the rest is noise
        x += synth.fm_iq(n_complex, fs=float(RATE), deviation_hz=2500.0, tones=[(400.0 + 50 * k, 0.8)],
                         amplitude=2000.0, noise_lsb=0, seed=k, center_hz=25000.0 * (k - 4)).astype(np.int64)
    x += np.random.default_rng(1).integers(-8, 9, size=x.size)
    return np.clip(x, -32768, 32767).astype(np.int16)


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return min(ts)


def kernel_ms(fn, names):
    """Device time of each named kernel over one call of fn, summed over its launches (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names}
    for e in prof.events():
        for n in names:
            if n in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
                out[n] += e.device_time_total / 1e3
    return out


def run(kind, c, n_taps, x_pin, d_x, reps):
    bins = [(j - c // 2) % K for j in range(c)]
    nbfm = fm.FmParams(mode=fm.MODE_FM, downsample=D, custom_atan=fm.ATAN_LUT, rate_out=25000, offset_tuning=1)
    taps = taps_for(n_taps)
    if kind == "raster":
        mx = fm.FmMix(nbfm, ddc=(M, taps, 30), raster=(K, bins))
    else:
        # a table mixer refuses +-R/2, so the Nyquist bin's channel (C = 768) takes bin 0's offset again: same work
        offs = [(b if 2 * b < K else b - K) * (RATE // K) if 2 * b != K else 0 for b in bins]
        mx = fm.FmMix(nbfm, RATE, offs, ddc=(M, taps, 15))
    n = x_pin.numel()
    cap = mx.max_output(n, CHUNK) + 8
    d_out = torch.empty((c, cap), dtype=torch.int16, device="cuda")
    h_out = torch.empty((c, cap), dtype=torch.int16).pin_memory()
    n_pcm = C.c_size_t(0)

    def device_call():
        mx.reset()
        mx.process_device(d_x.data_ptr(), n, CHUNK, d_out.data_ptr(), cap, sync=True)

    def host_call():
        mx.reset()
        _lib.check(_lib.lib().rxb200_fm_mix_process(mx._h, x_pin.data_ptr(), n, CHUNK, h_out.data_ptr(), cap,
                                                    C.byref(n_pcm), None))

    dev_ms = timed(device_call, reps)
    front_ms = mx.mix_ms()
    host_ms = timed(host_call, reps)
    names = ["raster_branch_kernel", "raster_dft_kernel"] if kind == "raster" else ["fm_ddc_kernel"]
    ks = kernel_ms(device_call, names)
    out = dict(kind=kind, c=c, taps=n_taps, capture_s=n / 2 / RATE, decim=M, pcm_per_channel=int(n_pcm.value),
               front_ms=round(front_ms, 3), device_call_ms=round(dev_ms, 3), host_call_ms=round(host_ms, 3),
               **{k.replace("_kernel", "_ms"): round(v, 3) for k, v in ks.items()})
    if kind == "raster":
        frames = n // 2 // M
        out["dft_tflops"] = round(2.0 * frames * 2 * K * 2 * c / (ks["raster_dft_kernel"] * 1e-3) / 1e12, 2)
    mx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--c", default="8,64,256,768")
    ap.add_argument("--kinds", default="raster,ddc")
    ap.add_argument("--taps", default="257,2049")
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip().splitlines()[:1])), flush=True)
    x = capture(RATE)                                         # one second
    x_pin = torch.from_numpy(x).pin_memory()
    d_x = x_pin.cuda()
    for n_taps in [int(v) for v in a.taps.split(",")]:
        for c in [int(v) for v in a.c.split(",")]:
            for kind in a.kinds.split(","):
                try:
                    print(json.dumps(run(kind, c, n_taps, x_pin, d_x, a.reps)), flush=True)
                except _lib.Rxb200Error as e:
                    print(json.dumps(dict(kind=kind, c=c, taps=n_taps, not_measured=str(e))), flush=True)
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
