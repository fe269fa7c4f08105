"""Times decimating mixing handles (rxb200_fm_mix_create_ddc) on one second of a 19.2 Msps capture: K = 8, 64 and 256
NBFM channels on a 25 kHz raster, M = 64 with a 257-tap Q15 low-pass into a D = 12 lut chain (300 kHz -> 25 kHz),
against the plain mixing handle on the same capture with the chain's boxcar alone at D = 768 (the same channel rate).

For each handle: fm_ddc_kernel / fm_mix_kernel device time (CUDA events, FmMix.mix_ms), the whole device call on a
device-resident capture, and the host call from a pinned capture buffer into a pinned PCM buffer (host clock around
synchronised calls).  Prints one JSON line per configuration.

    python tools/fm_ddc_time.py [--reps 3] [--k 8,64,256]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from rx_tools_b200 import _lib, fm, synth  # noqa: E402

RATE, M, T, D = 19_200_000, 64, 257, 12
CHUNK = 2 * M * 2048                    # 262144 int16: the plain handle's largest chunk; 4096 decimated int16


def lowpass(n_taps, cutoff):
    j = np.arange(n_taps) - (n_taps - 1) / 2.0
    h = np.sinc(2.0 * cutoff * j) * np.hamming(n_taps)
    return np.round(h / h.sum() * 32768.0).astype(np.int32)


def capture(n_complex, offsets):
    x = np.zeros(2 * n_complex, np.int64)
    for k, f in enumerate(offsets[:8]):                      # a few live channels; the rest is noise
        x += synth.fm_iq(n_complex, fs=float(RATE), deviation_hz=2500.0, tones=[(400.0 + 50 * k, 0.8)],
                         amplitude=2000.0, noise_lsb=0, seed=k, center_hz=float(f)).astype(np.int64)
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


def run(kind, k, x_pin, d_x, reps):
    offs = [25000 * (j - k // 2) for j in range(k)]
    nbfm = fm.FmParams(mode=fm.MODE_FM, downsample=D if kind == "ddc" else M * D, custom_atan=fm.ATAN_LUT,
                       rate_out=25000, offset_tuning=1)
    ddc = (M, lowpass(T, 12500 / RATE), 15) if kind == "ddc" else None
    mx = fm.FmMix(nbfm, RATE, offs, ddc=ddc)
    n = x_pin.numel()
    cap = mx.max_output(n, CHUNK) + 8
    d_out = torch.empty((k, cap), dtype=torch.int16, device="cuda")
    h_out = torch.empty((k, cap), dtype=torch.int16).pin_memory()
    n_pcm = C.c_size_t(0)

    def device_call():
        mx.reset()
        mx.process_device(d_x.data_ptr(), n, CHUNK, d_out.data_ptr(), cap, sync=True)

    def host_call():
        mx.reset()
        _lib.check(_lib.lib().rxb200_fm_mix_process(mx._h, x_pin.data_ptr(), n, CHUNK, h_out.data_ptr(), cap,
                                                    C.byref(n_pcm), None))

    dev_ms = timed(device_call, reps)
    kern_ms = mx.mix_ms()
    host_ms = timed(host_call, reps)
    out = dict(kind=kind, k=k, capture_s=n / 2 / RATE, decim=M if ddc else 1, taps=T if ddc else 0,
               chain_downsample=nbfm.downsample, pcm_per_channel=int(n_pcm.value),
               mix_or_ddc_kernel_ms=round(kern_ms, 3), device_call_ms=round(dev_ms, 3), host_call_ms=round(host_ms, 3))
    mx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--k", default="8,64,256")
    a = ap.parse_args()
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(0))), flush=True)
    n_complex = RATE                                          # one second
    x = capture(n_complex, [25000 * (j - 4) for j in range(8)])
    x_pin = torch.from_numpy(x).pin_memory()
    d_x = x_pin.cuda()
    for k in [int(v) for v in a.k.split(",")]:
        for kind in ("ddc", "mix"):
            try:
                print(json.dumps(run(kind, k, x_pin, d_x, a.reps)), flush=True)
            except _lib.Rxb200Error as e:
                print(json.dumps(dict(kind=kind, k=k, not_measured=str(e))), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
