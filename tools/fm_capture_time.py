"""Times the rx_fm shell's capture mode (RXB200_CAPTURE_RATE) end to end on the replay device, for two plans:
* the seven NOAA weather channels, 162.400-162.550 MHz, NBFM at the default 24 kHz (c = 1.008 Msps, M = 2);
* 19 FM-band channels under -M wbfm, 88.1-107.9 MHz every 1.1 MHz (c = 1.02 Msps, M = 21, R = 21.42 Msps, T = 673).

Each plan runs the shell on a seeded synthetic capture of --seconds seconds (a short synthetic stretch repeated) and on
one of a single block; the capture's duration over the wall times gives the real-time factor with and without the
shell's start-up (device and library set-up, first launches), which the short run measures (None when the difference
is within the noise).  The wall time includes the replay device loading the capture file and writing every channel's
file.  Prints the GPU's name and power limit, then one JSON line per plan.

    python tools/fm_capture_time.py [--seconds 10]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

import fm_capture as fcp  # noqa: E402

RX_FM = os.path.join(ROOT, "host", "rx_fm_b200")
PLANS = {"noaa7": (["162.4M:162.55M:25k"], [], {}),
         "fm_band_wbfm19": (["88.1M:107.9M:1.1M"], ["-M", "wbfm"], dict(wbfm=1))}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def shell_wall(argv, x, tmp):
    """Wall seconds of one shell run over capture x (written to tmp first, not timed)."""
    cap = os.path.join(tmp, "cap.cs16")
    x.tofile(cap)
    out = os.path.join(tmp, "out")
    t0 = time.perf_counter()
    r = subprocess.run([RX_FM] + argv + ["-d", f"driver=file,path={cap}", out], capture_output=True,
                       env=dict(os.environ, RXB200_CAPTURE_RATE="100000000"))
    wall = time.perf_counter() - t0
    if r.returncode != 0:
        raise SystemExit(r.stderr.decode()[-2000:])
    for f in os.listdir(tmp):
        if f.startswith("out."):
            os.remove(os.path.join(tmp, f))
    return wall


def run(name, seconds):
    fvals, args, kw = PLANS[name]
    p, freqs, pl, offs, taps = fcp.plan_of(fvals, args, kw)
    block = pl.decim * fcp.CHUNK
    piece = fcp.capture(block, pl.capture_rate, offs, 4242, deviation=75000.0 if kw else 2500.0)
    n_blocks = max(2, int(round(seconds * pl.capture_rate / block)))
    x = np.tile(piece, n_blocks)
    argv = [a for v in fvals for a in ("-f", v)] + args
    with tempfile.TemporaryDirectory() as tmp:
        shell_wall(argv, piece, tmp)                           # warm the file cache and the driver once
        short = shell_wall(argv, piece, tmp)
        full = shell_wall(argv, x, tmp)
    dur = n_blocks * block / pl.capture_rate
    return {"plan": name, "channels": len(freqs), "capture_rate": pl.capture_rate, "decim": pl.decim,
            "n_taps": pl.n_taps, "capture_s": round(dur, 3), "wall_s": round(full, 3),
            "one_block_wall_s": round(short, 3), "x_real_time": round(dur / full, 2),
            "x_real_time_after_start_up": (round((dur - block / pl.capture_rate) / (full - short), 2)
                                           if full > short else None)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=10.0)
    a = ap.parse_args()
    subprocess.run(["make", "-C", os.path.join(ROOT, "host"), "-s"], check=True)
    print("GPU:", card())
    for name in PLANS:
        print(json.dumps(run(name, a.seconds)))


if __name__ == "__main__":
    main()
