"""Regenerate tests/golden/power_decim_big_golden.json from the UNMODIFIED reference (oracle/_ref).

rx_power -F shapes whose hop buffer (2 N 2^P int16) is larger than shared memory: the planner's own shapes
(frequency_range(), src/rtl_power.c:431-543) for bins of 50, 40, 10 and 1 Hz, each with -F 0 and -F 9.  Every
entry keeps the command-line arguments, the seed of its uniform +-3000 input, the plan the reference chose, the
sha256 of the reference's avg rows and its samples counts.  Run: python tests/golden/make_power_decim_big_golden.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import oracle  # noqa: E402
from rx_tools_b200.synth import digest  # noqa: E402

OUT = os.path.join(HERE, "power_decim_big_golden.json")

# (name, -f argument, -F argument, window, peak hold, passes of accumulation, input seed)
SHAPES = [
    ("f50_fir0", "100M:100.5M:50", 0, "hamming", 0, 2, 501),
    ("f50_fir9", "100M:100.5M:50", 9, "blackman", 0, 2, 502),
    ("f40_fir0", "100M:100.1M:40", 0, "hann-poisson", 0, 2, 401),
    ("f40_fir9_peak", "100M:100.1M:40", 9, "hamming", 1, 3, 402),
    ("f10_fir0", "100M:100.1M:10", 0, "blackman", 0, 2, 101),
    ("f10_fir9", "100M:100.1M:10", 9, "hann-poisson", 0, 2, 102),
    ("f1_fir0", "100M:100.01M:1", 0, "hamming", 0, 2, 11),
    ("f1_fir9", "100M:100.01M:1", 9, "blackman", 0, 2, 12),
]


def hop_input(seed: int, n_pass: int, n_hops: int, buf_len: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    return rng.integers(-3000, 3001, size=(n_pass, n_hops, buf_len), dtype=np.int32).astype(np.int16)


def main():
    oracle.build()
    if not oracle.have_ref():
        sys.exit("oracle/_ref is not built: the golden values come from the reference itself")
    ref = oracle.RefPower()
    out = {}
    for name, freq, fir, window, peak, n_pass, seed in SHAPES:
        plan = ref.setup(freq, 0.0, 0, fir, peak, window)
        x = hop_input(seed, n_pass, plan.tune_count, plan.buf_len)
        avg, smp = ref.scan(x, n_pass)
        out[name] = dict(freq=freq, fir=fir, window=window, peak_hold=peak, n_pass=n_pass, seed=seed,
                         n_hops=plan.tune_count, bin_e=plan.bin_e, buf_len=plan.buf_len, downsample=plan.downsample,
                         downsample_passes=plan.downsample_passes, rate=plan.rate,
                         avg_sha256=digest(avg), samples=[int(s) for s in smp])
        print(name, "bin_e", plan.bin_e, "passes", plan.downsample_passes, "buf_len", plan.buf_len)
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", len(out), "entries to", os.path.basename(OUT))


if __name__ == "__main__":
    main()
