"""Mints tests/golden/power_mix_golden.json from the unmodified reference (oracle/_ref): for each named shape of
tests/power_mix.py -- a sweep plan in capture mode, a wideband capture of whole passes -- the sha256 of the model's hop
buffers (power_mix.Model over the library's NCO table), then the sha256 of the reference scanner()'s avg over them, its
samples, and the sha256 of the CSV the reference's csv_dbm() writes.

    python tests/golden/make_power_mix_golden.py     (needs oracle/_ref and librxb200.so; rewrites the file byte for byte)
"""
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

import hashlib  # noqa: E402

import oracle  # noqa: E402
import power_mix  # noqa: E402

TSTR = "2026-01-01, 00:00:00"


def main():
    oracle.build()
    if not oracle.have_ref():
        raise SystemExit("oracle/_ref is not built (the reference sources are needed)")
    ref = oracle.RefPower()
    out = {}
    for name in sorted(power_mix.SHAPES):
        c = power_mix.SHAPES[name]
        plan, win, R, offs, dd, x = power_mix.case_input(name)
        hb = power_mix.Model(R, offs, dd, plan.buf_len).hop_buffers(x)
        rp = ref.setup(c["freq"], c["crop"], c["boxcar"], c["fir"], c["peak"], c["window"])
        assert (rp.tune_count, rp.bin_e, rp.buf_len) == (plan.n_hops, plan.bin_e, plan.buf_len), name
        avg, smp = ref.scan(hb, hb.shape[0])
        with tempfile.TemporaryDirectory() as td:
            csv = ref.csv(os.path.join(td, "out.csv"), TSTR)
        out[name] = {"plan": [plan.n_hops, plan.bin_e, plan.buf_len, plan.downsample, plan.downsample_passes],
                     "capture_rate": int(R), "decim": int(dd[0]), "n_taps": int(dd[1].size), "shift": int(dd[2]),
                     "capture_sha256": power_mix.digest(x), "bufs_sha256": power_mix.digest(hb),
                     "avg_sha256": power_mix.digest(avg), "samples": [int(v) for v in smp],
                     "csv_sha256": hashlib.sha256(csv.encode()).hexdigest()}
    with open(os.path.join(HERE, "power_mix_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
