"""Mints tests/golden/power_tiles_golden.json from the unmodified reference (oracle/_ref): for each named shape of
tests/power_tiles.py -- a sweep plan cut into tiles, one burst per tile -- the tiling, the sha256 of each burst and of
the model's hop buffers (the tiles side by side, [P][n_hops][buf_len]), then the sha256 of the reference scanner()'s avg
over them, its samples, and the sha256 of the CSV the reference's csv_dbm() writes.

    python tests/golden/make_power_tiles_golden.py     (needs oracle/_ref and librxb200.so; rewrites the file byte for byte)
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
import power_tiles  # noqa: E402

TSTR = "2026-01-01, 00:00:00"


def main():
    oracle.build()
    if not oracle.have_ref():
        raise SystemExit("oracle/_ref is not built (the reference sources are needed)")
    ref = oracle.RefPower()
    out = {}
    for name in sorted(power_tiles.SHAPES):
        s = power_tiles.SHAPES[name]
        plan, win, tl, tiles, offs, dd, bs = power_tiles.case_input(name)
        _, hb = power_tiles.tile_buffers(name)
        rp = ref.setup(s["freq"], s["crop"], s["boxcar"], s["fir"], s["peak"], s["window"])
        assert (rp.tune_count, rp.bin_e, rp.buf_len) == (plan.n_hops, plan.bin_e, plan.buf_len), name
        avg, smp = ref.scan(hb, hb.shape[0])
        with tempfile.TemporaryDirectory() as td:
            csv = ref.csv(os.path.join(td, "out.csv"), TSTR)
        out[name] = {"plan": [plan.n_hops, plan.bin_e, plan.buf_len, plan.downsample, plan.downsample_passes],
                     "tiling": [tl.n_tiles, tl.hops_per_tile, tl.decim, tl.capture_rate, int(dd[1].size), int(dd[2])],
                     "burst_sha256": [power_mix.digest(b) for b in bs], "bufs_sha256": power_mix.digest(hb),
                     "avg_sha256": power_mix.digest(avg), "samples": [int(v) for v in smp],
                     "csv_sha256": hashlib.sha256(csv.encode()).hexdigest()}
    with open(os.path.join(HERE, "power_tiles_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
