"""Mints tests/golden/fm_mix_golden.json from the unmodified reference (oracle/_ref): for each shape of tests/fm_mix.py
-- a wideband capture with a channel at each offset -- and each channel, the sha256 of the reference's PCM and its
result_len per read when it demodulates the capture mixed down by that channel's offset (fm_mix.mix_model over the
library's table), read by read over fm_mix.READS.

    python tests/golden/make_fm_mix_golden.py        (needs oracle/_ref and librxb200.so; rewrites the file byte for byte)
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

import oracle  # noqa: E402
import fm_any_chunk  # noqa: E402
import fm_mix  # noqa: E402
from rx_tools_b200 import fm  # noqa: E402


def main():
    oracle.build()
    if not oracle.have_ref():
        raise SystemExit("oracle/_ref is not built (the reference sources are needed)")
    ref = oracle.RefFm()
    out = {}
    for name in sorted(fm_mix.SHAPES):
        p, rate, offs, x = fm_mix.case_input(name)
        chans = []
        for f in offs:
            y = fm_mix.mix_model(x, fm.mix_table(rate, f))
            pcm, rl, _ = fm_any_chunk.ref_run_seq(ref, p, y, fm_mix.READS, return_chunks=True)
            chans.append({"offset_hz": int(f), "result_len": [int(v) for v in rl],
                          "sha256": hashlib.sha256(pcm.tobytes()).hexdigest()})
        out[name] = {"params": {k: int(v) for k, v in vars(p).items()}, "capture_rate": int(rate),
                     "lens_int16": list(fm_mix.READS), "n_int16": int(x.size),
                     "capture_sha256": hashlib.sha256(x.tobytes()).hexdigest(), "channels": chans}
    with open(os.path.join(HERE, "fm_mix_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
