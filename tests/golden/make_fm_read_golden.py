"""Mints tests/golden/fm_read_golden.json from the unmodified reference (oracle/_ref): for each case of tests/fm_read.py
(golden_cases) -- the fm2b shape over reads of 2044 complex samples, of 1021:333:4093 and of 131071, and read sequences
that meet every residue of the read length for several pass counts -- the sha256 of the reference's PCM and its
result_len per read.  The fm2b parameters fm_read spells out are derived by the reference's own main() and must match.

    python tests/golden/make_fm_read_golden.py        (needs oracle/_ref; rewrites the file byte for byte)
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
import fm_read  # noqa: E402


def main():
    oracle.build()
    if not oracle.have_ref():
        raise SystemExit("oracle/_ref is not built (the reference sources are needed)")
    ref = oracle.RefFm()
    derived = ref.derive(wbfm=1, rate_s=300000, rate_r=48000, use_F=1, comp_fir_size=9)[0]
    assert derived == fm_read.FM2B, (derived, fm_read.FM2B)
    out = {}
    for name, (p, x, lens) in sorted(fm_read.golden_cases().items()):
        pcm, rl, _ = fm_any_chunk.ref_run_seq(ref, p, x, lens, return_chunks=True)
        out[name] = {"params": {k: int(v) for k, v in vars(p).items()}, "lens_int16": [int(v) for v in lens],
                     "n_int16": int(x.size), "result_len": [int(v) for v in rl],
                     "sha256": hashlib.sha256(pcm.tobytes()).hexdigest()}
    with open(os.path.join(HERE, "fm_read_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
