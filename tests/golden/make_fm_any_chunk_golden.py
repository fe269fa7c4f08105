"""Mints tests/golden/fm_any_chunk_golden.json from the unmodified reference (oracle/_ref): for each case of
tests/fm_any_chunk.py (golden_cases) -- the fm1, fm2a and fm5a shapes at chunks of 131071 / 131069 complex samples and
one ragged chunk sequence per mode -- the sha256 of the reference's PCM and its result_len per chunk.  The command-line
parameters fm_any_chunk spells out are derived by the reference's own main() + optimal_settings() and must match.

    python tests/golden/make_fm_any_chunk_golden.py        (needs oracle/_ref; rewrites the file byte for byte)
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


def main():
    oracle.build()
    if not oracle.have_ref():
        raise SystemExit("oracle/_ref is not built (the reference sources are needed)")
    ref = oracle.RefFm()
    for name, (p, cli) in fm_any_chunk.CLI.items():
        derived = ref.derive(**cli)[0]
        assert derived == p, (name, derived, p)
    out = {}
    for name, (p, x, lens) in sorted(fm_any_chunk.golden_cases().items()):
        pcm, rl, _ = fm_any_chunk.ref_run_seq(ref, p, x, lens, return_chunks=True)
        out[name] = {"params": {k: int(v) for k, v in vars(p).items()}, "lens_int16": [int(v) for v in lens],
                     "n_int16": int(x.size), "result_len": [int(v) for v in rl],
                     "sha256": hashlib.sha256(pcm.tobytes()).hexdigest()}
    with open(os.path.join(HERE, "fm_any_chunk_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
