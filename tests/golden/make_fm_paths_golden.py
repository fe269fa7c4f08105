"""Mints tests/golden/fm_paths_golden.json from the unmodified reference (oracle/_ref): for each named edge case of
tests/fm_paths.py (golden_cases) the sha256 of the reference's PCM and its result_len per chunk.  The three
`rx_fm -M wbfm ... -c <us>` cases are derived by the reference's own main() + optimal_settings() and must equal the
parameters fm_paths states for them.

    python tests/golden/make_fm_paths_golden.py        (needs oracle/_ref; rewrites the file byte for byte)
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.dirname(HERE)]

import oracle  # noqa: E402
import fm_paths  # noqa: E402

# name -> the reference command line's numbers (-s, -r, -c); every case is -M wbfm -F 9
CLI = {"cli_s300k_F9_r48k_c2000": (300_000, 48_000, 2000),
       "cli_s1200k_F9_r48k_c450": (1_200_000, 48_000, 450),
       "cli_s1200k_F9_c500": (1_200_000, 0, 500)}


def main():
    oracle.build()
    if not oracle.have_ref():
        raise SystemExit("oracle/_ref is not built (the reference sources are needed)")
    ref = oracle.RefFm()
    out = {}
    for name, (p, chunk, x) in sorted(fm_paths.golden_cases().items()):
        if name in CLI:
            s, r, tc = CLI[name]
            derived = ref.derive(rate_s=s, rate_r=r, use_F=1, comp_fir_size=9, wbfm=1, time_constant_us=tc)[0]
            assert derived == p, (name, derived, p)
        pcm, lens, _ = ref.run(p, x, chunk, return_chunks=True)
        out[name] = {"params": {k: int(v) for k, v in vars(p).items()}, "chunk_int16": int(chunk), "n_int16": int(x.size),
                     "result_len": [int(v) for v in lens], "sha256": hashlib.sha256(pcm.tobytes()).hexdigest()}
    with open(os.path.join(HERE, "fm_paths_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
