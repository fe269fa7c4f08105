"""Mints tests/golden/fm_two_stage_golden.json from the unmodified reference (oracle/_ref): for each shape of
tests/fm_two_stage.py -- a wideband capture, channels at arbitrary offsets, a coarse and a fine DDC -- and each channel,
the decimated length of every capture read and the sha256 of the decimated stream (fm_two_stage.two_stage_model over the
library's period-K table and NCO table), then the sha256 of the reference's PCM and its result_len per read when it
demodulates that stream read by read, reads with no output skipped.

    python tests/golden/make_fm_two_stage_golden.py     (needs oracle/_ref and librxb200.so; rewrites the file byte for byte)
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
import fm_ddc  # noqa: E402
import fm_two_stage  # noqa: E402


def _ddc(d):
    return {"decim": int(d[0]), "taps": [int(v) for v in d[1]], "shift": int(d[2])}


def main():
    oracle.build()
    if not oracle.have_ref():
        raise SystemExit("oracle/_ref is not built (the reference sources are needed)")
    ref = oracle.RefFm()
    out = {}
    for name in sorted(fm_two_stage.SHAPES):
        p, rate, K, offs, coarse, fine, x, reads = fm_two_stage.case_input(name)
        chans = []
        for dec in fm_two_stage.decimated_reads(x, rate, K, offs, coarse, fine, reads):
            y, lens = fm_ddc.nonempty(dec)
            pcm, rl, _ = fm_any_chunk.ref_run_seq(ref, p, y, lens, return_chunks=True)
            chans.append({"dec_len": [int(r.size) for r in dec], "dec_sha256": hashlib.sha256(y.tobytes()).hexdigest(),
                          "result_len": [int(v) for v in rl], "sha256": hashlib.sha256(pcm.tobytes()).hexdigest()})
        out[name] = {"params": {k: int(v) for k, v in vars(p).items()}, "capture_rate": int(rate), "n_bins": int(K),
                     "offsets_hz": [int(f) for f in offs], "coarse": _ddc(coarse), "fine": _ddc(fine),
                     "lens_int16": list(reads), "n_int16": int(x.size),
                     "capture_sha256": hashlib.sha256(x.tobytes()).hexdigest(), "channels": chans}
    with open(os.path.join(HERE, "fm_two_stage_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
