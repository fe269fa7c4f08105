"""Mints tests/golden/fm_capture_golden.json from the unmodified reference (oracle/_ref): for each command line of
tests/fm_capture.py -- a capture with a channel at each -f frequency, planned as the rx_fm shell's capture mode plans
it -- the plan, the blocks, and for each channel the sha256 of its decimated stream (fm_ddc.ddc_model over the
library's mixer table and rx_power's capture-mode filter), then the reference's result_len and squelch hits per chain
read and the sha256 of its PCM when it demodulates that stream one block at a time.

    python tests/golden/make_fm_capture_golden.py     (needs oracle/_ref and librxb200.so; rewrites the file byte for byte)
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
import fm_capture  # noqa: E402


def main():
    oracle.build()
    if not oracle.have_ref():
        raise SystemExit("oracle/_ref is not built (the reference sources are needed)")
    ref = oracle.RefFm()
    out = {}
    for name in sorted(fm_capture.SHAPES):
        argv, p, freqs, pl, offs, taps, x = fm_capture.case(name)
        blk = fm_capture.blocks(x.size // 2, pl.decim, fm_capture.min_chunk(p))
        lens = fm_capture.chain_reads(blk, pl.decim)
        chans = []
        for f, dec in zip(freqs, fm_capture.decimated(x, pl, offs, taps)):
            y = dec[:sum(lens)]
            pcm, rl, hits = fm_any_chunk.ref_run_seq(ref, fm_capture.oracle_params(p), y, lens, return_chunks=True)
            chans.append({"freq": int(f), "dec_sha256": hashlib.sha256(y.tobytes()).hexdigest(),
                          "result_len": [int(v) for v in rl], "hits": [int(v) for v in hits],
                          "sha256": hashlib.sha256(pcm.tobytes()).hexdigest()})
        out[name] = {"argv": argv, "params": {k: int(v) for k, v in vars(fm_capture.oracle_params(p)).items()},
                     "centre_hz": pl.centre_hz, "decim": pl.decim, "capture_rate": pl.capture_rate,
                     "n_taps": pl.n_taps, "offsets": offs, "blocks": blk, "n_int16": int(x.size),
                     "capture_sha256": hashlib.sha256(x.tobytes()).hexdigest(), "channels": chans}
    with open(os.path.join(HERE, "fm_capture_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
