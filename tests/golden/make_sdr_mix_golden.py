"""Writes tests/golden/sdr_mix_golden.json: the SHA-256 of every named shape of tests/sdr_mix.py through the numpy model
(the rule of include/rxb200.h, "rx_sdr channels of one capture") in every recorded format, with the capture's hash.

    python tests/golden/make_sdr_mix_golden.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import sdr_mix as sm  # noqa: E402


def main():
    out = {}
    for name in sm.SHAPES:
        x = sm.case_capture(name)
        y, _ = sm.model(name, x)
        out[name] = {"input_sha256": sm.digest(x), "shape": list(y.shape)}
        for fmt in sm.FORMATS:
            out[name][fmt] = sm.digest(sm.convert(y, fmt))
    with open(os.path.join(HERE, "sdr_mix_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
