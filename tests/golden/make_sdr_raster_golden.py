"""Writes tests/golden/sdr_raster_golden.json: the SHA-256 of every named shape of tests/sdr_raster.py through the
model (the raster rule of include/rxb200.h, "raster mixing handles", then rx_sdr's conversion of the int16) in every
recorded format, with the capture's hash.

    python tests/golden/make_sdr_raster_golden.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import sdr_raster as sr  # noqa: E402


def main():
    out = {}
    for name in sr.SHAPES:
        x = sr.case_capture(name)
        y, _ = sr.model(name, x)
        out[name] = {"input_sha256": sr.digest(x), "shape": list(y.shape)}
        for fmt in sr.FORMATS:
            out[name][fmt] = sr.digest(sr.convert(y, fmt))
    with open(os.path.join(HERE, "sdr_raster_golden.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
