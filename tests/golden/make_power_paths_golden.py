"""Regenerate tests/golden/power_paths_golden.json from the UNMODIFIED reference (oracle/_ref).

The named rx_power command lines of tests/power_paths.py (GOLDEN_CASES): a /1400 boxcar at bin_e 1, a /311 boxcar at
bin_e 7, -F 9 with 8 and 10 passes at bin_e 1, a planner shape at the shared-memory limit, bin_e 15 (sine and window
tables in global memory), peak hold over full-scale input, rms_power, ...  Every entry keeps the plan the reference
chose, the sha256 of the reference's avg rows and its samples counts.
Run: python tests/golden/make_power_paths_golden.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import oracle  # noqa: E402
import power_paths  # noqa: E402
from rx_tools_b200.synth import digest  # noqa: E402

OUT = os.path.join(HERE, "power_paths_golden.json")


def main():
    oracle.build()
    if not oracle.have_ref():
        sys.exit("oracle/_ref is not built: the golden values come from the reference itself")
    ref = oracle.RefPower()
    out = {}
    for name, c in sorted(power_paths.GOLDEN_CASES.items()):
        plan = ref.setup(c["freq"], c["crop"], c["boxcar"], c["fir"], c["peak"], c["window"])
        ours = power_paths.golden_plan(c)
        got = [plan.tune_count, plan.bin_e, plan.buf_len, plan.downsample, plan.downsample_passes]
        assert got == [ours.n_hops, ours.bin_e, ours.buf_len, ours.downsample, ours.downsample_passes], name
        avg, smp = ref.scan(power_paths.golden_input(c, ours), c["n_pass"])
        out[name] = dict(plan=got, avg_sha256=digest(avg), samples=[int(s) for s in smp])
        print(name, "plan", got)
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", len(out), "entries to", os.path.basename(OUT))


if __name__ == "__main__":
    main()
