#!/bin/bash
# The TMA input ring of the row front end (fm_rows.cuh) on one GPU session:
#   probe   tools/experiments/load_probe.bin (build it first) and one torch read of the same 1 GiB, for scale
#   tests   tests/test_fm_gpu.py on the default build
#   sweep   bench.py fm2b on the parent build and on CTA-shape variants (tools/build_variants.sh; RXB200_LIB),
#           ROUNDS rounds alternating the builds; each build's fm2b PCM is dumped once and compared byte for byte
#   tools/rows_ring_gpu.sh [out dir] [builds...]        builds: names under rx_tools_b200/variants/, "default" = the tree's
cd "$(dirname "$0")/.."
OUT=${1:-${TMPDIR:-/tmp}/rows_ring}; shift
BUILDS=${*:-"default"}
ROUNDS=${ROUNDS:-2}
mkdir -p $OUT
exec > >(tee $OUT/session.log) 2>&1
date; nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv
T0=$SECONDS
if [ -x tools/experiments/load_probe.bin ] && [ -z "$NO_PROBE" ]; then
	timeout 120 tools/experiments/load_probe.bin > $OUT/load_probe.txt 2>&1; echo "probe rc=$?"; cat $OUT/load_probe.txt
	timeout 120 python - <<'PY'
import torch
x = torch.empty(1 << 28, dtype=torch.int32, device="cuda").random_()
for _ in range(3): x.sum()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(10): x.sum()
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / 10
print("torch x.sum() int32 1 GiB                    %8.3f ms  %7.1f GB/s" % (ms, (1 << 30) / (ms * 1e6)))
PY
fi
if [ -z "$NO_TESTS" ]; then
	timeout 600 python -m pytest tests/test_fm_gpu.py -x -q -m gpu > $OUT/fm_tests.txt 2>&1; echo "test_fm_gpu rc=$? t=$((SECONDS-T0))"; tail -3 $OUT/fm_tests.txt
fi
lib_of() { [ "$1" = default ] && echo "$PWD/rx_tools_b200/librxb200.so" || echo "$PWD/rx_tools_b200/variants/librxb200_$1.so"; }
for r in $(seq 1 $ROUNDS); do
	for b in $BUILDS; do
		D=""; [ $r = 1 ] && D="--dump-outputs $OUT/dump_$b"
		RXB200_LIB=$(lib_of $b) timeout 300 python bench.py --workload fm2b --no-extras --no-cpu --steps 10 --warmup 3 $D \
			> $OUT/bench_${b}_$r.json 2> $OUT/bench_${b}_$r.err
		rc=$?; echo "$b round $r rc=$rc t=$((SECONDS-T0))"; [ $rc = 0 ] || tail -4 $OUT/bench_${b}_$r.err
	done
done
python - "$OUT" $BUILDS <<'PY'
import json, sys, os, hashlib
out, builds = sys.argv[1], sys.argv[2:]
for b in builds:
    vals = []
    for f in sorted(x for x in os.listdir(out) if x.startswith("bench_%s_" % b) and x.endswith(".json")):
        try:
            d = json.loads(open(os.path.join(out, f)).read().strip().splitlines()[-1])
            vals.append("%.0f (kernel %.3f ms, clocks %s)" % (d["value"], (d.get("roofline") or {}).get("kernel_ms", float("nan")), d.get("clocks")))
        except Exception as e:
            vals.append("no line: %s" % e)
    p = os.path.join(out, "dump_%s" % b, "pcm.npy")
    h = hashlib.sha256(open(p, "rb").read()).hexdigest()[:16] if os.path.exists(p) else "-"
    print("%-10s pcm %s  %s" % (b, h, " | ".join(vals)))
PY
rm -rf $OUT/dump_*                # the hashes above are the record; the PCM itself is too large to keep
date
