#!/bin/bash
# The row front end's TMA ring, final session: the `-m gpu` suite and smoke() on the tree's build, fm2b PCM of the
# parent build (rx_tools_b200/variants/librxb200_base.so) and the tree's build compared byte for byte, then the full
# bench.py line three times per build, alternating.
cd "$(dirname "$0")/.."
OUT=${1:-${TMPDIR:-/tmp}/rows_ring_final}; mkdir -p $OUT
exec > >(tee $OUT/session.log) 2>&1
date; nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv
T0=$SECONDS
timeout 900 python -m pytest tests -q -m gpu > $OUT/gpu_tests.txt 2>&1; echo "gpu suite rc=$? t=$((SECONDS-T0))"; tail -4 $OUT/gpu_tests.txt
timeout 120 python __graft_entry__.py smoke > $OUT/smoke.txt 2>&1; echo "smoke rc=$?"; tail -1 $OUT/smoke.txt
BASE=$PWD/rx_tools_b200/variants/librxb200_base.so NEW=$PWD/rx_tools_b200/librxb200.so
for b in base new; do
	L=$BASE; [ $b = new ] && L=$NEW
	RXB200_LIB=$L timeout 300 python bench.py --workload fm2b --no-extras --no-cpu --steps 3 --warmup 1 --dump-outputs $OUT/dump_$b > /dev/null 2> $OUT/dump_$b.err
	echo "dump $b rc=$?"
done
cmp $OUT/dump_base/pcm.npy $OUT/dump_new/pcm.npy && echo "fm2b pcm.npy identical ($(sha256sum < $OUT/dump_new/pcm.npy | cut -c1-16))"
rm -rf $OUT/dump_base $OUT/dump_new
for r in 1 2 3; do
	for b in base new; do
		L=$BASE; [ $b = new ] && L=$NEW
		RXB200_LIB=$L timeout 400 python bench.py --steps 10 --warmup 3 > $OUT/bench_${b}_$r.json 2> $OUT/bench_${b}_$r.err
		echo "bench $b $r rc=$? t=$((SECONDS-T0))"
	done
done
python - "$OUT" <<'PY'
import json, sys, os
out = sys.argv[1]
for b in ("base", "new"):
    for r in (1, 2, 3):
        try:
            d = json.loads(open(os.path.join(out, "bench_%s_%d.json" % (b, r))).read().strip().splitlines()[-1])
            ex = d.get("extra") or {}
            print("%-4s %d fm2b %.0f kernel %.3f ms clocks %s | fm2a %.0f fm5a %.0f power4 %.0f" % (
                b, r, d["value"], d["roofline"]["kernel_ms"], d.get("clocks"),
                ex["fm2a"]["value"], ex["fm5a"]["value"], ex["power4"]["value"]))
        except Exception as e:
            print(b, r, "no line:", e)
PY
date
