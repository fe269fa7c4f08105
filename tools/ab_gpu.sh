#!/bin/bash
# One GPU-box session: parity + fm2b throughput of every A/B build under rx_tools_b200/variants/, then the full
# `-m gpu` suite, the bench lines and the ncu captures on the fastest build that is parity-green.
# Everything lands in gpurun_out/ab/ as it is produced (the session may be cut short).
cd "$(dirname "$0")/.."
OUT=${AB_OUT:-gpurun_out/ab}; export OUT; mkdir -p $OUT
exec > >(tee $OUT/session.log) 2>&1
date; nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,power.draw --format=csv
python -c "import torch; print(torch.cuda.get_device_name(0))"
T0=$SECONDS
FM_TESTS="tests/test_fm_gpu.py tests/test_fuzz_gpu.py"
echo base > $OUT/green.txt
timeout 120 python bench.py --steps 10 --warmup 3 --no-e2e --no-cpu > $OUT/bench_base.json 2> $OUT/bench_base.err; echo "base bench rc=$? t=$((SECONDS-T0))"
for so in rx_tools_b200/variants/librxb200_*.so; do
	v=$(basename $so .so); v=${v#librxb200_}
	timeout 200 env RXB200_LIB=$PWD/$so python -m pytest $FM_TESTS -x -q -m gpu > $OUT/test_$v.log 2>&1; rc=$?
	tail -1 $OUT/test_$v.log
	if [ $rc -eq 0 ]; then echo $v >> $OUT/green.txt; fi
	timeout 120 env RXB200_LIB=$PWD/$so python bench.py --steps 10 --warmup 3 --no-e2e --no-cpu > $OUT/bench_$v.json 2> $OUT/bench_$v.err
	echo "$v tests rc=$rc bench rc=$? t=$((SECONDS-T0))"
done
WIN=$(python - <<'PY'
import json, os
best, bv = "base", 0.0
for v in open(os.environ["OUT"] + "/green.txt").read().split():
    try:
        val = json.loads(open(os.environ["OUT"] + f"/bench_{v}.json").read().strip().splitlines()[-1])["value"]
    except Exception:
        continue
    print(v, val, file=__import__("sys").stderr)
    if val > bv:
        best, bv = v, val
print(best)
PY
)
echo "winner: $WIN"; echo $WIN > $OUT/winner.txt
if [ "$WIN" != base ]; then cp rx_tools_b200/variants/librxb200_$WIN.so rx_tools_b200/librxb200.so; fi
# ---- the winner as the default library: full suite, smoke, bench lines
timeout 300 python -m pytest tests -x -q -m gpu > $OUT/gpu_tests_final.txt 2>&1; echo "full suite rc=$? t=$((SECONDS-T0))"; tail -2 $OUT/gpu_tests_final.txt
timeout 120 python __graft_entry__.py smoke > $OUT/smoke.txt 2>&1; echo "smoke rc=$?"; tail -1 $OUT/smoke.txt
timeout 240 python bench.py > $OUT/bench_fm2b_final.json 2> $OUT/bench_fm2b_final.err; echo "final bench rc=$? t=$((SECONDS-T0))"
# ---- ncu: launch list of the bench command, one full capture of the fused kernel
timeout 240 ncu --metrics gpu__time_duration.sum --clock-control none -c 60 --csv --log-file $OUT/launches_fm2b.csv \
	python bench.py --steps 2 --warmup 1 --no-e2e --no-cpu > $OUT/ncu_launch_run.log 2>&1; echo "ncu launches rc=$? t=$((SECONDS-T0))"
timeout 300 ncu --set full --clock-control none --import-source on -k regex:fm_fused -c 1 -o $OUT/prof_fm2b -f \
	python bench.py --steps 1 --warmup 1 --no-e2e --no-cpu > $OUT/ncu_full_run.log 2>&1; echo "ncu full rc=$? t=$((SECONDS-T0))"
# ---- the other rx_fm shapes on the winner
for w in fm2a fm1 fm5a; do
	timeout 120 python bench.py --workload $w --steps 5 --warmup 3 --no-e2e --no-cpu > $OUT/bench_${w}_final.json 2> $OUT/bench_${w}_final.err; echo "$w rc=$?"
done
# ---- CTA width against the shape (boxcar kernels exist in both widths), front end alone against the full chain
timeout 300 python tools/width_sweep.py > $OUT/width_sweep.txt 2>&1; echo "width sweep rc=$? t=$((SECONDS-T0))"; cat $OUT/width_sweep.txt
date
