#!/usr/bin/env bash
# Round-2 evidence in one gpurun call: GPU tests, the three bench lines, sanitizer passes, the ncu launch list and the
# --set full captures (train step, DS-CNN forward).  Summaries are made from the .ncu-rep files afterwards (tools/ncu_summary.py).
set -u
O=gpurun_out/${1:-ev}; mkdir -p $O
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,power.limit --format=csv > $O/smi.txt 2>&1; nproc >> $O/smi.txt
timeout 1500 python -m pytest tests -m gpu -q > $O/pytest_gpu.txt 2>&1; echo "pytest rc=$?" | tee -a $O/pytest_gpu.txt; tail -4 $O/pytest_gpu.txt
timeout 600 python bench.py > $O/bench.json 2> $O/bench.err; echo "bench rc=$?"; cut -c1-400 $O/bench.json
timeout 300 python bench.py --workload dscnn --steps 100 --warmup 10 > $O/bench_dscnn.json 2> $O/bench_dscnn.err; echo "dscnn rc=$?"; cut -c1-300 $O/bench_dscnn.json
TCR_DSCNN_TC=0 timeout 300 python bench.py --workload dscnn --steps 100 --warmup 10 > $O/bench_dscnn_fma.json 2> $O/bench_dscnn_fma.err; echo "dscnn fma rc=$?"; cut -c1-300 $O/bench_dscnn_fma.json
timeout 600 python bench.py --impl reference --steps 3 --warmup 1 > $O/bench_ref.json 2> $O/bench_ref.err; echo "ref rc=$?"; cut -c1-300 $O/bench_ref.json
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 150 --csv --log-file $O/launches.csv python bench.py --steps 2 --warmup 3 --no-cpu-baseline --no-e2e --no-extra > $O/under_ncu.log 2>&1; echo "launch list rc=$?"
timeout 900 ncu --set full --clock-control none --import-source on --kernel-name-base demangled -k regex:tcr:: -s 12 -c 14 -o $O/full python bench.py --steps 2 --warmup 3 --no-cpu-baseline --no-e2e --no-extra > $O/ncu_full.log 2>&1; echo "ncu full rc=$?"
timeout 600 ncu --set full --clock-control none --import-source on --kernel-name-base demangled -k regex:dscnn -s 12 -c 6 -o $O/dscnn python bench.py --workload dscnn --steps 3 --warmup 3 > $O/ncu_dscnn.log 2>&1; echo "ncu dscnn rc=$?"
TCR_DSCNN_TC=0 timeout 600 ncu --metrics gpu__time_duration.sum,sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active,sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active --clock-control none --kernel-name-base demangled -k regex:dscnn -s 12 -c 6 --csv --log-file $O/dscnn_fma.csv python bench.py --workload dscnn --steps 3 --warmup 3 > $O/ncu_dscnn_fma.log 2>&1; echo "ncu dscnn fma rc=$?"
for tool in memcheck racecheck synccheck; do
  timeout 900 compute-sanitizer --tool $tool --error-exitcode 7 python -c "
import sys; sys.path.insert(0,'tests'); sys.path.insert(0,'.')
from tcr_harness import TorchBackend
from parity_cases import run_case
from test_dscnn import _run
b = TorchBackend()
print(run_case(b, model='TCResNet8', wm=1.0, n=5, keep=0.5))
print(_run(b, 'S', 49, 40, 3))
" > $O/$tool.txt 2>&1 ; echo "$tool rc=$?" | tee -a $O/$tool.txt
  grep -E "RACECHECK SUMMARY|ERROR SUMMARY|hazard|Barrier error" $O/$tool.txt | head -6
done
