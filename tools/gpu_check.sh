#!/usr/bin/env bash
# One gpurun call: guarded smoke -> GPU parity tests -> compute-sanitizer on a tiny step -> bench -> ncu launch list.
# Everything lands in gpurun_out/ (merged back by gpurun).  Usage: tools/gpu_check.sh [quick|full]
set -u
MODE=${1:-full}
mkdir -p gpurun_out
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,power.limit,memory.total --format=csv > gpurun_out/smi.txt 2>&1
nproc >> gpurun_out/smi.txt
echo "== smoke" ; timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/smoke.txt 2>&1 ; echo "smoke rc=$?" | tee -a gpurun_out/smoke.txt
tail -3 gpurun_out/smoke.txt
echo "== pytest -m gpu" ; timeout 1500 python -m pytest tests -m gpu -x -q > gpurun_out/pytest_gpu.txt 2>&1 ; echo "pytest rc=$?" | tee -a gpurun_out/pytest_gpu.txt
tail -15 gpurun_out/pytest_gpu.txt
if [ "$MODE" = "full" ]; then
  echo "== compute-sanitizer (tiny step)"
  timeout 600 compute-sanitizer --tool memcheck --error-exitcode 7 python -c "
import sys; sys.path.insert(0,'tests'); sys.path.insert(0,'.')
from tcr_harness import TorchBackend
from parity_cases import run_case
b = TorchBackend()
print(run_case(b, model='TCResNet14', wm=1.5, window=480, stride=160, n=5, keep=0.5))
print(run_case(b, model='TCResNet8', wm=1.0, n=9, keep=0.5))
" > gpurun_out/sanitizer.txt 2>&1 ; echo "sanitizer rc=$?" | tee -a gpurun_out/sanitizer.txt
  tail -5 gpurun_out/sanitizer.txt
  # shared-memory races and divergent barriers: one TC-ResNet step on the default kernels (resident forward and backward-data,
  # grouped weight gradients) and the DS-CNN forward (mbarrier / TMA / wgmma pipeline); racecheck serialises heavily, so the cases are tiny
  for tool in racecheck synccheck; do
    echo "== compute-sanitizer --tool $tool"
    timeout 900 compute-sanitizer --tool $tool --error-exitcode 7 python -c "
import sys; sys.path.insert(0,'tests'); sys.path.insert(0,'.')
from tcr_harness import TorchBackend
from parity_cases import run_case
from test_dscnn import _run
b = TorchBackend()
print(run_case(b, model='TCResNet8', wm=1.0, n=5, keep=0.5))
print(_run(b, 'S', 49, 40, 3))
" > gpurun_out/$tool.txt 2>&1 ; echo "$tool rc=$?" | tee -a gpurun_out/$tool.txt
    grep -E "RACECHECK SUMMARY|ERROR SUMMARY|hazard|Barrier error" gpurun_out/$tool.txt | head -8
  done
fi
echo "== bench" ; timeout 900 python bench.py --steps 100 --warmup 10 > gpurun_out/bench.json 2> gpurun_out/bench.err ; echo "bench rc=$?"
cat gpurun_out/bench.json | cut -c1-3000 ; tail -5 gpurun_out/bench.err
echo "== bench TCResNet14-1.5 b1024" ; timeout 900 python bench.py --model TCResNet14 --width 1.5 --batch 1024 --steps 50 --warmup 5 --no-cpu-baseline > gpurun_out/bench_r14.json 2> gpurun_out/bench_r14.err ; echo "bench14 rc=$?"
cat gpurun_out/bench_r14.json | cut -c1-2500
echo "== ncu launch list"
timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -c 150 --csv --log-file gpurun_out/launches.csv python bench.py --steps 2 --warmup 3 --no-cpu-baseline --no-e2e > gpurun_out/bench_under_ncu.log 2>&1 ; echo "ncu rc=$?"
tail -30 gpurun_out/launches.csv | cut -c1-200
