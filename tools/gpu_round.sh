#!/bin/bash
# One GPU session of the development loop: micro-benchmarks, parity (quick subset first), bench, phase timers.
# Usage (through gpurun): bash tools/gpu_round.sh <tag> [quick|full]
TAG=${1:-x}
MODE=${2:-full}
OUT=gpurun_out
mkdir -p $OUT
echo "== go probe"; (go version 2>&1 || true) | head -1
nvidia-smi --query-gpu=name,clocks.max.sm,clocks.sm --format=csv,noheader
echo "== ubench"
"$(command -v nvcc || echo /usr/local/cuda/bin/nvcc)" -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/ubench_cluster tools/ubench_cluster.cu || exit 1
timeout 120 tools/ubench_cluster > $OUT/ubench_$TAG.txt 2>&1; grep -E "cs=16 tpb= 320|cs= 8 tpb= 320" $OUT/ubench_$TAG.txt | grep -E "argmax|arg-max|allreduce_w<6>"
echo "== quick parity"
timeout 900 python -m pytest tests/test_gpu_detail.py tests/test_config1.py tests/test_zz_prebound_gpu_share.py -x -q -m gpu 2>&1 | tail -15
if [ "$MODE" = "full" ]; then
  echo "== full gpu suite"
  timeout 2400 python -m pytest tests/ -x -q -m gpu 2>&1 | tail -15
fi
echo "== bench"
timeout 600 python bench.py --steps 3 --warmup 3 --no-cpu-baseline --no-batch 2>$OUT/bench_$TAG.err | tee $OUT/bench_$TAG.json | python -c "import sys,json; d=json.loads(sys.stdin.read()); print('value', round(d['value']), 'ms', round(d['ms_per_step'],1), 'e2e', round(d['e2e']['value']))"
echo "== phase timers"
timeout 600 python tools/profile_run.py --pods 100000 --phase-timers > $OUT/phase_$TAG.txt 2>&1; tail -3 $OUT/phase_$TAG.txt | cut -c1-1500
