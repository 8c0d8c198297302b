#!/bin/bash
# GPU parity tests, smoke, a short bench and the ncu launch list, run on one GPU machine; outputs go to the output directory below.
mkdir -p gpurun_out
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,power.draw,memory.total --format=csv > gpurun_out/gpu.txt 2>&1
python -m pytest tests -m gpu -x -q > gpurun_out/tests.log 2>&1; echo "pytest exit $?" >> gpurun_out/tests.log
tail -25 gpurun_out/tests.log
python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/smoke.log 2>&1; tail -2 gpurun_out/smoke.log
python bench.py --steps 8 --warmup 3 ${BENCH_FLAGS} > gpurun_out/bench.json 2> gpurun_out/bench.err; echo "bench exit $?"; cat gpurun_out/bench.json; tail -5 gpurun_out/bench.err
