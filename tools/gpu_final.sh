#!/bin/bash
# Round-end verification on the GPU: parity tests, smoke, kernel micro-benchmarks, both bench arms, ncu launch list of the timed
# region and one full capture of the (rewritten) multi-tensor weight fake-quant kernel.  Everything lands in gpurun_out/.
mkdir -p gpurun_out
timeout 500 python -m pytest tests -m gpu -q 2>&1 | grep -v "^  \|^$" | cut -c1-300 | tail -8
timeout 120 python -c "import __graft_entry__ as g; g.smoke()" 2>&1 | tail -1
timeout 250 python tools/kbench.py --only minmax,hist,lt,lc,ft,multi,quantile --reps 20 > gpurun_out/kbench.txt 2>&1; grep -v "var[1456]" gpurun_out/kbench.txt | cut -c1-110
timeout 400 python bench.py --impl reference --steps 4 --warmup 1 > gpurun_out/bench_ref.json 2> gpurun_out/bench_ref.err; echo "ref exit $?"; cut -c1-500 gpurun_out/bench_ref.json
timeout 600 python bench.py > gpurun_out/bench.json 2> gpurun_out/bench.err; echo "bench exit $?"; cut -c1-3000 gpurun_out/bench.json; tail -3 gpurun_out/bench.err
B="python bench.py --steps 4 --warmup 3 --rotate 2 --no-e2e --no-cpu-baseline"
timeout 300 ncu --nvtx --nvtx-include "timed/" --metrics gpu__time_duration.sum --clock-control none --csv --log-file gpurun_out/launches.csv $B > gpurun_out/bench_under_ncu.log 2>&1; tail -1 gpurun_out/bench_under_ncu.log | cut -c1-200
timeout 200 ncu --set full --clock-control none --import-source on --nvtx --nvtx-include "timed/" -k regex:multi_channel -c 1 -f -o gpurun_out/prof_multi_channel2 $B > gpurun_out/ncu_mc.log 2>&1; tail -1 gpurun_out/ncu_mc.log | cut -c1-200
ls -la gpurun_out | grep -E "prof_multi_channel2|launches|bench"
