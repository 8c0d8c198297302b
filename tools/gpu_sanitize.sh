#!/bin/bash
# compute-sanitizer memcheck over the GPU parity tests of OUR kernels (the comparison against the
# reference's own CUDA build is excluded: its kernels are not ours to fix), then racecheck over the shared-memory kernels.
# PYTORCH_NO_CUDA_MEMORY_CACHING=1: every tensor is its own cudaMalloc, so an out-of-bounds access cannot hide inside torch's pool.
mkdir -p gpurun_out
export PYTORCH_NO_CUDA_MEMORY_CACHING=1
timeout ${MEMCHECK_TIMEOUT:-420} compute-sanitizer --tool memcheck --error-exitcode 9 --print-limit 20 \
    python -m pytest tests/test_gpu_parity.py tests/test_gpu_next_rows.py tests/test_gpu_configs.py -m gpu -q -x -p no:cacheprovider \
    > gpurun_out/memcheck.log 2>&1
echo "memcheck exit $?" | tee -a gpurun_out/memcheck.log
grep -E "ERROR SUMMARY|passed|failed|Invalid|Out of bounds|misaligned" gpurun_out/memcheck.log | tail -8
timeout ${RACECHECK_TIMEOUT:-240} compute-sanitizer --tool racecheck --error-exitcode 9 --print-limit 20 \
    python -m pytest tests/test_gpu_parity.py -m gpu -q -x -p no:cacheprovider -k "hist or minmax or quantile or isotone or kl or mse or search" \
    > gpurun_out/racecheck.log 2>&1
echo "racecheck exit $?" | tee -a gpurun_out/racecheck.log
grep -E "RACECHECK SUMMARY|passed|failed|hazard" gpurun_out/racecheck.log | tail -8
