#!/bin/bash
# Profile capture (outputs are summarised by profiles/summarize.py).  Numbers printed by bench.py under ncu are NOT benchmark values.
set -x
mkdir -p gpurun_out
# 1. launch list of the bench command (per-launch device time; cold-cache + serialised: compare SHARES)
# (bench.py brackets its timed steps with cudaProfilerStart/Stop, so only those launches are listed)
ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off -c ${COUNT:-40000} --csv \
    --log-file gpurun_out/r01_launches.csv python bench.py --steps 1 --warmup 3 --no-e2e --no-cpu \
    > gpurun_out/r01_launches_bench.log 2>&1
# 2. full capture of the dominant GEMM (matvec, 128x128 tile config) and of the Jacobi round kernel
ncu --set full --clock-control none --import-source on -k regex:grouped_gemm_kernel -s 6 -c 2 \
    -o gpurun_out/r01_gemm python tests/dev_kernel_probe.py gemm > gpurun_out/r01_gemm.log 2>&1
ncu --set full --clock-control none --import-source on -k regex:jacobi_ -s 90 -c 6 \
    -o gpurun_out/r01_jacobi python tests/dev_kernel_probe.py svd > gpurun_out/r01_jacobi.log 2>&1
ls -la gpurun_out
