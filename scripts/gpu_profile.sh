#!/bin/bash
# Run on the GPU box via gpurun: tests, bench, ncu launch list and one full capture per hot kernel.
set -x
mkdir -p gpurun_out
python -m pytest tests -q -m gpu 2>&1 | tail -5 > gpurun_out/pytest_gpu_summary.log
python bench.py --steps 50 --warmup 5 > gpurun_out/bench.json 2> gpurun_out/bench.err
tail -c 600 gpurun_out/bench.err
KREGEX='regex:icp_dense_kernel|icp_dense_pending_kernel|target_extents_kernel|normals_7x11_kernel|project_scatter_kernel|project_resolve_kernel|icp_finalize_kernel'
ncu --metrics gpu__time_duration.sum --clock-control none -k "$KREGEX" -s 14 -c 28 --csv \
    --log-file gpurun_out/launches.csv python bench.py --steps 4 --warmup 2 --cpu-pairs 0 --rotate 1 --train-steps 0 --stream-frames 0 > gpurun_out/bench_under_ncu.log 2>&1
ncu --set full --clock-control none --import-source on -k "$KREGEX" -s 14 -c 7 -f -o gpurun_out/prof_r01 \
    python bench.py --steps 4 --warmup 2 --cpu-pairs 0 --rotate 1 --train-steps 0 --stream-frames 0 > gpurun_out/bench_under_ncu_full.log 2>&1
ls -la gpurun_out
