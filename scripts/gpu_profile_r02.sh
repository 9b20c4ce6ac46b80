#!/bin/bash
# Round-2 evidence run (on the GPU box via gpurun): tests, bench, ncu launch lists and full captures.
mkdir -p gpurun_out
if [ "$1" != "notests" ]; then python -m pytest tests -q -m gpu 2>&1 | tail -3 > gpurun_out/pytest_gpu_summary.log; fi
python bench.py --steps 50 --warmup 5 > gpurun_out/bench_r02.json 2> gpurun_out/bench_r02.err
KREGEX='regex:icp_dense_kernel|icp_dense_pending_kernel|target_extents_kernel|normals_7x11_kernel|project_scatter_kernel|project_resolve_kernel|icp_finalize_kernel'
ncu --metrics gpu__time_duration.sum --clock-control none -k "$KREGEX" -s 14 -c 28 --csv \
    --log-file gpurun_out/r02_launches.csv python bench.py --steps 4 --warmup 2 --cpu-pairs 0 --rotate 1 --train-steps 0 --stream-frames 0 > gpurun_out/bench_under_ncu.log 2>&1
ncu --set full --clock-control none --import-source on -k "$KREGEX" -s 14 -c 7 -f -o gpurun_out/prof_r02 \
    python bench.py --steps 4 --warmup 2 --cpu-pairs 0 --rotate 1 --train-steps 0 --stream-frames 0 > gpurun_out/bench_under_ncu_full.log 2>&1
ncu --metrics gpu__time_duration.sum,sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active --clock-control none --csv \
    --log-file gpurun_out/r02_train_launches.csv python scripts/gpu_train_step_once.py > gpurun_out/train_once.log 2>&1
# full captures of the wgmma kernels of the LAST training step (3 steps x ~60 conv launches: skip the first 2 steps)
ncu --set full --clock-control none -k 'regex:conv_rows_tc_kernel|conv_wgrad2_tc_kernel|stem_fprop_tc_kernel|conv_fprop_tc_kernel|conv_wgrad_tc_kernel' \
    -s 124 -c 62 -f -o gpurun_out/prof_r02_conv python scripts/gpu_train_step_once.py > gpurun_out/train_once_full.log 2>&1
# the 62-launch report is ~80 MB (gpurun brings back at most 64 MiB): keep its raw-metric table only
ncu -i gpurun_out/prof_r02_conv.ncu-rep --page raw --csv > gpurun_out/r02_conv_raw.csv 2> /dev/null
rm -f gpurun_out/prof_r02_conv.ncu-rep
du -sh gpurun_out; ls -la gpurun_out | tail -14
