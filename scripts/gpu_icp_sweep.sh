#!/bin/bash
# ICP sweep (profiling only): window-growing steps before a lane is handed to the block-search kernel
for ms in 16 24 32 48 64; do
  echo "== max_strips=$ms"
  DELORA_ICP_MAX_STRIPS=$ms timeout 200 python scripts/gpu_explore.py 2>&1 | grep -E "^icp_dense|^icp_identityT|^icp_badT|^full step"
done
