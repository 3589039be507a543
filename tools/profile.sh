#!/usr/bin/env bash
# Launch list + full ncu capture of our kernels for the MNIST-CNN step (1 GPU, via gpurun):
#   gpurun --timeout 600 -- tools/profile.sh
set -euo pipefail
OUT=gpurun_out
mkdir -p $OUT
ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --cache-control none --csv \
    --log-file $OUT/launches.csv python tests/gpu/profile_step.py
# every wgmma kernel of the step + the fused optimizer/collective kernel, one capture each
PROFILE_STEPS=1 ncu --set full --clock-control none --import-source on --profile-from-start off \
    -k regex:"tfy_conv3x3|tfy_dense|tfy_gemm|tfy_fused_step" -f -o $OUT/prof_step_kernels \
    python tests/gpu/profile_step.py
# read back on the CPU box with:  python tools/ncu_summary.py gpurun_out/prof_*.ncu-rep
