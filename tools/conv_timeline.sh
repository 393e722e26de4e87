#!/bin/bash
# Debug aid: builds tests/cuda/test_conv_tc.cu + conv_tc.cu with -DB2P_CONV_TIMELINE (clock64() stamps of the first CTAs at the
# phase boundaries of conv_tc_body), to be run on an H100:  build/test_conv_tc_tl | grep timeline
# and tools/conv_layers.cu the same way (the bench's layer shapes: consumer clocks in patch waits, weight waits, MMA waits,
# the rest of the main loop and the epilogue):  build/conv_layers_tl
# (production builds compile the stamps away).
set -e
cd "$(dirname "$0")/.."
mkdir -p build
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -DB2P_CONV_TIMELINE "$@" \
     -o build/test_conv_tc_tl tests/cuda/test_conv_tc.cu pytorch_realtime_multi-person_pose_estimation_b200/csrc/conv_tc.cu -lcuda
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -DB2P_CONV_TIMELINE "$@" \
     -o build/conv_layers_tl tools/conv_layers.cu pytorch_realtime_multi-person_pose_estimation_b200/csrc/conv_tc.cu -lcuda
echo "built build/test_conv_tc_tl build/conv_layers_tl"
