#!/bin/bash
# Build libtgingest.so variants with different __launch_bounds__ budgets (LB_*: resident CTAs per SM the compiler budgets
# registers for) into build_variants/; tools/variants_bench.sh (Telegram, config-2 step) and tools/variants_yt.sh (YouTube) time them on the GPU box.
# The lane emitter's variants (lane<LB_LANE>s<LANE_STAGE>) come with build_variants/lane_occupancy_<variant>, which prints
# the resident CTAs per SM the runtime gives them.  Usage: tools/variants.sh
set -e
cd "$(dirname "$0")/../distributed_crawler_b200/csrc"
NV="/usr/local/cuda/bin/nvcc -O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-Wall"
mkdir -p ../../build_variants
build() { name=$1; shift; $NV -shared "$@" -o ../../build_variants/libtgingest_$name.so tgingest.cu -lcudart 2>/dev/null & }
for k in ${LBS:-4 5 6 7 8}; do
  build all$k -DLB_SIZE=$k -DLB_ESC=$k -DLB_MAPS=$k -DLB_PARSE=$k
  build yt$k -DLB_YT=$k
done
wait
for k in ${LANE_LBS:-2 3 4}; do
  for st in ${LANE_STAGES:-128 256}; do
    build lane${k}s$st -DLB_LANE=$k -DLANE_STAGE=$st
    $NV -DLB_LANE=$k -DLANE_STAGE=$st -o ../../build_variants/lane_occupancy_lane${k}s$st ../../tools/lane_occupancy.cu -lcudart 2>/dev/null &
  done
  wait
done
ls -la ../../build_variants
