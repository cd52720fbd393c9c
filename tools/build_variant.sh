#!/bin/bash
# Development tool: build an A/B variant of libpulse_b200 with extra -D flags on ONE translation unit.
#   tools/build_variant.sh <name> <file.cu> [-DFLAG=VALUE ...]   ->  pulse_b200/build/libpulse_<name>.so
# Examples:  tools/build_variant.sh trace gemm_wgmma.cu -DPULSE_GEMM_VARIANT=3     (phase-trace build for tools/gemm_trace.py)
#            tools/build_variant.sh t2 im_step.cu -DPULSE_STEP_TEAMS=2               (2 consumer teams, 146 registers)
# Use with PULSE_ALT_LIB=$PWD/pulse_b200/build/libpulse_<name>.so on tools/bench_update_gemms.py, tools/gemm_trace.py, tools/microbench.py.
set -e
cd "$(dirname "$0")/.."
NAME=$1; SRC=$2; shift 2
python -m pulse_b200.build > /dev/null
BASE=$(basename "$SRC" .cu)
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Iinclude -Ipulse_b200/csrc "$@" \
  -c pulse_b200/csrc/$SRC -o pulse_b200/build/variant_${NAME}_$BASE.o
OBJS=$(ls pulse_b200/build/*.o | grep -v "/$BASE.o\|variant_")
nvcc -gencode arch=compute_90a,code=sm_90a --shared -o pulse_b200/build/libpulse_$NAME.so $OBJS pulse_b200/build/variant_${NAME}_$BASE.o -lcudart
echo pulse_b200/build/libpulse_$NAME.so
