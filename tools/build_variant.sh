#!/bin/bash
# build a named variant of the engine next to the default build:  tools/build_variant.sh <name> [-D...]
#   -> ra_b200/csrc/libra_engine_<name>.so   (use with RA_ENGINE_SO=..., see tools/bench_variants.sh)
set -e
v=$1; shift
cd "$(dirname "$0")/../ra_b200/csrc"
/usr/local/cuda/bin/nvcc -O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC,-fopenmp -Xptxas -v \
  "$@" -shared -o libra_engine_$v.so engine.cu host_flood.cu -lgomp 2> build_$v.log || { cat build_$v.log; exit 1; }
grep -A3 "Compiling entry function '_Z16raft_step_kernelILi261" build_$v.log | grep -E "Used|spill" | tr '\n' ' '; echo " [$v $*]"
