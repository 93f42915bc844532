#!/bin/bash
# builds metagraph_b200/_lib/libmgb_<tag>.so with extra nvcc flags (probes of kernel variants; select with MGB_LIB)
#   scripts/build_variant.sh timers -DMGB_PHASE_TIMERS
set -e
tag=$1; shift
cd "$(dirname "$0")/.."
obj=build/obj_$tag; mkdir -p $obj
F="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC,-fopenmp -diag-suppress 550,177 $*"
for u in api.cu api_generic.cu api_canonical.cu boss_build.cpp dbg_load.cpp; do
  nvcc $F -c -o $obj/${u%.*}.o metagraph_b200/csrc/$u &
done
wait
nvcc $F -shared -o metagraph_b200/_lib/libmgb_$tag.so $obj/*.o -lgomp
ls -la metagraph_b200/_lib/libmgb_$tag.so
