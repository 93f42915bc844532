#!/bin/bash
# builds metagraph_b200/_lib/libmgb_<tag>.so with extra nvcc flags (probes of kernel variants; select with MGB_LIB)
#   scripts/build_variant.sh timers -DMGB_PHASE_TIMERS
#   scripts/build_variant.sh prep -DMGB_PREP_TIMERS          (k_prepare_exact's phase split, printed under MGB_DEBUG)
# Probes that bound a phase of k_prepare_exact by leaving it out (wrong results by design; time them with
# scripts/kernel_split.py): -DMGB_PROBE_NO_WRITES (no header or record stores), -DMGB_PROBE_NO_LAYOUT (no load after the
# hash buckets: no kh_pos, kh_vals / pl_pos or layout words; every read whose k-mer is found passes at p = 0)
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
