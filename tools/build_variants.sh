#!/bin/bash
# Builds variant libraries (compile-time switches) into build_variants/ for the A/B loop of tools/gpu_checks.sh.
#   usage: tools/build_variants.sh name1="-DSJ_X=1" name2="-DSJ_Y=2 -DSJ_Z=3" ...
#   e.g.   tools/build_variants.sh emit6="-DSJ_S2_EMIT_MIN_BLOCKS=6" num4="-DSJ_S2_NUMBERS_MIN_BLOCKS=4" \
#                                  coop32="-DSJ_S2_COOP_MIN=32" fm0="-DSJ_S2_FAST_MEASURE=0"
# The switches and what was measured with them are listed at the top of simdjson-go_b200/csrc/stage2.cuh
# (stage 2) and stage1.cuh (K1: SJ_S1_WARPS, SJ_S1_STEPS, SJ_S1_CTAS_PER_SM, ...).
set -eu
cd "$(dirname "$0")/.."
OUT=${SJ_VARIANT_DIR:-build_variants}
mkdir -p "$OUT"
F="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -shared -Xcompiler -fPIC"
pids=()
for spec in "$@"; do
  name=${spec%%=*}
  flags=${spec#*=}
  ( nvcc $F $flags -o "$OUT/$name.so" simdjson-go_b200/csrc/sj_api.cu && echo "built $OUT/$name.so  [$flags]" ) &
  pids+=($!)
done
rc=0
for p in "${pids[@]}"; do wait $p || rc=1; done
exit $rc
