#!/bin/bash
# A/B of stage-2 variants (build_variants/*.so) against the in-tree library: parity first, then the BASELINE inputs
#   usage: bash tools/gpu_esc_ab.sh name [name ...]
set -u
O=${SJ_TOOLS_OUT:-tools_out}
mkdir -p $O
for V in "$@"; do
  ( SJ_B200_LIB=$PWD/build_variants/$V.so timeout 900 python -m pytest tests/test_gpu_stage2.py -m gpu -q -x --timeout 600 ) > $O/pytest_$V.log 2>&1
  echo "$V: $(tail -1 $O/pytest_$V.log)"
done
for V in "" "$@"; do
  lib=${V:+$PWD/build_variants/$V.so}
  echo "== ${V:-in-tree}"
  SJ_B200_LIB=$lib timeout 300 python tools/config_bench.py 256 2>&1 | cut -d'|' -f2,10,11 | tail -6
done
