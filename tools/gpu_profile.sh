#!/bin/bash
# `ncu --set full` captures (with source correlation) of the two streaming stage-2 kernels on one of the
# BASELINE inputs (default twitterescaped, 64 MiB).  Reports land in $SJ_TOOLS_OUT (default tools_out/); read them with
#   python tools/ncu_source_lines.py tools_out/k2r_<input>.ncu-rep 60
#   ncu -i tools_out/k2r_<input>.ncu-rep --page raw --csv
#   usage: bash tools/gpu_profile.sh [input] [MiB]
set -u
O=${SJ_TOOLS_OUT:-tools_out}
IN=${1:-twitterescaped}
MIB=${2:-64}
mkdir -p $O
B="python tools/config_bench.py $MIB $IN"
timeout 280 ncu --set full --import-source on --clock-control none -k regex:s2s_emit_kernel -s 3 -c 1 -o $O/k2r_$IN -f $B > $O/ncu_k2r_$IN.log 2>&1
timeout 280 ncu --set full --import-source on --clock-control none -k 'regex:stage1_flatten_kernel<[a-z]+, false, true>' -s 3 -c 1 -o $O/k1parse_$IN -f $B > $O/ncu_k1parse_$IN.log 2>&1
ls -la $O/*.ncu-rep
