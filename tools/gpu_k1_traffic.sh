#!/bin/bash
# ncu --set full of K1 on the bench batch and on twitter-shaped input; reports to $SJ_TOOLS_OUT (default tools_out/)
set -u
O=${SJ_TOOLS_OUT:-tools_out}
mkdir -p $O
timeout 600 ncu --set full --clock-control none --import-source on -k regex:stage1_flatten -s 8 -c 1 -o $O/k1_bench -f \
   python bench.py --steps 1 --warmup 1 --inflight 1 --no-cpu --twitter-mib 0 --stream-gib 0 > $O/ncu_k1_bench.log 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:stage1_flatten -s 3 -c 1 -o $O/k1_twitter -f \
   python tools/quick_stage1_bench.py twitter 256 > $O/ncu_k1_twitter.log 2>&1
ls -la $O/k1_*.ncu-rep
