#!/bin/bash
# quick check after a kernel change: GPU suite, the BASELINE configs, launch list of one config
set -u
O=${SJ_TOOLS_OUT:-tools_out}
mkdir -p $O
( time timeout 1200 python -m pytest tests -m gpu -q --timeout 900 -x ) > $O/pytest_gpu.log 2>&1
echo "pytest rc=$?" >> $O/pytest_gpu.log; tail -4 $O/pytest_gpu.log
timeout 300 python tools/config_bench.py 256 > $O/config_stream.md 2>&1; cat $O/config_stream.md | cut -d'|' -f2,7,10,11
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -c 300 --csv --log-file $O/launches_twesc_64MiB.csv \
      python tools/config_bench.py 64 ${1:-twitterescaped} > $O/configs_under_ncu.log 2>&1
python tools/summarize_launches.py $O/launches_twesc_64MiB.csv 2>&1 | tail -14
