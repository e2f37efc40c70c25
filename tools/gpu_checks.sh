#!/bin/bash
# One run that checks everything on the GPU machine: GPU suite, smoke(), the bench line with all its legs and the
# CPU arm, the launch list of the bench batch, the other BASELINE configs, the per-file fixture table.  Results land in
# $SJ_TOOLS_OUT (default tools_out/).   usage: bash tools/gpu_checks.sh
set -u
O=${SJ_TOOLS_OUT:-tools_out}
mkdir -p $O
nvidia-smi --query-gpu=name,clocks.max.sm --format=csv,noheader > $O/gpu.txt 2>&1; nproc >> $O/gpu.txt
( time timeout 1200 python -m pytest tests -m gpu -q --timeout 900 ) > $O/pytest_gpu.log 2>&1
echo "pytest rc=$?" >> $O/pytest_gpu.log; tail -4 $O/pytest_gpu.log
python -c "import __graft_entry__ as g; g.smoke()" > $O/smoke.log 2>&1; tail -1 $O/smoke.log
timeout 600 python bench.py > $O/bench_n1.json 2> $O/bench_n1.err; echo "bench rc=$?"; tail -2 $O/bench_n1.err
timeout 300 python bench.py --impl reference > $O/bench_reference.json 2> $O/bench_reference.err; cut -c1-200 $O/bench_reference.json
python - "$O" <<'PY'
import json, sys
d=json.loads([l for l in open(sys.argv[1] + '/bench_n1.json') if l.startswith('{')][-1])
for k in ('value','ms_per_step','e2e','e2e_nocopy','stream','roofline','roofline_twitter','roofline_parse','parse_count_where','cpu_baseline','gpu_launches','clocks'): print(k, d.get(k))
PY
timeout 200 ncu --metrics gpu__time_duration.sum --clock-control none -c 500 --csv --log-file $O/launches_bench_ndjson128MiB.csv \
    python bench.py --steps 2 --warmup 1 --batch-mib 128 --inflight 1 --no-cpu --twitter-mib 0 --stream-gib 0 > $O/bench_under_ncu.log 2>&1
python tools/summarize_launches.py $O/launches_bench_ndjson128MiB.csv 2>/dev/null | head -14
timeout 300 python tools/config_bench.py 256 > $O/config_stream.md 2>&1; cat $O/config_stream.md | cut -d'|' -f2,7,10,11
timeout 300 python tools/fixture_bench.py 200 > $O/fixture_bench.md 2>&1; cut -d'|' -f2,4,5,9 $O/fixture_bench.md | tail -15
