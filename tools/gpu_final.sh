#!/bin/bash
# last check of a round in ONE call: GPU suite + smoke() on the in-tree library, then the BASELINE inputs.
#   usage: bash tools/gpu_final.sh
set -u
O=${SJ_TOOLS_OUT:-tools_out}
mkdir -p $O
( time timeout 500 python -m pytest tests -m gpu -q --timeout 400 ) > $O/pytest_gpu.log 2>&1
echo "pytest rc=$?" >> $O/pytest_gpu.log; tail -5 $O/pytest_gpu.log | head -2
python -c "import __graft_entry__ as g; g.smoke()" > $O/smoke.log 2>&1; tail -1 $O/smoke.log
IN=twitterescaped,twitter,gsoc-2018,parking-citations
echo "== in-tree"; timeout 200 python tools/config_bench.py 256 $IN | cut -d'|' -f2,10,11 | tail -4
