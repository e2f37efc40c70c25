#!/bin/bash
# last check of a round in ONE call: GPU suite + smoke() on the in-tree library, the BASELINE inputs, and (optional) variants
# present in build_variants/ -- parity first, then the same inputs.   usage: bash tools/gpu_final.sh
set -u
O=${SJ_TOOLS_OUT:-tools_out}
mkdir -p $O
( time timeout 500 python -m pytest tests -m gpu -q --timeout 400 ) > $O/pytest_gpu.log 2>&1
echo "pytest rc=$?" >> $O/pytest_gpu.log; tail -5 $O/pytest_gpu.log | head -2
python -c "import __graft_entry__ as g; g.smoke()" > $O/smoke.log 2>&1; tail -1 $O/smoke.log
IN=twitterescaped,twitter,gsoc-2018,parking-citations
echo "== in-tree"; timeout 200 python tools/config_bench.py 256 $IN | cut -d'|' -f2,10,11 | tail -4
for V in $(ls build_variants/*.so 2>/dev/null | xargs -n1 basename 2>/dev/null | sed "s/\.so$//"); do  # (every variant present; the arguments are only a label)
  ( SJ_B200_LIB=$PWD/build_variants/$V.so timeout 300 python -m pytest tests/test_gpu_stage2.py -m gpu -q -x --timeout 300 ) > $O/pytest_$V.log 2>&1
  echo "== $V: $(tail -1 $O/pytest_$V.log)"
  SJ_B200_LIB=$PWD/build_variants/$V.so timeout 200 python tools/config_bench.py 256 $IN | cut -d'|' -f2,10,11 | tail -4
done
