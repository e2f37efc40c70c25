#!/bin/bash
# compute-sanitizer over the whole path on small inputs (SURVEY.md section 5 asked for it; K1 relies on relaxed look-back
# descriptors, cross-proxy shared-memory reuse and hand-rolled mbarrier hand-shakes).  Logs land in $SJ_TOOLS_OUT (default tools_out/).
# usage: bash tools/sanitize.sh
set -u
O=${SJ_TOOLS_OUT:-tools_out}
mkdir -p $O
for tool in memcheck racecheck synccheck; do
  mode=full
  [ $tool = racecheck ] && mode=quick
  ( time timeout 240 compute-sanitizer --tool $tool --error-exitcode 9 python tools/sanitize_run.py $mode ) > $O/sanitizer_$tool.log 2>&1
  echo "$tool rc=$? : $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY|sanitize_run ok' $O/sanitizer_$tool.log | tr '\n' ' ')"
done
