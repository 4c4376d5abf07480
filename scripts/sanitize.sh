#!/bin/bash
# compute-sanitizer over the toy-shape GPU parity tests of every kernel family that hand-rolls mbarrier / wgmma
# pipelines (GEMM forward + dgrad/wgrad, attention forward / causal / GQA / backward, conv, LN-modulate and the training
# row kernels).  Run on an H100:   bash scripts/sanitize.sh [memcheck|racecheck|synccheck|initcheck ...]
# Writes $SANITIZE_OUT/sanitize_<tool>.log (default sanitize_out/) and a one-line-per-tool summary
# $SANITIZE_OUT/sanitize_summary.json.  The selection keeps each tool under a few minutes (sanitizers slow kernels 10-100x).
set -u
cd "$(dirname "$0")/.."
OUT=${SANITIZE_OUT:-sanitize_out}
mkdir -p "$OUT"
TOOLS=${@:-"memcheck racecheck synccheck"}
NODES=$(python scripts/sanitize_select.py)
echo "{" > "$OUT/sanitize_summary.json"
first=1
for tool in $TOOLS; do
  log="$OUT/sanitize_${tool}.log"
  timeout 2400 compute-sanitizer --tool $tool --print-limit 20 --error-exitcode 99 \
      python -m pytest $NODES -m gpu -q -p no:cacheprovider > "$log" 2>&1
  rc1=$?
  rc2=0
  errs=$(grep -c "========= .*\(Invalid\|Race\|hazard\|Barrier error\|Uninitialized\)" "$log" || true)
  summ=$(grep "ERROR SUMMARY" "$log" | tr '\n' ';')
  passed=$(grep -E "passed|failed" "$log" | tr '\n' ';')
  [ $first -eq 0 ] && echo "," >> "$OUT/sanitize_summary.json"
  first=0
  printf '"%s": {"rc": [%d, %d], "error_lines": %s, "summary": "%s", "pytest": "%s"}' "$tool" $rc1 $rc2 "${errs:-0}" "$summ" "$passed" >> "$OUT/sanitize_summary.json"
  echo "[$tool] rc=$rc1,$rc2 $summ $passed"
done
echo "}" >> "$OUT/sanitize_summary.json"
