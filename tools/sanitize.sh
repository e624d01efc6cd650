#!/bin/bash
# compute-sanitizer passes over every kernel of the library; logs go to $1 (default: a new temporary directory)
OUT=${1:-$(mktemp -d)}
mkdir -p "$OUT"
for tool in memcheck racecheck synccheck; do
  timeout 900 compute-sanitizer --tool $tool --print-limit 20 python tools/san_workload.py > "$OUT/sanitizer_$tool.log" 2>&1
  echo "$tool rc=$?"; tail -4 "$OUT/sanitizer_$tool.log"
done
echo "logs in $OUT"
