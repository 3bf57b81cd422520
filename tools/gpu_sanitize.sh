#!/bin/bash
# Runs tools/sanitize.py under each compute-sanitizer tool (memcheck with the leak check); logs go to $OUT.
OUT=${OUT:-sanitizer_logs}
mkdir -p "$OUT"
for tool in memcheck racecheck synccheck; do
  extra=""; [ $tool = memcheck ] && extra="--leak-check full"
  timeout 900 compute-sanitizer --tool $tool $extra --print-limit 30 python tools/sanitize.py > "$OUT/sanitizer_$tool.log" 2>&1; echo "$tool rc $?"
  grep -E "ERROR SUMMARY|LEAK SUMMARY|leaked|sanitize workload ok|RACECHECK SUMMARY|hazard" "$OUT/sanitizer_$tool.log" | head -5
done
