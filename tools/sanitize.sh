#!/bin/bash
# compute-sanitizer memcheck + racecheck (+ initcheck / synccheck) over every libnsb kernel (SURVEY 5: race detection).
# usage (on an H100 machine with compute-sanitizer): bash tools/sanitize.sh   -> $OUT/sanitize_*.txt, summary on stdout.
set -u
cd "$(dirname "$0")/.."
OUT=${OUT:-tool_out}          # reports go here (git-ignored)
mkdir -p "$OUT"
CS=${CS:-/usr/local/cuda/bin/compute-sanitizer}
for tool in ${TOOLS:-memcheck racecheck synccheck initcheck}; do
  extra=""
  [ "$tool" = racecheck ] && extra="--racecheck-report all"
  SAN_RAYS=${SAN_RAYS:-96} timeout ${SAN_TIMEOUT:-600} $CS --tool $tool $extra --print-limit 20 \
      python tools/sanitize_driver.py > $OUT/sanitize_$tool.txt 2>&1
  echo "== $tool: exit $? =="
  grep -E "ERROR SUMMARY|RACECHECK SUMMARY|sanitize_driver: ok|Error:|hazard" $OUT/sanitize_$tool.txt | sort | uniq -c | head -12
done
