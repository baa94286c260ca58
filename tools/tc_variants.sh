#!/bin/bash
# Time every kernel variant under tools/_variants/ (NSB_LIB A/B) with tools/tc_check.py; optional ncu capture of the default.
cd "$(dirname "$0")/.."
OUT=${OUT:-tool_out}          # reports go here (git-ignored)
mkdir -p "$OUT"
for so in nersemble_b200/libnsb.so tools/_variants/*.so; do
  echo "== $so"
  NSB_LIB=$PWD/$so timeout 200 python tools/tc_check.py 2>&1 | tail -6 | grep -v "^frame"
done
if [ -n "$NCU" ]; then
  ncu --set full --import-source on --clock-control none -k regex:field_kernel_tc -s 4 -c 1 -o $OUT/$NCU -f \
      python tools/tc_check.py > $OUT/$NCU.log 2>&1
  ncu -i $OUT/$NCU.ncu-rep --page raw --csv > $OUT/$NCU.raw.csv 2>/dev/null
  ncu -i $OUT/$NCU.ncu-rep --page source --csv > $OUT/$NCU.source.csv 2>/dev/null
fi
