#!/bin/bash
# TEST INFRASTRUCTURE: run the reference + seam + harness binary in one of its modes.
#   usage: oracle/run_harness.sh <cpu|shadow|gpu|dump> <cmd-stem under tests/golden/cmd> <ngen> [report-file]
# Needs the prebuilt oracle/_ref (built where /root/reference exists; shipped to the GPU box).
set -euo pipefail
cd "$(dirname "$0")/.."
MODE=$1; STEM=$2; NGEN=$3; REPORT=${4:-/dev/stderr}
TMP=$(mktemp -d)
sed -e "s/NGEN/$NGEN/" -e "s#OUTPREFIX#$TMP/out#" tests/golden/cmd/$STEM.nex > $TMP/run.nex
BIN=oracle/_ref/mb_b200
[ "${SSE:-0}" = "1" ] && BIN=oracle/_ref/mb_b200_sse
START=$(date +%s.%N)
MB200_MODE=$MODE MB200_REPORT=$TMP/report.json timeout -s KILL ${MB200_TIMEOUT:-900} $BIN $TMP/run.nex > $TMP/run.log 2>$TMP/run.err || { tail -5 $TMP/run.log $TMP/run.err; exit 1; }
END=$(date +%s.%N)
grep -E "Using H100|Using standard|likelihood calculator" $TMP/run.log | head -3 || true
head -5 $TMP/run.err || true
python3 - "$TMP/report.json" "$START" "$END" "$STEM" "$NGEN" >> $REPORT <<'PY'
import json, sys
rep = json.loads(open(sys.argv[1]).read().strip().splitlines()[-1])
rep["wall_s"] = float(sys.argv[3]) - float(sys.argv[2]); rep["workload"] = sys.argv[4]; rep["ngen"] = int(sys.argv[5])
print(json.dumps(rep))
PY
rm -rf $TMP
