#!/bin/bash
# Which Hopper (sm_90a) instructions the shipped library contains, per kernel (evidence that the tensor-core path is
# warpgroup-MMA / bulk-async-copy code, not mma.sync):  HGMMA = wgmma.mma_async, WARPGROUP = wgmma fences and waits,
# UBLKCP = cp.async.bulk (TMA engine), SYNCS = mbarrier operations.
# usage: profiles/sass_counts.sh [library]   (needs cuobjdump; no GPU)
LIB=${1:-$(dirname "$0")/../mrbayes_b200/lib/libmb200.so}
cuobjdump -sass "$LIB" 2>/dev/null | awk '
  /Function : / { f = $3 }
  /HGMMA|WARPGROUP|UBLKCP|UTMALDG|UTMASTG|SYNCS/ {
      n = split($0, a, " ");
      for (i = 1; i <= n; i++) if (a[i] ~ /^(HGMMA|WARPGROUP|UBLKCP|UTMALDG|UTMASTG|SYNCS)/) { split(a[i], b, "."); c[f " " b[1]]++ } }
  END { for (k in c) print c[k], k }' | sort -k2,2 -k3,3 | while read n f m; do printf "%-28s %-12s %s\n" "$(echo $f | c++filt | sed -e 's/^void //' -e 's/(.*//')" "$m" "$n"; done
