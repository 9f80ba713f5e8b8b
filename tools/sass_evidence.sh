#!/bin/bash
# Instruction evidence from the in-tree build (no GPU needed): per kernel, how many wgmma / TMA / vector-reduction
# instructions the SASS holds, and the ptxas resource lines.
#   tools/sass_evidence.sh > sass_evidence.txt
cd "$(dirname "$0")/.."
echo "# SASS evidence (cuobjdump -sass of the in-tree build, sm_90a): instruction counts per kernel"
for o in build/mlp.o build/raster_fwd.o build/raster_bwd.o build/mc.o build/meshrast.o build/densify.o build/loss.o build/dpsr.o build/knn.o; do
  [ -f "$o" ] || continue
  echo "## $o"
  cuobjdump -sass "$o" 2>/dev/null | awk '
    /Function :/ {fn=$3}
    /HGMMA|WARPGROUP|UBLKCP|SYNCS|REDG|ATOMG|REDUX|MUFU.EX2/ {
      for (i=1;i<=NF;i++) if ($i ~ /^(HGMMA|WARPGROUP|UBLKCP|SYNCS|REDG|ATOMG|REDUX|MUFU\.EX2)/) {split($i,a,"."); c[fn" "a[1]]++}
    }
    END {for (k in c) printf "  %-90s x%d\n", k, c[k]}' | sort
done
echo
echo "# ptxas -v (registers / shared memory / spills per kernel)"
for l in build/*.ptxas.log; do
  echo "## $l"
  grep -E "Compiling entry function|Used [0-9]+ registers|spill" "$l" | sed 's/ptxas info    : //' | paste - - - 2>/dev/null | sed -E 's/Compiling entry function .(_Z[A-Za-z0-9_]+). for .sm_100a.//' | head -60
done
