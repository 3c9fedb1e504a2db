#!/bin/bash
# Regenerate profiles/sass_evidence.txt: counts of the SASS mnemonics that prove which hardware paths the
# kernels use (wgmma = HGMMA/WARPGROUP, TMA = UTMALDG/UBLKCP, one-sided pushes = REDG,
# mbarriers = SYNCS, peer pulls = LDG.E.128, shared-memory selection = ATOMS, warp reductions = SHFL).
OUT=profiles/sass_evidence.txt
echo "# SASS evidence (cuobjdump -sass of the in-tree objects, sm_90a)" > $OUT
for o in flink-parameter-server_b200/ops/build/*.o; do
  echo >> $OUT; echo "## $(basename $o)" >> $OUT
  cuobjdump -sass $o 2>/dev/null | grep -oE "\b(HGMMA[.0-9A-Za-z]*|WARPGROUP[.A-Z]*|UTMALDG[.0-9A-Z]*|UBLKCP[.A-Z]*|REDG[.A-Za-z0-9_]*|ATOMG[.A-Za-z0-9_]*|ATOMS[.A-Za-z0-9_]*|SYNCS[.A-Z0-9]*|LDG\.E\.128[.A-Z]*|SHFL\.[A-Z]*|FMNMX[0-9]*|MEMBAR[.A-Z]*|LD\.E[.A-Z0-9]*SYS|ST\.E[.A-Z0-9]*SYS)\b" | sort | uniq -c | sort -rn >> $OUT
done
wc -l $OUT
