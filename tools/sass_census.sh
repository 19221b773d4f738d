#!/bin/bash
# SASS census of the shipped library: how many wgmma / TMA / mbarrier instructions each kernel holds (no GPU needed).
# usage: bash tools/sass_census.sh [libcenterpose_b200.so]
SO=${1:-centerpose_b200/lib/libcenterpose_b200.so}
echo "# $(basename $SO): per kernel — HGMMA (wgmma.mma_async), UTMALDG (TMA loads), WARPGROUP (wgmma fence / arrive / wait), SYNCS (mbarrier), total SASS instructions"
cuobjdump -sass "$SO" | awk '
  /Function :/ { name = $3 }
  /^ +\/\*[0-9a-f]+\*\/ / { tot[name]++ }
  /HGMMA/ { mma[name]++ } /UTMALDG/ { tma[name]++ } /WARPGROUP/ { wg[name]++ } /SYNCS/ { sy[name]++ }
  END { for (n in tot) if (mma[n] + tma[n] > 0) printf "%5d %5d %5d %5d %6d  %s\n", mma[n], tma[n], wg[n], sy[n], tot[n], n }' | sort -k6 | c++filt
