#!/bin/bash
# Counts the SASS mnemonics that show which hardware paths each object of libgeob200.so uses:
#   HGMMA = wgmma.mma_async (warpgroup tensor-core MMA), UTMALDG = cp.async.bulk.tensor (TMA tiled load),
#   UBLKCP = cp.async.bulk (TMA 1-D bulk copy), SYNCS = mbarrier ops, LDGSTS = cp.async (per-thread),
#   HMMA/IMMA/DMMA = warp-level mma.sync (expected 0: the tensor-core kernels use wgmma).
# usage: tools/sass_mnemonics.sh   (after the build)
cd "$(dirname "$0")/../geotransformer_b200/csrc" || exit 1
echo "cuobjdump -sass of every object linked into geotransformer_b200/libgeob200.so (nvcc $(nvcc --version | grep -o 'release [0-9.]*'), -gencode arch=compute_90a,code=sm_90a)"
printf "%-18s %8s %8s %7s %6s %7s %11s\n" object HGMMA UTMALDG UBLKCP SYNCS LDGSTS warp_mma
for f in *.o; do
  cuobjdump -sass "$f" 2>/dev/null | awk -v name="$f" '
    / HGMMA/{a++} / UTMALDG/{t++} / UBLKCP/{b++} / SYNCS/{s++} / LDGSTS/{g++}
    /[ .]HMMA|[ .]IMMA|[ .]DMMA/{ m++ }
    END{printf "%-18s %8d %8d %7d %6d %7d %11d\n", name, a, t, b, s, g, m}'
done
