#!/bin/bash
# Which Hopper staging / synchronisation instructions the shipped kernels contain, printed to stdout (needs cuobjdump; no GPU)
cd "$(dirname "$0")/.."
echo "# SASS evidence: cuobjdump -sass of the NVRTC-built sm_90a cubins that build() leaves in datafusion-comet_b200/.jitcache (the benchmark plans) -- per kernel the"
echo "# staging instructions: UBLKCP = cp.async.bulk (TMA 1-D bulk copy global -> shared), SYNCS = mbarrier ops (arrive.expect_tx / try_wait), ELECT = elect.sync; global atomics / REDs and shuffles."
for f in datafusion-comet_b200/.jitcache/*.cubin; do
  cuobjdump -sass $f 2>/dev/null | awk -v F=$(basename $f | cut -c1-20) '/Function :/ {fn=$3} /UBLKCP/ {u[fn]++} /SYNCS/ {s[fn]++} /ELECT/ {e[fn]++} /ATOMG|REDG/ {a[fn]++} /SHFL/ {sh[fn]++} END {for (k in s) printf "%s  %-20s sm_90a  UBLKCP %3d  SYNCS %3d  ELECT %2d  ATOMG/REDG %3d  SHFL %3d\n", F, k, u[k], s[k], e[k], a[k], sh[k]}'
done
echo "# AOT kernels in libcomet_b200.so (nvcc -gencode arch=compute_90a,code=sm_90a):"
cuobjdump -sass datafusion-comet_b200/libcomet_b200.so 2>/dev/null | awk '/Function :/ {fn=$3} /MATCH/ {m[fn]++} /SHFL/ {sh[fn]++} /ATOMS|ATOMG|REDG/ {a[fn]++} /LDS|STS/ {l[fn]++} /EXIT/ {x[fn]++} END {for (k in x) printf "  %-64s SHFL %3d MATCH %2d atomics %3d LDS/STS %4d\n", substr(k,1,64), sh[k], m[k], a[k], l[k]}' | sort
