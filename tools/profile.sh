#!/bin/bash
# Profiling recipe (Nsight Compute), 1 GPU.  Raw outputs go to $OUT (default prof_out/, git-ignored); afterwards,
# on any machine:
#   python tools/ncu_traffic.py prof_out/prof_${TAG}_*.ncu-rep       -> profiles/ncu_traffic.json (bench.py's traffic)
#   python tools/ncu_summary.py prof_out/prof_${TAG}_bwd_...ncu-rep  -> per-kernel summary on stdout
set -x
OUT=${OUT:-prof_out}
mkdir -p "$OUT"
TAG=${1:-r02}
# 1. every launch with its device time (cold-cache, serialised: compare SHARES)
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 200 --csv \
    --log-file $OUT/launches_${TAG}.csv python bench.py --seq 65536 --steps 2 --warmup 3 --no-e2e --no-cpu --no-parity \
    > $OUT/launches_${TAG}.out 2>&1
# 2. one full capture per tile kernel and launch shape the bench uses: N=8 ring round (Sq = Sk = 32768) and the
#    N=1 L2-blocked sub-launches (fwd: all rows x one K/V block; bwd: one row block x all keys)
cap() {  # kernel Sq Sk
  timeout 900 ncu --set full --clock-control none --import-source on -k regex:$1_chunk_kernel -s 1 -c 1 \
      -o $OUT/prof_${TAG}_$1_Sq$2_Sk$3_H32_c0 -f python tools/launch_one.py --kernel $1 --Sq $2 --Sk $3 --n 1 \
      > $OUT/prof_${TAG}_$1_$2_$3.out 2>&1
}
cap bwd 32768 32768
cap fwd 32768 32768
if [ "${2:-}" = "all" ]; then
  cap bwd 32768 262144
  cap fwd 262144 32768
fi
ls -la "$OUT"
