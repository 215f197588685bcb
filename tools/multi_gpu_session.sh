#!/bin/bash
# One multi-GPU session (N = number of GPUs of the machine): parity first, then numbers.  Outputs go to $OUT
# (default session_out/, git-ignored).
#   bash tools/multi_gpu_session.sh 2 r02
#   bash tools/multi_gpu_session.sh 8 r02
# Everything is wrapped in `timeout`: a transport that hangs costs its own limit, not the session.
N=${1:-2}; TAG=${2:-r02}
OUT=${OUT:-session_out}
mkdir -p "$OUT"
python -c "import torch; print(torch.cuda.device_count(), torch.cuda.get_device_name(0))"  # pages the image in (can take minutes on a cold box)
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1"
port() { echo $((29500 + RANDOM % 400)); }
run() { echo "=== $*"; "$@"; echo "--- rc=$?"; }

# (the copy-engine ring is the default on one node; the NCCL steps name their transport)
# 1. ring parity, reference protocol: flat ring over NCCL (+ hierarchical rings when N >= 4)
DBL=""; [ "$N" -ge 4 ] && DBL="2"; [ "$N" -ge 8 ] && DBL="2,4"
BA_RING_TRANSPORT=nccl RING_CHECK_DOUBLE=$DBL run timeout 300 $TR --master-port $(port) tests/ring_check.py > $OUT/ring_check_${TAG}_n${N}_nccl.txt 2>&1
grep -E "ring_check|MISMATCH|Error|rc=" $OUT/ring_check_${TAG}_n${N}_nccl.txt | tail -20
# 2. the same over the copy-engine transport (first runs of csrc/ring_ce.cu): short timeout
BA_RING_TRANSPORT=ce run timeout 180 $TR --master-port $(port) tests/ring_check.py > $OUT/ring_check_${TAG}_n${N}_ce.txt 2>&1
grep -E "ring_check|MISMATCH|Error|rc=" $OUT/ring_check_${TAG}_n${N}_ce.txt | tail -14
CE_OK=0; grep -q "rc=0" $OUT/ring_check_${TAG}_n${N}_ce.txt && ! grep -q FAIL $OUT/ring_check_${TAG}_n${N}_ce.txt && CE_OK=1
echo "CE_OK=$CE_OK"

# 3. the reference itself on this box (the north-star denominator is its 8-GPU number; smaller N for the record)
run timeout 400 $TR --master-port $(port) tools/ref_on_gpu.py --seq 262144 --steps 3 --warmup 2 --out $OUT/ref_on_gpu_${TAG}.json > $OUT/ref_on_gpu_${TAG}_n${N}_c3.log 2>&1
if [ "$N" -ge 8 ]; then
  run timeout 300 $TR --master-port $(port) tools/ref_on_gpu.py --seq 524288 --causal --steps 2 --warmup 1 --out $OUT/ref_on_gpu_${TAG}.json > $OUT/ref_on_gpu_${TAG}_n${N}_c4.log 2>&1
fi
cat $OUT/ref_on_gpu_${TAG}.json; tail -3 $OUT/ref_on_gpu_${TAG}_n${N}_c3.log

# 4. bench: flat ring over NCCL (headline config first, with e2e and the comm A/B), then the other configurations
CFG="65536,524288c"; [ "$N" -ge 8 ] && [ "${FULL:-0}" = 1 ] && CFG="65536,524288c,1048576"
BA_RING_TRANSPORT=nccl run timeout 400 $TR --master-port $(port) bench.py --gpus $N --steps 3 --warmup 3 > $OUT/bench_${TAG}_n${N}_nccl.json 2> $OUT/bench_${TAG}_n${N}_nccl.err
BA_RING_TRANSPORT=nccl run timeout 500 $TR --master-port $(port) bench.py --gpus $N --steps 2 --warmup 3 --no-e2e --no-parity --configs $CFG > $OUT/bench_${TAG}_n${N}_nccl_cfg.json 2> $OUT/bench_${TAG}_n${N}_nccl_cfg.err
# 4b. NCCL's send/recv kernels are SM-resident and slow the tile kernels down while they co-run (round 1: fwd +8.7 %
#     at N = 8); the ring needs < 100 GB/s per hop, so cap the CTAs NCCL may use
for c in ${NCCL_CTAS:-2 4}; do
  BA_RING_TRANSPORT=nccl BA_NCCL_MAX_CTAS=$c run timeout 300 $TR --master-port $(port) bench.py --gpus $N --steps 3 --warmup 3 --no-e2e --no-parity > $OUT/bench_${TAG}_n${N}_ncclcta${c}.json 2> $OUT/bench_${TAG}_n${N}_ncclcta${c}.err
done
# 5. the same over the copy engines
if [ "$CE_OK" = 1 ]; then
  BA_RING_TRANSPORT=ce run timeout 400 $TR --master-port $(port) bench.py --gpus $N --steps 3 --warmup 3 --no-e2e --configs 262144,65536 > $OUT/bench_${TAG}_n${N}_ce.json 2> $OUT/bench_${TAG}_n${N}_ce.err
fi
# 6. hierarchical ring beside the flat one
if [ "$N" -ge 4 ]; then
  run timeout 300 $TR --master-port $(port) bench.py --gpus $N --steps 3 --warmup 3 --no-e2e --no-parity --double-ring $((N / 2)) > $OUT/bench_${TAG}_n${N}_double.json 2> $OUT/bench_${TAG}_n${N}_double.err
fi
python - <<PY
import json, glob
for f in sorted(glob.glob("$OUT/bench_${TAG}_n${N}_*.json")):
    for l in open(f):
        if not l.startswith('{"metric'): continue
        d = json.loads(l); o = d.get("overlap") or {}; r = d.get("roofline") or {}
        print(f.split("/")[-1], d["config"]["seq_len"], "causal" if "causal zig" in d["config"]["workload"] else "", "TFLOPS %.0f" % d["value"],
              "ms %.1f" % d["ms_per_step"], "fwd %.0f" % d["fwd_tflops"], "nonk %.2f%%" % (100 * o.get("non_kernel_frac", 0)),
              "bwdk %.0f" % r.get("achieved", 0), "fwdk %.0f" % (r.get("fwd_kernel") or {}).get("achieved", 0),
              "parity", (d.get("parity") or {}).get("ok"), "ab", (d.get("comm_ab") or {}).get("exposed_comm_frac"),
              "e2e", (d.get("e2e") or {}).get("value"))
PY
