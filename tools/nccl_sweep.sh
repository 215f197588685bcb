#!/bin/bash
# A/B NCCL P2P settings for the ring at small S_local (2 GPUs, S_local = 8192): prints non-kernel fraction
OUT=${OUT:-session_out}
mkdir -p "$OUT"
run() {
  tag=$1; shift
  env "$@" timeout 150 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
      --master-port 295$((RANDOM % 90 + 10)) bench.py --gpus 2 --steps 10 --warmup 3 --no-cpu --no-e2e --configs 16384,32768 \
      > $OUT/nccl_$tag.json 2> $OUT/nccl_$tag.err
  python - "$tag" <<PY
import json, sys
tag = sys.argv[1]
for line in open(f"$OUT/nccl_{tag}.json"):
    if not line.startswith('{"metric'): continue
    d = json.loads(line); o = d["overlap"]
    print(tag, d["config"]["seq_len"], "ms/step %.3f" % d["ms_per_step"], "kernel %.3f" % o["kernel_ms_per_step"],
          "non-kernel %.1f%%" % (100 * o["non_kernel_frac"]), "tflops %.0f" % d["value"], flush=True)
PY
}
run base X=1
run minch16 NCCL_MIN_P2P_NCHANNELS=16
run minch32 NCCL_MIN_P2P_NCHANNELS=32
run ce NCCL_P2P_USE_CUDA_MEMCPY=1
