"""Sliding-window attention: fwd+bwd time and TFLOP/s over the visible (query, key) pairs, per window.

    python tools/bench_window.py [--seq 65536,262144] [--left 1024,4096,16384,-1] [--steps 10] [--warmup 3]
    torchrun --nproc-per-node=N tools/bench_window.py --ring ...     (burst_attn_func over N GPUs, zigzag shards)

Workload: bf16, d = 128, bs = 1, H = 32, causal, window_size = (left, 0); left = -1 is full causal attention.  One GPU:
flash_attn_func on the whole sequence; --ring: burst_attn_func on this rank's zigzag shard.  Each step (forward +
backward) is timed with CUDA events, windows alternating step by step after warm-up.  FLOPs count the visible pairs
only: 4 d per pair and head forward, 10 d backward (bench.py's model).  Prints one JSON line per (S, left) with the
median / min ms per step and TFLOP/s, then the card name, power limit and SM clock read in the same process; rank 0 only.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "burst-attention_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from burst_attn import burst_attn_func  # noqa: E402
from burst_attn.flash_triton import flash_attn_func  # noqa: E402
from oracle.attention_oracle import shard  # noqa: E402

H, D = 32, 128


def _device_info(dev):
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        idx = dev.index if dev.index is not None else 0
        out = subprocess.run(["nvidia-smi", f"--id={idx}", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, sm, smax = (x.strip() for x in out.split(","))
        return {"card": name, "power_limit_w": float(plim), "sm_mhz": int(sm), "sm_max_mhz": int(smax)}
    except Exception as e:  # noqa: BLE001
        return {"card": torch.cuda.get_device_name(dev), "nvidia_smi": f"unavailable ({type(e).__name__})"}


def visible_pairs(S, left):
    """Causal pairs (i, j), j <= i, with i - j <= left (left < 0: no limit)."""
    if left < 0 or left >= S - 1:
        return S * (S + 1) // 2
    return (left + 1) * S - left * (left + 1) // 2


def _step(q, k, v, do, left, ring):
    qq, kk, vv = (t.detach().requires_grad_() for t in (q, k, v))
    w = (left, -1)
    if ring:
        o = burst_attn_func(qq, kk, vv, None, "cuda", True, False, False, None, [None, None], w)
    else:
        o = flash_attn_func(qq, kk, vv, None, True, None, w)
    return torch.autograd.grad(o, (qq, kk, vv), do)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", default="65536", help="comma-separated global sequence lengths")
    ap.add_argument("--left", default="1024,4096,16384,-1")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ring", action="store_true", help="burst_attn_func over the torchrun ranks")
    args = ap.parse_args()

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert torch.cuda.is_available(), "bench_window.py measures on the GPU; there is no CPU path"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if args.ring and world > 1:
        dist.init_process_group("nccl", device_id=dev)
    lefts = [int(x) for x in args.left.split(",")]
    results = []
    for S in (int(x) for x in args.seq.split(",")):
        g = torch.Generator(device=dev).manual_seed(1234)

        def mk():
            full = torch.randn(1, S, H, D, device=dev, generator=g, dtype=torch.bfloat16)
            return shard(full, rank, world, "zigzag").contiguous() if args.ring else full

        q, k, v, do = mk(), mk(), mk(), mk()
        times = {left: [] for left in lefts}
        for i in range(args.warmup + args.steps):
            for left in lefts:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                _step(q, k, v, do, left, args.ring)
                e1.record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[left].append(e0.elapsed_time(e1))
        info = _device_info(dev)
        for left in lefts:
            ms = statistics.median(times[left])
            flops = 14 * D * H * visible_pairs(S, left)  # 4 d forward + 10 d backward per visible pair and head
            results.append({"seq": S, "left": left, "world": world if args.ring else 1, "causal": True,
                            "visible_pairs": visible_pairs(S, left), "ms_per_step": round(ms, 3),
                            "ms_min": round(min(times[left]), 3),
                            "tflops_visible": round(flops / (world if args.ring else 1) / (ms * 1e-3) / 1e12, 1),
                            **info})
        del q, k, v, do
        torch.cuda.empty_cache()
    if rank == 0:
        for r in results:
            print(json.dumps(r), flush=True)
        print(json.dumps({"device": _device_info(dev), "torch": torch.__version__}), flush=True)
    if args.ring and world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
