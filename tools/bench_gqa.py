"""Grouped-query attention: native GQA against the workaround it replaces, fwd+bwd, same process, alternating.

    python tools/bench_gqa.py [--seq S] [--hkv 32,8,1] [--steps 10] [--warmup 3] [--causal]
    torchrun --nproc-per-node=N tools/bench_gqa.py ...            (ring over N GPUs, S = 262144 by default)

Workload: bf16, d = 128, bs = 1, Hq = 32, Hkv in --hkv; S = 65536 on one GPU, 262144 over N (S / N per rank).
  native     : burst_attn_func(q, k, v) with k, v of Hkv heads
  workaround : k, v repeat_interleave'd to Hq heads, the MHA call, dK / dV summed back over each group
Both are timed per step with CUDA events (forward + backward, including the expand and the group sum), alternating
step by step after warm-up.  Reported per (Hkv, variant): median / min ms per step, fwd+bwd TFLOP/s (FLOPs as for
MHA with Hq heads), per-kernel times from NativeOps.enable_timing (one extra step), peak device memory of one step,
and the forward hop bytes computed from shapes.  The card name, power limit and SM clock are read in the same call.
Prints one JSON line per (Hkv, variant) and a final line with the device; rank 0 only.
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
from burst_attn.chunk_ops import get_ops  # noqa: E402
from oracle.attention_oracle import attention_flops, shard  # noqa: E402

HQ, D = 32, 128


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


def _step(variant, q, k, v, do, causal, G):
    """One fwd+bwd; returns the gradients with the shapes of q, k, v."""
    qq, kk, vv = (t.detach().requires_grad_() for t in (q, k, v))
    if variant == "native" or G == 1:
        o = burst_attn_func(qq, kk, vv, None, "cuda", causal)
        return torch.autograd.grad(o, (qq, kk, vv), do)
    ke, ve = kk.repeat_interleave(G, dim=2), vv.repeat_interleave(G, dim=2)
    o = burst_attn_func(qq, ke, ve, None, "cuda", causal)
    dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)  # autograd of repeat_interleave = the group sum
    return dq, dk, dv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=None, help="global sequence length (default 65536 / 262144 on N>1)")
    ap.add_argument("--hkv", default="32,8,1")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--causal", action="store_true")
    args = ap.parse_args()

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert torch.cuda.is_available(), "bench_gqa.py measures on the GPU; there is no CPU path"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    S = args.seq or (65536 if world == 1 else 262144)
    assert S % (2 * world) == 0
    s_loc = S // world
    layout = "zigzag" if args.causal else "contiguous"
    ops = get_ops()

    results = []
    for hkv in (int(x) for x in args.hkv.split(",")):
        assert HQ % hkv == 0
        G = HQ // hkv
        g = torch.Generator(device=dev).manual_seed(1234 + hkv)

        def mk(h):
            full = torch.randn(1, s_loc * world, h, D, device=dev, generator=g, dtype=torch.bfloat16)
            return shard(full, rank, world, layout).contiguous()

        q, do, k, v = mk(HQ), mk(HQ), mk(hkv), mk(hkv)
        variants = ["native"] if G == 1 else ["native", "workaround"]
        times = {vname: [] for vname in variants}
        for i in range(args.warmup + args.steps):
            for vname in variants:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                _step(vname, q, k, v, do, args.causal, G)
                e1.record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[vname].append(e0.elapsed_time(e1))
        info = _device_info(dev)  # read right after the timed steps
        for vname in variants:
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            base = torch.cuda.memory_allocated(dev)
            torch.cuda.reset_peak_memory_stats(dev)
            ops.enable_timing(True)
            _step(vname, q, k, v, do, args.causal, G)
            torch.cuda.synchronize()
            kern = {name: {"launches": n, "ms": round(ms, 3)} for name, (n, ms) in ops.kernel_ms().items()}
            ops.enable_timing(False)
            peak = torch.cuda.max_memory_allocated(dev) - base
            ms = statistics.median(times[vname])
            heads_on_wire = hkv if vname == "native" else HQ
            flops = attention_flops(1, S, HQ, D, args.causal, "fwd_bwd")
            results.append({
                "hkv": hkv, "hq": HQ, "variant": vname, "world": world, "seq": S, "causal": args.causal,
                "ms_per_step": round(ms, 3), "ms_min": round(min(times[vname]), 3),
                "ms_all": [round(t, 3) for t in times[vname]],
                "tflops": round(flops / world / (ms * 1e-3) / 1e12, 1),
                "peak_mem_gib": round(peak / 2 ** 30, 3),
                "fwd_hop_bytes": 2 * s_loc * heads_on_wire * D * 2 if world > 1 else 0,
                "kernels": kern, **info})
    if rank == 0:
        for r in results:
            print(json.dumps(r), flush=True)
        print(json.dumps({"device": _device_info(dev), "torch": torch.__version__}), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
