#!/usr/bin/env python
"""The reference's benchmark harness (benchmarks/benchmark.py, benchmarks/utils.py) re-stated for this repo:
same method matrix, same settings grid, forward and backward timed SEPARATELY (backward alone on a retained
graph, benchmark.py:158-198), same FLOPs formula (:17-20) and the same jsonl row the reference writes
(utils.py:73-86: batch_size, seqlen, num_heads, double_ring, dim, method, forward, forward_backward, causal;
times in seconds) -- so both README tables can be regenerated on H100s with one command per table:

  torchrun --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 tools/benchmark_harness.py \
      --seqlens 65536,131072,262144,524288,1048576 --batch 1 --out table_seq.jsonl        (README.md:71-79)
  torchrun ... tools/benchmark_harness.py --seqlens 65536 --batch 1,2,4,8 --out table_batch.jsonl  (:89-103)

Methods: "burst" (burst_attn_func, contiguous / zigzag shards), "burst_striped" (burst_attn_func_striped),
"flash" (single-GPU attention over the FULL sequence on every rank -- the reference uses flash_attn_func, here
it is this repo's own tile kernels with no ring; skipped above --flash-max-seq).  The reference's "ring" and
"normal" methods are its broken / CPU-eager baselines (SURVEY.md App. A.7-8) and have no counterpart.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "burst-attention_b200"))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from burst_attn import burst_attn_func, burst_attn_func_striped  # noqa: E402


def flops(batch, seqlen, nheads, headdim, causal, mode="fwd"):
    f = 4 * batch * seqlen ** 2 * nheads * headdim // (2 if causal else 1)
    return f if mode == "fwd" else (2.5 * f if mode == "bwd" else 3.5 * f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seqlens", default="65536,262144")
    ap.add_argument("--batch", default="1")
    ap.add_argument("--heads", type=int, default=32)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--methods", default="burst,burst_striped,flash")
    ap.add_argument("--causal", default="0,1")
    ap.add_argument("--double-ring", type=int, default=0, help="intra-node ring size L (0: flat ring only)")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "fp16"])
    ap.add_argument("--flash-max-seq", type=int, default=262144)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    world, rank, local = (int(os.environ.get(k, d)) for k, d in (("WORLD_SIZE", 1), ("RANK", 0), ("LOCAL_RANK", 0)))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    dtype = torch.bfloat16 if a.dtype == "bf16" else torch.float16
    double_group = [None, None]
    if a.double_ring and world > 1:
        os.environ["BA_DOUBLE_RING"] = "1"
        L = a.double_ring
        rows = [list(range(n * L, (n + 1) * L)) for n in range(world // L)]
        mk = lambda ranks: dist.new_subgroups_by_enumeration(ranks, backend="nccl")[0]  # noqa: E731
        double_group = [mk(rows), mk([list(c) for c in zip(*rows)])]

    # "flash": every rank alone over the full sequence -> a one-rank group (new_group is collective: all ranks
    # create all groups)
    self_group = None
    if world > 1 and "flash" in a.methods.split(","):
        self_group = [dist.new_group([r]) for r in range(world)][rank]

    def timed(fn, n):
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1) / n / 1e3], device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    out_f = open(a.out, "a") if (a.out and rank == 0) else None
    for b in [int(x) for x in a.batch.split(",")]:
        for S in [int(x) for x in a.seqlens.split(",")]:
            for causal in [bool(int(x)) for x in a.causal.split(",")]:
                for method in a.methods.split(","):
                    if method == "burst_striped" and not causal:
                        continue  # identical to burst when nothing is masked
                    if method == "flash" and S > a.flash_max_seq:
                        continue
                    s_loc = S if method == "flash" else S // world
                    func = burst_attn_func_striped if method == "burst_striped" else burst_attn_func
                    g = torch.Generator(device=dev).manual_seed(1234 + rank)
                    q, k, v, do = (torch.randn(b, s_loc, a.heads, a.dim, device=dev, generator=g).to(dtype) for _ in range(4))
                    q, k, v = (t.requires_grad_() for t in (q, k, v))
                    grp = self_group if method == "flash" else None

                    def fwd():
                        return func(q, k, v, None, "cuda", causal, True, False, grp,
                                    [None, None] if method == "flash" else double_group)

                    for _ in range(a.warmup):
                        torch.autograd.grad(fwd(), (q, k, v), do)
                    with torch.no_grad():
                        t_f = timed(fwd, a.iters)
                    o = fwd()
                    t_b = timed(lambda: torch.autograd.grad(o, (q, k, v), do, retain_graph=True), a.iters)
                    ratio = 1 if method == "flash" else world
                    row = {"batch_size": b, "seqlen": S, "num_heads": a.heads, "double_ring": bool(a.double_ring),
                           "dim": a.dim, "method": method, "forward": t_f, "forward_backward": t_f + t_b,
                           "causal": causal,
                           # beyond the reference's row: what its print_rank lines show
                           "backward": t_b, "world": world, "dtype": a.dtype,
                           "fwd_tflops_per_gpu": flops(b, S, a.heads, a.dim, causal, "fwd") / t_f / 1e12 / ratio,
                           "bwd_tflops_per_gpu": flops(b, S, a.heads, a.dim, causal, "bwd") / t_b / 1e12 / ratio,
                           "fwd_bwd_tflops_per_gpu": flops(b, S, a.heads, a.dim, causal, "fwd_bwd") / (t_f + t_b) / 1e12 / ratio}
                    if rank == 0:
                        print(json.dumps(row), flush=True)
                        if out_f:
                            out_f.write(json.dumps(row) + "\n")
                            out_f.flush()
                    del q, k, v, do, o
                    torch.cuda.empty_cache()
    if world > 1:
        dist.barrier()
        from burst_attn import comm
        comm.destroy_rings()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
