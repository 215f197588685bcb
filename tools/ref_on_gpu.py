#!/usr/bin/env python
"""The UNMODIFIED reference (MayDomine/Burst-Attention, copied by build() into the git-ignored
``oracle/_ref``) on this machine's GPUs: ``burst_attn_func(q, k, v, None, "cuda", causal, optimize_bwd_comm=False)``
through its own ring (torch backend, ``dist.batch_isend_irecv``) and its own kernels (the flash-attn wheel of
this image, FA2 ``mma.sync``), timed like ``bench.py`` times ours -- the denominator of BASELINE.json's
"north_star" target (>= 1.5x the reference's own 8xGPU fwd+bwd at seq 262144 on the same box; BASELINE.md 4).

Nothing of the reference is edited.  Two shims make its imports resolve in this image (SURVEY.md 8c):
  * ``bmtrain`` is absent -> a stub module; the reference then picks its torch backend
    (burst_attn/comm.py:36-37,106-114);
  * the reference calls flash-attn's PRIVATE entry points with the signature of flash-attn <= 2.5
    (burst_attn/burst_utils.py:150-160,211-248: ``window_size=(-1,-1)``, 8 return values); flash-attn 2.8.3
    split ``window_size``, added ``softcap`` and returns 4 values -> two adapter functions are installed on
    ``flash_attn.flash_attn_interface`` BEFORE the reference imports them.
``optimize_bwd_comm=True`` needs a patched flash-attn (``softmax_d``, burst_utils.py:203-210) that does not exist
here, so the reference runs its stock O-travels backward.

  torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 tools/ref_on_gpu.py --seq 262144 [--causal]
prints one JSON line (rank 0).  None of this repo's kernels or drivers are imported.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
H, D = 32, 128


def load_reference():
    sys.path.insert(0, os.path.join(ROOT, "baseline"))
    import ref_shim
    mod = ref_shim.load()  # bmtrain stub + flash-attn 2.8.3 adapters + the package under the alias burst_attn_ref
    assert os.path.realpath(mod.__file__).startswith(os.path.realpath(REF)), mod.__file__
    return mod.burst_attn_func


def shard(t, rank, world, layout):
    if layout == "contiguous":
        return t.chunk(world, dim=1)[rank].contiguous()
    c = t.chunk(2 * world, dim=1)  # zigzag halves {i, 2W-1-i} (reference test/test_burst.py:46-52)
    return torch.cat([c[rank], c[2 * world - 1 - rank]], dim=1).contiguous()


def dense_fp32(q, k, v, do, causal):
    q, k, v = (t.float().permute(0, 2, 1, 3).detach().requires_grad_() for t in (q, k, v))
    s = (q @ k.transpose(-1, -2)) * D ** -0.5
    if causal:
        S = s.shape[-1]
        s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool, device=s.device).tril(), float("-inf"))
    o = torch.softmax(s, -1) @ v
    g = torch.autograd.grad(o, (q, k, v), do.float().permute(0, 2, 1, 3))
    return [t.permute(0, 2, 1, 3) for t in (o, *g)]


def parity(func, rank, world, dev):
    """The reference's own protocol (test/test_burst.py:159-219) against fp32 dense attention: proves the two
    shims did not change what the reference computes."""
    ok = True
    for causal in (False, True):
        g = torch.Generator().manual_seed(7)
        q, k, v, do = (torch.randn(2, 256 * world, 8, D, generator=g).to(torch.float16).to(dev) for _ in range(4))
        ref = dense_fp32(q, k, v, do, causal)
        layout = "zigzag" if causal else "contiguous"
        ql, kl, vl = (shard(t, rank, world, layout).requires_grad_() for t in (q, k, v))
        o = func(ql, kl, vl, None, "cuda", causal, False, False, None)
        grads = torch.autograd.grad(o, (ql, kl, vl), shard(do, rank, world, layout))
        for got, r in zip((o, *grads), ref):
            ok &= torch.allclose(got.float(), shard(r, rank, world, layout), rtol=1e-3, atol=1e-2)
    flag = torch.tensor([0 if ok else 1], device=dev)
    if world > 1:
        dist.all_reduce(flag)
    return flag.item() == 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq", type=int, default=262144)
    ap.add_argument("--causal", action="store_true")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    world, rank, local = (int(os.environ.get(k, d)) for k, d in (("WORLD_SIZE", 1), ("RANK", 0), ("LOCAL_RANK", 0)))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29541")
    dist.init_process_group("nccl", device_id=dev, rank=rank, world_size=world)  # the reference's ring needs one
    func = load_reference()
    par = parity(func, rank, world, dev)

    S, S_loc = args.seq, args.seq // world
    gen = torch.Generator(device=dev).manual_seed(1234 + rank)
    mk = lambda: torch.randn(1, S_loc, H, D, device=dev, generator=gen, dtype=torch.float32).to(torch.bfloat16)
    q, k, v, do = mk(), mk(), mk(), mk()

    def step():
        qq, kk, vv = (t.detach().requires_grad_() for t in (q, k, v))
        o = func(qq, kk, vv, None, "cuda", args.causal, False, False, None)
        return torch.autograd.grad(o, (qq, kk, vv), do)

    def fwd_only():
        with torch.no_grad():
            return func(q, k, v, None, "cuda", args.causal, False, False, None)

    def timed(fn, n):
        dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        dist.barrier()
        torch.cuda.synchronize()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item()) / n

    for _ in range(args.warmup):
        step()
    ms = timed(step, args.steps)
    ms_f = timed(fwd_only, args.steps)
    div = 2.0 if args.causal else 1.0
    fl = 4.0 * S * S * H * D / div
    if rank == 0:
        import flash_attn
        line = {"impl": "reference-on-gpu", "what": "unmodified reference burst_attn_func(flash='cuda', optimize_bwd_comm=False) "
                f"from oracle/_ref, flash-attn {flash_attn.__version__} kernels, torch-backend ring",
                "n_gpus": world, "seq": S, "causal": args.causal, "dtype": "bf16", "steps": args.steps,
                "warmup": args.warmup, "ms_per_step": ms, "fwd_ms": ms_f,
                "fwd_bwd_tflops": 3.5 * fl / (ms * 1e-3) / 1e12, "fwd_tflops": fl / (ms_f * 1e-3) / 1e12,
                "fwd_bwd_tflops_per_gpu": 3.5 * fl / (ms * 1e-3) / 1e12 / world,
                "parity_vs_fp32_dense_fp16_ref_tolerances": par}
        s = json.dumps(line)
        print(s, flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(s + "\n")
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
