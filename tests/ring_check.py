"""Multi-GPU parity check of the ring path (run under torchrun, one rank per GPU):
the reference's own protocol (test/test_burst.py:159-219): b=2, s=256*W, n=32, d=128,
fp16, full-sequence oracle, shard with get_chunk, rtol=1e-3/atol=1e-2 -- for the
non-causal, zigzag-causal and striped-causal drivers, fwd + bwd."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "burst-attention_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from burst_attn import burst_attn_func, burst_attn_func_striped  # noqa: E402
from oracle import attention_oracle as orc  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    fails = run_cases(rank, world, dev)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)
    # (to follow the parity cases with bench configurations in one expensive multi-GPU session, launch
    #  bench.py --configs ... as a second torchrun command in the same job)


def _double_group(world, intra):
    """[(intra, intra_dq), (inter, inter_dq)] as the reference's get_group builds them (test_burst.py:120-156)."""
    rows = [list(range(n * intra, (n + 1) * intra)) for n in range(world // intra)]
    cols = [list(c) for c in zip(*rows)]
    mk = lambda ranks: dist.new_subgroups_by_enumeration(ranks, backend="nccl")[0]  # noqa: E731
    return [(mk(rows), mk(rows)), (mk(cols), mk(cols))]


def run_cases(rank, world, dev):
    n_heads = int(os.environ.get("RING_CHECK_HEADS", "8"))
    fails = 0
    # RING_CHECK_DOUBLE=<intra sizes, comma list>: run every case over the hierarchical (double) ring as well
    # (intra-node rings of L consecutive ranks, reference test/test_burst.py:120-156).
    fails += _run_cases(rank, world, dev, n_heads, [None, None])
    for tok in os.environ.get("RING_CHECK_DOUBLE", "").split(","):
        intra = int(tok) if tok.strip() else 0
        if intra and world % intra == 0 and 1 < intra < world:
            os.environ["BA_DOUBLE_RING"] = "1"
            fails += _run_cases(rank, world, dev, n_heads, _double_group(world, intra), f"double L={intra}")
    return fails


def _run_cases(rank, world, dev, n_heads, double_group, tag="flat"):
    fails = 0
    for dtype, tol in ((torch.float16, dict(rtol=1e-3, atol=1e-2)), (torch.bfloat16, dict(rtol=1.6e-2, atol=2e-2))):
        for name, func, causal, layout in (("none", burst_attn_func, False, "contiguous"),
                                           ("zigzag", burst_attn_func, True, "zigzag"),
                                           ("striped", burst_attn_func_striped, True, "striped")):
            g = torch.Generator().manual_seed(7)  # identical full tensors on every rank
            b, s, n, d = 2, 256 * world, n_heads, 128
            q, k, v, do = (torch.randn(b, s, n, d, generator=g).to(dtype) for _ in range(4))
            o_ref, _, dq_ref, dk_ref, dv_ref = orc.dense_attention_bwd(q, k, v, do, None, causal)
            sh = lambda t: orc.shard(t, rank, world, layout).to(dev)
            ql, kl, vl = (sh(t).requires_grad_() for t in (q, k, v))
            k_before = kl.detach().clone()
            o = func(ql, kl, vl, None, "cuda", causal, True, False, None, double_group)
            dq, dk, dv = torch.autograd.grad(o, (ql, kl, vl), sh(do))
            torch.cuda.synchronize()
            ok = True
            for nm, got, ref in (("o", o, o_ref), ("dq", dq, dq_ref), ("dk", dk, dk_ref), ("dv", dv, dv_ref)):
                r = orc.shard(ref, rank, world, layout)
                try:
                    torch.testing.assert_close(got.detach().double().cpu(), r, **tol)
                except AssertionError as e:
                    ok = False
                    print(f"[rank {rank}] {name} {dtype} {nm} MISMATCH: {str(e).splitlines()[-3:]}", flush=True)
            if not torch.equal(kl.detach(), k_before):
                ok = False
                print(f"[rank {rank}] {name}: user k was clobbered", flush=True)
            flag = torch.tensor([0 if ok else 1], device=dev)
            dist.all_reduce(flag)
            if rank == 0:
                print(f"ring_check W={world} {tag:10s} {os.environ.get('BA_RING_TRANSPORT', 'nccl'):4s} {name:8s} {str(dtype):15s} {'PASS' if flag.item() == 0 else 'FAIL'}", flush=True)
            fails += int(flag.item())
    return fails


if __name__ == "__main__":
    main()
