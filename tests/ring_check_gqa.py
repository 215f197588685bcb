"""Multi-GPU parity check of grouped-query attention on the ring path (run under torchrun, one rank per GPU): the
reference's protocol (b=2, s=256*W, d=128, full-sequence fp64 oracle, shard with get_chunk, fp16 rtol=1e-3 /
atol=1e-2) with Hq = 8 query heads and Hkv in {2, 1} K/V heads, for the non-causal, zigzag-causal and
striped-causal drivers, fwd + bwd, over NCCL and over the copy-engine transport, and over the hierarchical ring
(intra-node rings of 2) at W >= 4.  The oracle runs on K/V expanded to Hq heads; dK / dV are its group sums."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "burst-attention_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from burst_attn import burst_attn_func, burst_attn_func_striped  # noqa: E402
from oracle import attention_oracle as orc  # noqa: E402
from ring_check import _double_group  # noqa: E402

HQ = 8


def _run_cases(rank, world, dev, double_group, tag):
    fails = 0
    for hkv in (2, 1):
        G = HQ // hkv
        for dtype, tol in ((torch.float16, dict(rtol=1e-3, atol=1e-2)), (torch.bfloat16, dict(rtol=1.6e-2, atol=2e-2))):
            for name, func, causal, layout in (("none", burst_attn_func, False, "contiguous"),
                                               ("zigzag", burst_attn_func, True, "zigzag"),
                                               ("striped", burst_attn_func_striped, True, "striped")):
                g = torch.Generator().manual_seed(7)  # identical full tensors on every rank
                b, s, d = 2, 256 * world, 128
                q, do = (torch.randn(b, s, HQ, d, generator=g).to(dtype) for _ in range(2))
                k, v = (torch.randn(b, s, hkv, d, generator=g).to(dtype) for _ in range(2))
                kr, vr = (t.double().requires_grad_() for t in (k, v))
                qr = q.double().requires_grad_()
                o_ref, _ = orc.dense_attention(qr, kr.repeat_interleave(G, 2), vr.repeat_interleave(G, 2), None, causal)
                dq_ref, dk_ref, dv_ref = torch.autograd.grad(o_ref, (qr, kr, vr), do.double())
                sh = lambda t: orc.shard(t, rank, world, layout).to(dev)  # noqa: E731
                ql, kl, vl = (sh(t).requires_grad_() for t in (q, k, v))
                o = func(ql, kl, vl, None, "cuda", causal, True, False, None, double_group)
                dq, dk, dv = torch.autograd.grad(o, (ql, kl, vl), sh(do))
                torch.cuda.synchronize()
                ok = dk.shape == kl.shape and dv.shape == vl.shape
                for nm, got, ref in (("o", o, o_ref), ("dq", dq, dq_ref), ("dk", dk, dk_ref), ("dv", dv, dv_ref)):
                    r = orc.shard(ref.detach(), rank, world, layout)
                    try:
                        torch.testing.assert_close(got.detach().double().cpu(), r, **tol)
                    except AssertionError as e:
                        ok = False
                        print(f"[rank {rank}] {name} Hkv={hkv} {dtype} {nm} MISMATCH: {str(e).splitlines()[-3:]}",
                              flush=True)
                flag = torch.tensor([0 if ok else 1], device=dev)
                dist.all_reduce(flag)
                if rank == 0:
                    print(f"ring_check_gqa W={world} {tag:10s} {os.environ.get('BA_RING_TRANSPORT', 'default'):7s} "
                          f"Hq={HQ} Hkv={hkv} {name:8s} {str(dtype):15s} {'PASS' if flag.item() == 0 else 'FAIL'}",
                          flush=True)
                fails += int(flag.item())
    return fails


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    fails = 0
    for transport in ("nccl", "ce"):
        os.environ["BA_RING_TRANSPORT"] = transport
        fails += _run_cases(rank, world, dev, [None, None], "flat")
    os.environ.pop("BA_RING_TRANSPORT")
    if world >= 4 and world % 2 == 0:
        os.environ["BA_DOUBLE_RING"] = "1"
        fails += _run_cases(rank, world, dev, _double_group(world, 2), "double L=2")
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
