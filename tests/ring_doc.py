"""Packed-document ring jobs for the multi-rank harness of ``tests/ring_harness.py``: W processes on one GPU under gloo
with the staged transport, running ``burst_attn_func`` / ``burst_attn_func_striped`` with ``cu_seqlens`` (and a
window), checked after reassembly against the fp64 document oracle of the whole sequence under the 16-bit error model
(``lowp_doc``: the whole sequence as one launch with the document mask)."""
from __future__ import annotations

import os

import torch
import torch.distributed as dist

import ring_harness as rh


def doc_job(world, mode, cu, window=(-1, -1), causal=None, B=2, H=4, Hkv=2, D=128, S_local=256, seq_dim=1, intra=0,
            det=False, dtype=torch.bfloat16, seed=0):
    causal = mode != "none" if causal is None else causal
    jid = f"docring_w{world}_{'flat' if not intra else f'{intra}x{world // intra}'}_{mode}{'_causal' if causal else ''}" \
          f"_win{window[0]}_{window[1]}_{'bhsd_' if seq_dim == 2 else ''}{'det_' if det else ''}n{len(cu) - 1}_s{seed}"
    return dict(id=jid, world=world, mode=mode, cu=list(cu), window=tuple(window), causal=causal, B=B, H=H, Hkv=Hkv,
                D=D, S=S_local * world, seq_dim=seq_dim, intra=intra, det=det, dtype=dtype, seed=seed)


def inputs(job):
    g = torch.Generator().manual_seed(job["seed"])
    B, S, H, Hkv, D = job["B"], job["S"], job["H"], job["Hkv"], job["D"]
    q, do = (torch.randn(B, S, H, D, generator=g).to(job["dtype"]) for _ in range(2))
    k, v = (torch.randn(B, S, Hkv, D, generator=g).to(job["dtype"]) for _ in range(2))
    return q, k, v, do


def _run_job(job, rank, world, device, groups):
    from burst_attn import burst_attn_func, burst_attn_func_striped
    from oracle import attention_oracle as orc
    layout, seq_dim = rh._LAYOUT[job["mode"]], job["seq_dim"]
    lay = (lambda t: t) if seq_dim == 1 else (lambda t: t.permute(0, 2, 1, 3).contiguous())
    unlay = (lambda t: t) if seq_dim == 1 else (lambda t: t.permute(0, 2, 1, 3))
    q, k, v, do = (lay(orc.shard(t, rank, world, layout)).to(device) for t in inputs(job))
    func = burst_attn_func_striped if job["mode"] == "striped" else burst_attn_func
    dg = groups[job["intra"]] if job["intra"] else [None, None]
    cu = torch.tensor(job["cu"], dtype=torch.int32, device=device)

    def call():
        qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
        o = func(qq, kk, vv, None, "cuda" if seq_dim == 1 else None, job["causal"], False, job["det"], None, list(dg),
                 job["window"], None, cu)
        lse = o.grad_fn.saved_tensors[3].detach().cpu().clone()  # (q, k, v, lse, out), before grad frees them
        dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
        out = {n: unlay(t.detach()).cpu().contiguous() for n, t in zip(("o", "dq", "dk", "dv"), (o, dq, dk, dv))}
        return dict(out, lse=lse)

    out, problems = call(), []
    if job["det"]:
        again = call()
        problems += [f"rank {rank}: deterministic mode: {n} differs bitwise" for n in out if not torch.equal(out[n],
                                                                                                        again[n])]
    return out, problems


def run_doc_cases(rank, world, port, jobs, outdir):
    from burst_attn import chunk_ops
    os.environ["BA_RING_TRANSPORT"] = "nccl"
    torch.cuda.set_device(0)
    device = torch.device("cuda", 0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rh.install_staged_transport()
    groups = {i: rh.double_group(rank, world, i, False) for i in sorted({j["intra"] for j in jobs if j["intra"]})}
    try:
        chunk_ops._set_ops_for_testing(chunk_ops.NativeOps())
        for job in jobs:
            out, problems = _run_job(job, rank, world, device, groups)
            torch.save(dict(out, problems=problems), os.path.join(outdir, f"{job['id']}.rank{rank}.pt"))
        torch.cuda.synchronize()
        dist.barrier()
    finally:
        chunk_ops._set_ops_for_testing(None)
        dist.destroy_process_group()


def whole_mask(cu, causal, window):
    """The document mask (``lowp_doc``) of the whole sequence as one launch, with the call's causal / window band."""
    left, right = window
    lo = -left if left >= 0 else None
    hi = 0 if causal else (right if right >= 0 else None)
    return ("doc", lo, hi, tuple(cu), 0, 0, 1)


def load_and_check(job, outdir):
    """Reassemble the ranks' outputs (after their own checks) and check them against the fp64 oracle under the
    16-bit model of the whole sequence."""
    import lowp_doc
    import lowp_model as lm
    from oracle import attention_oracle as orc
    lowp_doc.install()
    parts = [torch.load(os.path.join(outdir, f"{job['id']}.rank{r}.pt")) for r in range(job["world"])]
    problems = [p for part in parts for p in part["problems"]]
    assert not problems, f"{job['id']}: " + "; ".join(problems)
    layout = rh._LAYOUT[job["mode"]]
    got = {n: orc.unshard([p[n] for p in parts], layout, dim=2 if n == "lse" else 1)
           for n in ("o", "lse", "dq", "dk", "dv")}
    q, k, v, do = inputs(job)
    scale = job["D"] ** -0.5
    masks = [whole_mask(job["cu"], job["causal"], job["window"])]
    args = (q, [k], [v], do, scale, masks)
    model, ref = lm.lowp_chain(*args), lm.oracle_chain(*args)
    lm.assert_api_within_model(job["id"], got, ref, model, job["dtype"], lm.scores_absmax(q, [k], scale, masks))
