"""ALiBi ring jobs for the multi-rank harness of ``tests/ring_harness.py``: W processes on one GPU under gloo with the
staged transport, running ``burst_attn_func`` / ``burst_attn_func_striped`` with ``alibi_slopes`` (and optionally a
``window_size``), the reassembled full sequence checked against the fp64 ALiBi oracle (``alibi_oracle``)."""
from __future__ import annotations

import os
import time

import torch
import torch.distributed as dist

import alibi_oracle as ao
import ring_band as rb
import ring_harness as rh

U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}


def alibi_job(world, mode, dtype, D, Hkv, S_local, window=(-1, -1), per_batch=False, **kw):
    """``ring_band.window_job`` with ALiBi; ``per_batch``: (B, H) slopes instead of (H,)."""
    job = rb.window_job(world, mode, dtype, D, Hkv, S_local, window, **kw)
    job["id"] = "alibi_" + job["id"] + ("bh_" if per_batch else "")
    job["per_batch"] = per_batch
    return job


def _slopes(job):
    c = job["case"]
    return ao.slopes_for(c["B"], c["H"], job["per_batch"], seed=1)


def _run_job(job, rank, world, device, groups):
    import lowp_model as lm
    from burst_attn import burst_attn_func, burst_attn_func_striped
    from oracle import attention_oracle as orc
    mode, seq_dim, layout = job["mode"], job["seq_dim"], rh._LAYOUT[job["mode"]]
    x = lm.make_inputs(job["case"])
    lay = (lambda t: t) if seq_dim == 1 else (lambda t: t.permute(0, 2, 1, 3).contiguous())
    unlay = (lambda t: t) if seq_dim == 1 else (lambda t: t.permute(0, 2, 1, 3))
    sh = lambda t: lay(orc.shard(t, rank, world, layout)).to(device)  # noqa: E731
    q, k, v, do = sh(x["q"]), sh(x["ks"][0]), sh(x["vs"][0]), sh(x["do"])
    func = burst_attn_func_striped if mode == "striped" else burst_attn_func
    dg = groups[(job["intra"], job["dq_groups"])] if job["intra"] else [None, None]
    slopes = _slopes(job).to(device)
    if job["l2"]:
        os.environ["BA_L2_BLOCK"] = str(job["l2"])
    else:
        os.environ.pop("BA_L2_BLOCK", None)
    problems = []

    def call():
        qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
        o = func(qq, kk, vv, x["scale"], "cuda" if seq_dim == 1 else None, job["causal"], False, job["det"], None,
                 list(dg), job["window"], slopes)
        lse = o.grad_fn.saved_tensors[3].detach().clone()  # (q, k, v, lse, out), before grad frees them
        dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
        out = dict(o=unlay(o.detach()), lse=lse, dq=unlay(dq), dk=unlay(dk), dv=unlay(dv))
        return {n: t.cpu().contiguous() for n, t in out.items()}

    out = call()
    if job["det"]:
        again = call()
        for n in out:
            if not torch.equal(out[n], again[n]):
                problems.append(f"rank {rank}: deterministic mode: {n} differs bitwise between two runs")
    os.environ.pop("BA_L2_BLOCK", None)
    return out, problems


def run_alibi_cases(rank, world, port, jobs, outdir):
    """Worker: ``ring_band.run_window_cases`` for ALiBi jobs."""
    from burst_attn import chunk_ops
    os.environ["BA_RING_TRANSPORT"] = "nccl"
    torch.cuda.set_device(0)
    device = torch.device("cuda", 0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rh.install_staged_transport()
    groups = {key: rh.double_group(rank, world, *key)
              for key in sorted({(j["intra"], j["dq_groups"]) for j in jobs if j["intra"]})}
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


class AlibiRuns(rh.WorldRuns):
    def __init__(self, jobs, tmp_path_factory, timeout):
        super().__init__(jobs, "native", tmp_path_factory, timeout)

    def outdir(self, world):
        if world not in self.done:
            out = str(self.tmp.mktemp(f"alibiring_w{world}"))
            t0 = time.monotonic()
            try:
                rh.spawn(run_alibi_cases, world, (self.jobs[world], out), timeout=self.timeout)
                self.done[world] = (out, None)
            except BaseException as e:  # noqa: BLE001
                self.done[world] = (None, e)
            print(f"\nW={world}: {len(self.jobs[world])} ALiBi jobs on {world} ranks in {time.monotonic() - t0:.1f} s")
        out, err = self.done[world]
        if err is not None:
            raise RuntimeError(f"the W={world} ranks failed: {err}")
        return out


def check_alibi_case(job, got):
    """The reassembled outputs against the fp64 ALiBi oracle of the whole sequence: O within 2 u, the gradients
    within 4 u (relative, Frobenius), lse as ``lowp_model.assert_lse`` checks it."""
    import lowp_model as lm
    x = lm.make_inputs(job["case"])
    q, k, v, do = (t.double() for t in (x["q"], x["ks"][0], x["vs"][0], x["do"]))
    H, Hkv = q.shape[2], k.shape[2]
    G = H // Hkv
    o, lse, dq, dk, dv = ao.dense_attention_bwd(q, k.repeat_interleave(G, 2), v.repeat_interleave(G, 2), do,
                                                x["scale"], job["causal"], job["window"],
                                                ao.as_bh(_slopes(job), q.shape[0]))
    dk, dv = (t.unflatten(2, (Hkv, G)).sum(3) for t in (dk, dv))
    u = U[job["case"]["dtype"]]
    for name, ref, ku in (("o", o, 2), ("dq", dq, 4), ("dk", dk, 4), ("dv", dv, 4)):
        e = float((got[name].double() - ref).norm() / ref.norm())
        assert e <= ku * u, f"{job['id']} {name}: relative error {e:.3e} > {ku} u"
    # lse: lowp_model's check, with the magnitude the fp32 score arithmetic works at (|q| |k| scale + |bias| over
    # the keys each row sees); -inf exactly where the oracle's is
    import band_oracle as bo
    kx = k.repeat_interleave(G, 2)
    S = q.shape[1]
    a = torch.einsum("bqhd,bkhd->bhqk", q.abs(), kx.abs()) * abs(x["scale"])
    a = a - ao.bias(ao.as_bh(_slopes(job), q.shape[0]), torch.arange(S), torch.arange(S))
    m = bo.window_mask(S, S, job["window"], job["causal"])
    if m is not None:
        a = a.masked_fill(~m, 0.0)
    lm.assert_lse(f"lse[{job['id']}]", got["lse"], lse, a.amax(-1))
    # per (b, s, h) row against the 16-bit model (lowp_alibi) of the whole sequence as one chunk: d = a - c
    import lowp_alibi as la
    al = [(ao.as_bh(_slopes(job), q.shape[0]).contiguous(), 0, 1)]
    args = (x["q"], x["ks"], x["vs"], x["do"], x["scale"], [job["mask"]], al)
    absmax = la.absmax_prefix(x["q"], x["ks"], x["scale"], [job["mask"]], al)[-1]
    lm.assert_api_within_model(job["id"], got, la.oracle_alibi_chain(*args), la.lowp_alibi_chain(*args),
                               job["case"]["dtype"], absmax)
