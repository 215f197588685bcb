"""Windowed ring jobs for the multi-rank harness of ``tests/ring_harness.py``: the same W processes on one GPU under
gloo with the staged transport, running ``burst_attn_func`` / ``burst_attn_func_striped`` with a ``window_size``, and
the same check of the reassembled full sequence against the fp64 oracle and the 16-bit model, with the window as
one band over the whole sequence (``lowp_band``)."""
from __future__ import annotations

import os
import time

import torch
import torch.distributed as dist

import ring_harness as rh


def window_job(world, mode, dtype, D, Hkv, S_local, window, B=2, scale="d", seq_dim=1, intra=0, dq_groups=False,
               l2=None, det=False, causal=None):
    """One job as ``ring_harness.ring_job`` (``mode``: the shard layout "none" (contiguous) | "zigzag" | "striped")
    with ``window_size=window``.  ``causal`` defaults to the layout's (zigzag and striped causal); striped shards may
    also run without it."""
    import lowp_model as lm
    causal = mode != "none" if causal is None else causal
    topo = "flat" if not intra else f"{intra}x{world // intra}" + ("dq" if dq_groups else "")
    tag = f"winring_w{world}_{topo}_{mode}{'_causal' if causal else ''}_win{window[0]}_{window[1]}_" + \
        ("bhsd_" if seq_dim == 2 else "") + (f"l2-{l2}_" if l2 else "") + ("det_" if det else "")
    case = lm._case(S_local * world, [(S_local * world, None)], D, dtype, scale=scale, B=B, H=4, Hkv=Hkv, tag=tag)
    left, right = window
    right = 0 if causal else right
    mask = None  # the window over the full sequence (off = 0) as one band
    if left >= 0 or right >= 0:
        mask = ("band", -left if left >= 0 else None, right if right >= 0 else None)
    elif causal:
        mask = ("causal_offset", 0)
    return dict(id=case["id"], case=case, world=world, mode=mode, causal=causal, window=tuple(window), mask=mask,
                seq_dim=seq_dim, intra=intra, dq_groups=dq_groups, l2=l2, det=det, fault=None)


def _run_job(job, rank, world, device, groups):
    """This rank's part of one job (``ring_harness._run_job`` with the window passed)."""
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
    if job["l2"]:
        os.environ["BA_L2_BLOCK"] = str(job["l2"])
    else:
        os.environ.pop("BA_L2_BLOCK", None)
    problems = []

    def call():
        qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
        kept = [t.detach().clone() for t in (qq, kk, vv)]
        o = func(qq, kk, vv, x["scale"], "cuda" if seq_dim == 1 else None, job["causal"], False, job["det"], None,
                 list(dg), job["window"])
        lse = o.grad_fn.saved_tensors[3].detach().clone()  # (q, k, v, lse, out), before grad frees them
        dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
        for name, t, t0 in zip("qkv", (qq, kk, vv), kept):
            if not torch.equal(t.detach(), t0):
                problems.append(f"rank {rank}: the user's {name} was modified")
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


def run_window_cases(rank, world, port, jobs, outdir):
    """Worker: every job on this rank with the native kernels (every rank on cuda:0), outputs to
    ``outdir/<job id>.rank<r>.pt`` as ``ring_harness.run_ring_cases`` writes them."""
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
            assert job["world"] == world, (job["id"], world)
            out, problems = _run_job(job, rank, world, device, groups)
            torch.save(dict(out, problems=problems), os.path.join(outdir, f"{job['id']}.rank{rank}.pt"))
        torch.cuda.synchronize()
        dist.barrier()
    finally:
        chunk_ops._set_ops_for_testing(None)
        dist.destroy_process_group()


class WindowRuns(rh.WorldRuns):
    """``ring_harness.WorldRuns`` for windowed jobs (native kernels)."""

    def __init__(self, jobs, tmp_path_factory, timeout):
        super().__init__(jobs, "native", tmp_path_factory, timeout)

    def outdir(self, world):
        if world not in self.done:
            out = str(self.tmp.mktemp(f"winring_w{world}"))
            t0 = time.monotonic()
            try:
                rh.spawn(run_window_cases, world, (self.jobs[world], out), timeout=self.timeout)
                self.done[world] = (out, None)
            except BaseException as e:  # noqa: BLE001
                self.done[world] = (None, e)
            print(f"\nW={world}: {len(self.jobs[world])} windowed jobs on {world} ranks in {time.monotonic() - t0:.1f} s")
        out, err = self.done[world]
        if err is not None:
            raise RuntimeError(f"the W={world} ranks failed: {err}")
        return out


def check_window_case(job, got):
    """``ring_harness.check_ring_case`` with the job's window as the mask of the whole sequence."""
    import lowp_band
    import lowp_model as lm
    lowp_band.install()
    x = lm.make_inputs(job["case"])
    masks = [job["mask"]]
    args = (x["q"], x["ks"], x["vs"], x["do"], x["scale"], masks)
    model, ref = lm.lowp_chain(*args), lm.oracle_chain(*args)
    absmax = lm.scores_absmax(x["q"], x["ks"], x["scale"], masks)
    lm.assert_api_within_model(job["id"], got, ref, model, job["case"]["dtype"], absmax)
