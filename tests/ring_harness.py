"""Shared harness of the multi-rank tests: W ranks as W processes under one gloo process group.

* ``spawn`` runs a target on every rank and never leaves a process behind: a rank still alive at the timeout (or
  shortly after another rank failed) is terminated, then killed, and the call fails with every rank's traceback.
* ``install_staged_transport`` replaces the hop of ``comm.Ring`` (for CPU and CUDA tensors alike) by one staged
  through the CPU and sent over gloo at ``wait``.  Between ``post`` and ``wait`` the destinations hold NaN and the
  sources must not change, as with the asynchronous GPU transports: a kernel that reads a receive buffer too early
  sees NaN, one that writes a source while its hop is in flight fails the snapshot check.  Several ranks can then
  share one GPU: no NCCL communicator is ever created.
* ``run_ring_cases`` is the worker: it runs ``burst_attn_func`` / ``burst_attn_func_striped`` through autograd on
  this rank's shard of each job (``ring_job``: optionally with a window, ALiBi slopes or packed documents), with the
  native kernels (or the CPU oracle, or a fault injected into either), and saves O, lse, dQ, dK and dV.
  ``check_ring_case`` compares the full sequence, reassembled in the parent, with the fp64 oracle under the 16-bit
  error model of ``lowp_model``.
"""
from __future__ import annotations

import os
import socket
import sys
import time
import traceback

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _entry(target, rank, world, port, errq, args):
    try:
        for p in (ROOT, os.path.join(ROOT, "burst-attention_b200"), os.path.join(ROOT, "tests")):
            if p not in sys.path:
                sys.path.insert(0, p)
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        target(rank, world, port, *args)
    except BaseException as e:  # noqa: BLE001
        errq.put(f"rank {rank}: {type(e).__name__}: {e}\n{traceback.format_exc()}")
        raise


def spawn(target, world, args=(), timeout=240.0, grace=20.0):
    """Run ``target(rank, world, port, *args)`` on ``world`` processes and fail with every rank's traceback.

    Ranks still alive ``timeout`` seconds after the start, or ``grace`` seconds after another rank exited with an
    error (its peers are then usually blocked in a collective), are terminated and, if that does not end them,
    killed: no process outlives the call."""
    ctx = mp.get_context("spawn")
    errq = ctx.SimpleQueue()
    port = free_port()
    procs = [ctx.Process(target=_entry, args=(target, r, world, port, errq, tuple(args))) for r in range(world)]
    for p in procs:
        p.start()
    deadline = time.monotonic() + timeout
    from multiprocessing.connection import wait as wait_any
    while any(p.is_alive() for p in procs):
        now = time.monotonic()
        if now >= deadline:
            break
        wait_any([p.sentinel for p in procs if p.is_alive()], timeout=min(1.0, deadline - now))
        if any(p.exitcode not in (None, 0) for p in procs):
            deadline = min(deadline, time.monotonic() + grace)
    stuck = [r for r, p in enumerate(procs) if p.is_alive()]
    for p in procs:
        if p.is_alive():
            p.terminate()
    for p in procs:
        p.join(5)
        if p.is_alive():
            p.kill()
            p.join()
    errs = []
    while not errq.empty():
        errs.append(errq.get())
    msg = "\n".join(errs)
    assert not stuck, f"ranks {stuck} still running after {timeout:.0f} s (or after a peer failed); terminated\n{msg}"
    assert not errs, msg
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]


# --------------------------------------------------------------------------- #
# staged transport
# --------------------------------------------------------------------------- #
def install_staged_transport():
    """Patch ``comm.Ring.commit`` / ``wait`` (and ``empty``, to know which buffers it handed out) in this process.

    commit: at most one hop in flight per ring; on the copy-engine transport every destination must come from
    ``Ring.empty``; the sources are snapshotted to the CPU and the destinations filled with NaN on their device.
    wait: every source must still equal its snapshot; the snapshots then travel over gloo as bytes, with the
    send/recv order of ``Ring._commit_torch``, and are copied into the destinations."""
    from burst_attn import comm

    plain_empty = comm.Ring.empty
    exchange = comm.Ring._commit_torch

    def empty(self, shape, dtype, device):
        t = plain_empty(self, shape, dtype, device)
        self.__dict__.setdefault("_owned", set()).add(t.data_ptr())
        return t

    def commit(self):
        if not self._pending:
            return
        srcs = [s for s, _ in self._pending]
        dsts = [d for _, d in self._pending]
        self._pending = []
        assert not getattr(self, "_staged", None), "two hops in flight on one ring"
        if self.transport == "ce":  # copy-engine rings can only receive into buffers carved from their arena
            assert all(d.data_ptr() in getattr(self, "_owned", ()) for d in dsts), \
                "a hop destination was not allocated through Ring.empty / empty_like"
        snap = [s.detach().cpu().clone() for s in srcs]  # clone: .cpu() of a CPU tensor is the tensor itself
        for d in dsts:
            d.fill_(float("nan"))
        self._staged = (srcs, dsts, snap)
        self._reqs = ["staged"]

    def wait(self, force_wait_inter=False):
        for r in self._reqs:
            assert r == "staged"
            srcs, dsts, snap = self._staged
            self._staged = None
            for s, c in zip(srcs, snap):
                assert torch.equal(s.detach().cpu(), c), "a hop's source was modified between post and wait"
            send = [c.contiguous().view(-1).view(torch.uint8) for c in snap]
            recv = [torch.empty(d.numel() * d.element_size(), dtype=torch.uint8) for d in dsts]
            for q in exchange(self, send, recv):
                q.wait()
            for d, b in zip(dsts, recv):
                d.copy_(b.view(d.dtype).view(d.shape))
        self._reqs = []

    comm.Ring.empty = empty
    comm.Ring.commit = commit
    comm.Ring.wait = wait


def double_group(rank, world, intra, dq_groups):
    """Hierarchical ring: nodes of `intra` consecutive ranks (reference test/test_burst.py:120-156)."""
    from burst_attn.burst_attn_interface import _Topology, get_partition_id
    from oracle import attention_oracle as orc
    os.environ["BA_DOUBLE_RING"] = "1"
    rows = [list(range(n * intra, (n + 1) * intra)) for n in range(world // intra)]
    cols = [list(c) for c in zip(*rows)]
    mk = lambda ranks: dist.new_subgroups_by_enumeration(ranks, backend="gloo")[0]  # noqa: E731
    groups = [mk(rows), mk(cols)]
    if dq_groups:
        groups = [(groups[0], mk(rows)), (groups[1], mk(cols))]
    topo = _Topology(None, groups)
    assert topo.hier and (topo.L, topo.M) == (intra, world // intra)
    plain = [g[0] if isinstance(g, tuple) else g for g in groups]
    seen = sorted(get_partition_id(plain, r) for r in range(1, world + 1))
    assert seen == list(range(world)), seen  # every shard is visited exactly once
    assert get_partition_id(plain, 1) == rank
    for r in range(1, world + 1):  # the oracle's restatement is pinned to the reference (tests/golden)
        assert get_partition_id(plain, r) == orc.get_partition_id_double(r, rank % intra, rank // intra, intra,
                                                                        world // intra)
    return groups


# --------------------------------------------------------------------------- #
# ring-level faults, for the comparator's negative controls
# --------------------------------------------------------------------------- #
FAULTS = (
    "striped_not_strict",  # a causal_offset of -1 is passed as 0: the diagonal key of a later rank leaks in
    "lost_dq_hop",         # the first accumulate of a backward is skipped: one arriving dQ partial is lost
    "fwd_state_dropped",   # the second fwd_chunk of a forward gets first=True: the carried state is lost
)


class FaultOps:
    """Chunk operators that delegate to ``ops`` and inject one fault of ``FAULTS``."""

    def __init__(self, ops, fault):
        assert fault in FAULTS, fault
        self._ops, self.fault = ops, fault
        self._fwd_calls = 0
        self._skipped = False

    def __getattr__(self, name):  # name, tile_head_dims, launches, ...
        return getattr(self._ops, name)

    def _offset(self, causal, off):
        return 0 if self.fault == "striped_not_strict" and causal and off == -1 else off

    def fwd_chunk(self, q, k, v, o_acc, lse, o_out, scale, causal, causal_offset, first, last, seq_dim, **kw):
        self._fwd_calls = 1 if first else self._fwd_calls + 1
        if self.fault == "fwd_state_dropped" and self._fwd_calls == 2:
            first = True
        self._ops.fwd_chunk(q, k, v, o_acc, lse, o_out, scale, causal, self._offset(causal, causal_offset), first,
                            last, seq_dim, **kw)

    def bwd_chunk(self, d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, scale, causal, causal_offset, seq_dim,
                  deterministic=False, **kw):
        self._ops.bwd_chunk(d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, scale, causal,
                            self._offset(causal, causal_offset), seq_dim, deterministic, **kw)

    def delta(self, o, d_o, out, seq_dim):  # the first operation of every backward
        self._skipped = False
        self._ops.delta(o, d_o, out, seq_dim)

    def cast(self, src, dst, seq_dim):
        self._ops.cast(src, dst, seq_dim)

    def accumulate(self, src, dst, seq_dim):
        if self.fault == "lost_dq_hop" and not self._skipped:
            self._skipped = True
            return
        self._ops.accumulate(src, dst, seq_dim)


# --------------------------------------------------------------------------- #
# jobs: one call of the public API on a ring, forward and backward
# --------------------------------------------------------------------------- #
_LAYOUT = {"none": "contiguous", "zigzag": "zigzag", "striped": "striped"}


def ring_job(world, mode, dtype, D, Hkv, S_local, B=2, scale="d", seq_dim=1, intra=0, dq_groups=False, l2=None,
             det=False, fault=None, window=None, causal=None, slopes=None, cu=None, seed=0):
    """One job: ``mode`` "none" | "zigzag" | "striped" (the shard layout: contiguous, zigzag, striped) on a flat ring
    (``intra=0``) or a hierarchical one of nodes of ``intra`` ranks, ``S_local`` rows per rank, Hq = 4 query heads,
    ``seq_dim`` 2 for the [B,H,S,D] layout, ``l2``: BA_L2_BLOCK, ``det``: deterministic (run twice, must be bitwise
    equal), ``fault``: one of FAULTS.  ``causal`` defaults to the layout's (zigzag and striped causal); striped shards
    may also run without it.  Optional fields of the call:

    * ``window``: ``window_size`` (a windowed job);
    * ``slopes``: ALiBi slopes of shape (H,) ("h") or (B, H) ("bh"), with ``window`` (default (-1, -1));
    * ``cu``: ``cu_seqlens`` (a document job), with ``window`` (default (-1, -1)).  Its inputs come from a generator of
      their own seeded by ``seed``, and the library's default softmax scale, instead of ``lowp_model.make_inputs``."""
    import lowp_model as lm
    causal = mode != "none" if causal is None else causal
    S = S_local * world
    topo = "flat" if not intra else f"{intra}x{world // intra}" + ("dq" if dq_groups else "")
    opts = ("bhsd_" if seq_dim == 2 else "") + (f"l2-{l2}_" if l2 else "") + ("det_" if det else "")
    if (slopes is not None or cu is not None) and window is None:
        window = (-1, -1)
    job = dict(world=world, mode=mode, dtype=dtype, causal=causal, window=None if window is None else tuple(window),
               slopes=slopes, cu=None if cu is None else list(cu), seed=seed, seq_dim=seq_dim, intra=intra,
               dq_groups=dq_groups, l2=l2, det=det, fault=fault, case=None)
    if cu is not None:
        win = f"_win{window[0]}_{window[1]}_"
        job["id"] = f"docring_w{world}_{topo}_{mode}{'_causal' if causal else ''}{win}{opts}n{len(cu) - 1}_s{seed}"
        job["shape"] = (B, S, Hkv, D)
    elif window is not None:
        tag = f"winring_w{world}_{topo}_{mode}{'_causal' if causal else ''}_win{window[0]}_{window[1]}_{opts}"
        job["case"] = lm._case(S, [(S, None)], D, dtype, scale=scale, B=B, H=4, Hkv=Hkv, tag=tag)
        job["id"] = job["case"]["id"]
        if slopes is not None:
            job["id"] = f"alibi_{job['id']}{'bh_' if slopes == 'bh' else ''}"
    else:
        tag = f"ring_w{world}_{topo}_{mode}_{opts}" + (f"{fault}_" if fault else "")
        job["case"] = lm._case(S, [(S, None if mode == "none" else 0)], D, dtype, scale=scale, B=B, H=4, Hkv=Hkv,
                               tag=tag)
        job["id"] = job["case"]["id"]
    return job


def job_inputs(job):
    """The job's full-sequence 16-bit inputs, dict(q, ks, vs, do, scale), the same on every rank: the case's
    (``lowp_model.make_inputs``, seeded by the case id) or a document job's own."""
    import lowp_model as lm
    if job["case"] is not None:
        return lm.make_inputs(job["case"])
    B, S, Hkv, D = job["shape"]
    g = torch.Generator().manual_seed(job["seed"])
    q, do = (torch.randn(B, S, 4, D, generator=g).to(job["dtype"]) for _ in range(2))
    k, v = (torch.randn(B, S, Hkv, D, generator=g).to(job["dtype"]) for _ in range(2))
    return dict(q=q, ks=[k], vs=[v], do=do, scale=D ** -0.5)


def job_slopes(job):
    """The ALiBi slopes of the call, fp32 (H,) or (B, H), or None."""
    import mask_oracle as mo
    if job["slopes"] is None:
        return None
    c = job["case"]
    return mo.slopes_for(c["B"], c["H"], job["slopes"] == "bh", seed=1)


def whole_mask(job):
    """The kernels' mask of the whole sequence as one chunk (``mask_oracle.mask_of``), from the job's causal flag,
    window and documents."""
    if job["window"] is None:
        return ("causal_offset", 0) if job["causal"] else None
    left, right = job["window"]
    lo = -left if left >= 0 else None
    hi = 0 if job["causal"] else (right if right >= 0 else None)
    if job["cu"] is not None:
        return ("doc", lo, hi, tuple(job["cu"]), 0, 0, 1)
    return None if lo is None and hi is None else ("band", lo, hi)


def _run_job(job, rank, world, device, groups):
    """This rank's part of one job; returns (outputs in the logical [B,S,H,D] / [B,H,S] layouts, local problems)."""
    from burst_attn import burst_attn_func, burst_attn_func_striped
    from oracle import attention_oracle as orc
    mode, seq_dim, layout = job["mode"], job["seq_dim"], _LAYOUT[job["mode"]]
    x = job_inputs(job)
    lay = (lambda t: t) if seq_dim == 1 else (lambda t: t.permute(0, 2, 1, 3).contiguous())
    unlay = (lambda t: t) if seq_dim == 1 else (lambda t: t.permute(0, 2, 1, 3))
    sh = lambda t: lay(orc.shard(t, rank, world, layout)).to(device)  # noqa: E731
    q, k, v, do = sh(x["q"]), sh(x["ks"][0]), sh(x["vs"][0]), sh(x["do"])
    func = burst_attn_func_striped if mode == "striped" else burst_attn_func
    dg = groups[(job["intra"], job["dq_groups"])] if job["intra"] else [None, None]
    scale = None if job["case"] is None else x["scale"]  # document jobs: the library's default scale
    slopes = job_slopes(job)
    extra = dict(window_size=job["window"] or (-1, -1), alibi_slopes=None if slopes is None else slopes.to(device),
                 cu_seqlens=None if job["cu"] is None else torch.tensor(job["cu"], dtype=torch.int32, device=device))
    if job["l2"]:
        os.environ["BA_L2_BLOCK"] = str(job["l2"])
    else:
        os.environ.pop("BA_L2_BLOCK", None)
    problems = []

    def call():
        qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
        kept = [t.detach().clone() for t in (qq, kk, vv)]
        o = func(qq, kk, vv, scale, "cuda" if seq_dim == 1 else None, job["causal"], False, job["det"], None,
                 list(dg), **extra)
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


def run_ring_cases(rank, world, port, jobs, ops_kind, outdir):
    """Worker: every job on this rank, outputs to ``outdir/<job id>.rank<r>.pt``.  ``ops_kind``: "native" (the
    kernels, every rank on cuda:0) or "oracle" (the fp64 CPU oracle on CPU tensors)."""
    from burst_attn import chunk_ops
    os.environ["BA_RING_TRANSPORT"] = "nccl"  # never ce / local; the hop is staged through the CPU anyway
    if ops_kind == "native":
        torch.cuda.set_device(0)
        device = torch.device("cuda", 0)
        base = chunk_ops.NativeOps()
    else:
        from oracle_ops import OracleOps
        device = torch.device("cpu")
        base = OracleOps()
    dist.init_process_group("gloo", rank=rank, world_size=world)
    install_staged_transport()
    groups = {key: double_group(rank, world, *key)
              for key in sorted({(j["intra"], j["dq_groups"]) for j in jobs if j["intra"]})}
    try:
        for job in jobs:
            assert job["world"] == world, (job["id"], world)
            chunk_ops._set_ops_for_testing(base if job["fault"] is None else FaultOps(base, job["fault"]))
            out, problems = _run_job(job, rank, world, device, groups)
            torch.save(dict(out, problems=problems), os.path.join(outdir, f"{job['id']}.rank{rank}.pt"))
        if device.type == "cuda":
            torch.cuda.synchronize()
        dist.barrier()
    finally:
        chunk_ops._set_ops_for_testing(None)
        dist.destroy_process_group()


class WorldRuns:
    """Runs the jobs of each world size in one ``spawn`` on first use, and remembers the output directory (or the
    failure, which every later use raises again)."""

    def __init__(self, jobs, ops_kind, tmp_path_factory, timeout):
        self.jobs, self.ops_kind, self.tmp, self.timeout = jobs, ops_kind, tmp_path_factory, timeout
        self.done = {}

    def outdir(self, world):
        if world not in self.done:
            out = str(self.tmp.mktemp(f"ring_w{world}"))
            t0 = time.monotonic()
            try:
                spawn(run_ring_cases, world, (self.jobs[world], self.ops_kind, out), timeout=self.timeout)
                self.done[world] = (out, None)
            except BaseException as e:  # noqa: BLE001
                self.done[world] = (None, e)
            print(f"\nW={world}: {len(self.jobs[world])} jobs on {world} ranks in {time.monotonic() - t0:.1f} s")
        out, err = self.done[world]
        if err is not None:
            raise RuntimeError(f"the W={world} ranks failed: {err}")
        return out


def load_ring_case(job, outdir):
    """In the parent: the full-sequence outputs of ``job`` reassembled from every rank (dict o, lse, dq, dk, dv),
    after the ranks' own checks (user inputs unmodified, deterministic runs bitwise equal)."""
    from oracle import attention_oracle as orc
    world, layout = job["world"], _LAYOUT[job["mode"]]
    parts = [torch.load(os.path.join(outdir, f"{job['id']}.rank{r}.pt")) for r in range(world)]
    problems = [p for part in parts for p in part["problems"]]
    assert not problems, f"{job['id']}: " + "; ".join(problems)
    return {n: orc.unshard([p[n] for p in parts], layout, dim=2 if n == "lse" else 1)
            for n in ("o", "lse", "dq", "dk", "dv")}


def check_ring_case(job, got):
    """``got`` (``load_ring_case``) against the fp64 oracle and the 16-bit model of the whole sequence as one chunk:
    the model's error terms are sums over keys, independent of how the ring splits them, and the ring's extra
    rounding is fp32.  ALiBi jobs are first held to the fp64 oracle within 2 u (O) and 4 u (the gradients), relative
    in the Frobenius norm.  Raises AssertionError."""
    import lowp_alibi as la
    import lowp_model as lm
    import mask_oracle as mo
    x = job_inputs(job)
    masks = [whole_mask(job)]
    args = (x["q"], x["ks"], x["vs"], x["do"], x["scale"], masks)
    dtype = job["dtype"]
    if job["slopes"] is None:
        model, ref = lm.lowp_chain(*args), lm.oracle_chain(*args)
        lm.assert_api_within_model(job["id"], got, ref, model, dtype, lm.scores_absmax(x["q"], x["ks"], x["scale"],
                                                                                      masks))
        return
    q, k, v, do = (t.double() for t in (x["q"], x["ks"][0], x["vs"][0], x["do"]))
    H, Hkv = q.shape[2], k.shape[2]
    G = H // Hkv
    slopes = mo.as_bh(job_slopes(job), q.shape[0])
    kx = k.repeat_interleave(G, 2)
    o, lse, dq, dk, dv = mo.dense_attention_bwd(q, kx, v.repeat_interleave(G, 2), do, x["scale"], job["causal"],
                                                job["window"], slopes)
    dk, dv = (t.unflatten(2, (Hkv, G)).sum(3) for t in (dk, dv))
    u = lm.unit_roundoff(dtype)
    for name, ref, ku in (("o", o, 2), ("dq", dq, 4), ("dk", dk, 4), ("dv", dv, 4)):
        e = float((got[name].double() - ref).norm() / ref.norm())
        assert e <= ku * u, f"{job['id']} {name}: relative error {e:.3e} > {ku} u"
    # lse: lowp_model's check, with the magnitude the fp32 score arithmetic works at (|q| |k| scale + |bias| over
    # the keys each row sees); -inf exactly where the oracle's is
    S = q.shape[1]
    a = torch.einsum("bqhd,bkhd->bhqk", q.abs(), kx.abs()) * abs(x["scale"])
    a = a - mo.bias(slopes, torch.arange(S), torch.arange(S))
    m = mo.window_mask(S, S, job["window"], job["causal"])
    if m is not None:
        a = a.masked_fill(~m, 0.0)
    lm.assert_lse(f"lse[{job['id']}]", got["lse"], lse, a.amax(-1))
    # per (b, s, h) row against the 16-bit model of the whole sequence as one chunk: d = a - c
    al = [(slopes.contiguous(), 0, 1)]
    absmax = la.absmax_prefix(x["q"], x["ks"], x["scale"], masks, al)[-1]
    lm.assert_api_within_model(job["id"], got, lm.oracle_chain(*args, alibis=al), lm.lowp_chain(*args, alibis=al),
                               dtype, absmax)
