"""Grouped-query attention (K/V with fewer heads than Q) through the ring drivers on CPU: world 1 in-process, worlds
2 and 4 and the hierarchical ring (intra rings of 2) under gloo.  The chunk operators are the oracle's, wrapped so
that they see GQA operands (K/V expanded per group before the oracle call, dK/dV summed back over each group); the
results are compared, through autograd, with dense attention on expanded K/V.  Each forward hop must carry 1/G of
the bytes the same call with MHA K/V (Hq heads) would post."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "burst-attention_b200"), os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

HQ = 4
HKV_CASES = (2, 1)  # G = 2 (GQA) and G = Hq (MQA)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gqa_ops():
    from oracle_ops import OracleOps

    def expand(t, G, seq_dim):
        return t if G == 1 else t.repeat_interleave(G, dim=3 - seq_dim)

    def group_sum(t, G, seq_dim):
        hd = 3 - seq_dim
        return t if G == 1 else t.unflatten(hd, (t.shape[hd] // G, G)).sum(hd + 1)

    class GqaOracleOps(OracleOps):
        """OracleOps for K/V with Hq / G heads: expand K/V per group, sum dK/dV back over each group."""

        def fwd_chunk(self, q, k, v, o_acc, lse, o_out, scale, causal, causal_offset, first, last, seq_dim, bias=None):
            G = q.shape[3 - seq_dim] // k.shape[3 - seq_dim]
            super().fwd_chunk(q, expand(k, G, seq_dim), expand(v, G, seq_dim), o_acc, lse, o_out, scale, causal,
                              causal_offset, first, last, seq_dim, bias=bias)

        def bwd_chunk(self, d_o, q, k, v, delta, lse, dq_acc, dk_acc, dv_acc, scale, causal, causal_offset, seq_dim,
                      deterministic=False, bias=None):
            G = q.shape[3 - seq_dim] // k.shape[3 - seq_dim]
            ke, ve = expand(k, G, seq_dim), expand(v, G, seq_dim)
            dk_e, dv_e = torch.zeros(ke.shape, dtype=dk_acc.dtype), torch.zeros(ve.shape, dtype=dv_acc.dtype)
            super().bwd_chunk(d_o, q, ke, ve, delta, lse, dq_acc, dk_e, dv_e, scale, causal, causal_offset, seq_dim,
                              deterministic, bias=bias)
            dk_acc.add_(group_sum(dk_e, G, seq_dim))
            dv_acc.add_(group_sum(dv_e, G, seq_dim))

    return GqaOracleOps()


def _check_case(rank, world, case, seq_dim, hkv, double_group=(None, None)):
    """One GQA call of the ring driver on this rank against dense attention on expanded K/V."""
    from burst_attn import burst_attn_func, burst_attn_func_striped, comm
    from oracle import attention_oracle as orc

    func, causal, layout = {
        "none": (burst_attn_func, False, "contiguous"),
        "zigzag": (burst_attn_func, True, "zigzag"),
        "striped": (burst_attn_func_striped, True, "striped"),
    }[case]
    G = HQ // hkv
    torch.manual_seed(4321 + hkv)  # same full tensors on every rank
    B, S, D = 2, 8 * 2 * world, 16
    q, do = (torch.randn(B, S, HQ, D, dtype=torch.float64) for _ in range(2))
    k, v = (torch.randn(B, S, hkv, D, dtype=torch.float64) for _ in range(2))
    scale = D ** -0.5
    qr, kr, vr = (t.clone().requires_grad_() for t in (q, k, v))
    o_ref, _ = orc.dense_attention(qr, kr.repeat_interleave(G, dim=2), vr.repeat_interleave(G, dim=2), scale, causal)
    g_ref = torch.autograd.grad(o_ref, (qr, kr, vr), do)

    def sh(t):
        x = orc.shard(t, rank, world, layout)
        return x if seq_dim == 1 else x.permute(0, 2, 1, 3).contiguous()

    def unlay(t):
        return t if seq_dim == 1 else t.permute(0, 2, 1, 3)

    ql, kl, vl = (sh(t).requires_grad_() for t in (q, k, v))
    flash = "cuda" if seq_dim == 1 else None

    posted = []  # bytes handed to the ring per forward hop
    plain_post = comm.Ring.post

    def post(self, srcs, dsts):
        posted.append(sum(s.numel() * s.element_size() for s in srcs))
        return plain_post(self, srcs, dsts)

    comm.Ring.post = post
    try:
        o = func(ql, kl, vl, None, flash, causal, True, False, None, list(double_group))
    finally:
        comm.Ring.post = plain_post
    g = torch.autograd.grad(o, (ql, kl, vl), sh(do))

    tol = dict(rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(unlay(o.detach()), orc.shard(o_ref.detach(), rank, world, layout), **tol)
    for got, ref, inp in zip(g, g_ref, (ql, kl, vl)):
        assert got.shape == inp.shape
        torch.testing.assert_close(unlay(got), orc.shard(ref, rank, world, layout), **tol)

    # forward hops: K and V of this rank's shard, Hkv heads -- 1/G of the MHA hop with the same Hq
    assert len(posted) == world - 1, posted
    mha_hop = 2 * B * (S // world) * HQ * D * q.element_size()
    for n in posted:
        assert n * G == mha_hop, (n, G, mha_hop)


def _worker(rank, world, port, case, seq_dim, errq, intra=0):
    try:
        for p in (ROOT, os.path.join(ROOT, "burst-attention_b200"), os.path.join(ROOT, "tests")):
            if p not in sys.path:
                sys.path.insert(0, p)
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        from burst_attn import chunk_ops
        chunk_ops._set_ops_for_testing(_gqa_ops())
        double_group = (None, None)
        if intra:  # hierarchical ring: nodes of `intra` consecutive ranks
            os.environ["BA_DOUBLE_RING"] = "1"
            rows = [list(range(n * intra, (n + 1) * intra)) for n in range(world // intra)]
            cols = [list(c) for c in zip(*rows)]
            mk = lambda ranks: dist.new_subgroups_by_enumeration(ranks, backend="gloo")[0]  # noqa: E731
            double_group = (mk(rows), mk(cols))
        for hkv in HKV_CASES:
            _check_case(rank, world, case, seq_dim, hkv, double_group)
        dist.barrier()
        dist.destroy_process_group()
    except Exception as e:  # noqa: BLE001
        import traceback
        errq.put(f"rank {rank}: {type(e).__name__}: {e}\n{traceback.format_exc()}")
        raise


def _spawn(world, case, seq_dim, intra=0):
    ctx = mp.get_context("spawn")
    errq = ctx.SimpleQueue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, case, seq_dim, errq, intra)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(240)
    errs = []
    while not errq.empty():
        errs.append(errq.get())
    assert not errs, "\n".join(errs)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]


@pytest.mark.parametrize("case,seq_dim", [("none", 1), ("zigzag", 1), ("striped", 1), ("none", 2)])
def test_gqa_world1(case, seq_dim):
    from burst_attn import chunk_ops
    chunk_ops._set_ops_for_testing(_gqa_ops())
    try:
        for hkv in HKV_CASES:
            _check_case(0, 1, case, seq_dim, hkv)
    finally:
        chunk_ops._set_ops_for_testing(None)


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("case,seq_dim", [("none", 1), ("zigzag", 1), ("striped", 1), ("none", 2)])
def test_gqa_ring_matches_dense(world, case, seq_dim):
    _spawn(world, case, seq_dim)


@pytest.mark.parametrize("case", ["none", "zigzag", "striped"])
def test_gqa_double_ring_matches_dense(case):
    """Hierarchical ring, W = 4 as 2 nodes of 2: K/V (Hkv heads) hop inside the node and prefetch across nodes."""
    _spawn(4, case, 1, intra=2)


@pytest.mark.parametrize("seq_dim", [1, 2])
def test_q_heads_not_a_multiple_of_kv_heads_raises(seq_dim):
    from burst_attn import burst_attn_func, chunk_ops
    chunk_ops._set_ops_for_testing(_gqa_ops())
    try:
        q = torch.randn(1, 16, 3, 16, dtype=torch.float64)
        kv = torch.randn(1, 16, 2, 16, dtype=torch.float64)
        if seq_dim == 2:
            q, kv = q.transpose(1, 2).contiguous(), kv.transpose(1, 2).contiguous()
        with pytest.raises(AssertionError, match="multiple"):
            burst_attn_func(q, kv, kv, None, "cuda" if seq_dim == 1 else None, False)
    finally:
        chunk_ops._set_ops_for_testing(None)


@pytest.mark.parametrize("blk", [16, 1000])
def test_gqa_single_gpu_wrappers_cpu(monkeypatch, blk):
    """flash_attn_func / flash_attn_kvpacked_func with nheads_k | nheads (flash-attn's GQA), per-key bias per query
    head, L2 blocking on and off: the Python logic on CPU with the GQA oracle operators; gradients come back with
    the shapes of the inputs."""
    from burst_attn import chunk_ops
    from burst_attn.flash_triton import flash_attn_func, flash_attn_kvpacked_func
    from oracle import attention_oracle as orc
    monkeypatch.setenv("BA_L2_BLOCK", str(blk))
    ops = _gqa_ops()
    ops.tile_head_dims = (16,)
    chunk_ops._set_ops_for_testing(ops)
    try:
        torch.manual_seed(17)
        B, S, D = 2, 70, 16
        for hkv in HKV_CASES:
            G = HQ // hkv
            q, do = (torch.randn(B, S, HQ, D, dtype=torch.float64) for _ in range(2))
            kv = torch.randn(B, S, 2, hkv, D, dtype=torch.float64)
            k, v = kv[:, :, 0].contiguous(), kv[:, :, 1].contiguous()
            bias = torch.randn(1, HQ, 1, S, dtype=torch.float64)
            bias[..., 2::7] = float("-inf")
            for causal in (False, True):
                qr, kr, vr = (t.clone().requires_grad_() for t in (q, k, v))
                o_ref, _ = orc.dense_attention(qr, kr.repeat_interleave(G, 2), vr.repeat_interleave(G, 2), None,
                                               causal, bias=bias)
                dq, dk, dv = torch.autograd.grad(o_ref, (qr, kr, vr), do)
                qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
                o = flash_attn_func(qq, kk, vv, bias, causal)
                g = torch.autograd.grad(o, (qq, kk, vv), do)
                torch.testing.assert_close(o.detach(), o_ref.detach(), rtol=1e-5, atol=1e-5)
                for a, r, inp in zip(g, (dq, dk, dv), (qq, kk, vv)):
                    assert a.shape == inp.shape
                    torch.testing.assert_close(a, r, rtol=1e-5, atol=1e-5)
                qq, pkv = q.clone().requires_grad_(), kv.clone().requires_grad_()
                o = flash_attn_kvpacked_func(qq, pkv, bias, causal)
                gq, gkv = torch.autograd.grad(o, (qq, pkv), do)
                assert gkv.shape == pkv.shape
                torch.testing.assert_close(gq, dq, rtol=1e-5, atol=1e-5)
                torch.testing.assert_close(gkv[:, :, 0], dk, rtol=1e-5, atol=1e-5)
                torch.testing.assert_close(gkv[:, :, 1], dv, rtol=1e-5, atol=1e-5)
        k2 = torch.randn(B, S, 2, D, dtype=torch.float64)
        with pytest.raises(AssertionError, match="multiple"):
            flash_attn_func(q[:, :, :3], k2, k2, None, False)
        with pytest.raises(AssertionError, match="multiple"):
            flash_attn_kvpacked_func(q[:, :, :3], torch.stack([k2, k2], dim=2), None, False)
    finally:
        chunk_ops._set_ops_for_testing(None)
