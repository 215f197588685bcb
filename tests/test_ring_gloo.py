"""World-size 2 to 8 CPU tests (gloo) of the N>1 path: the ring drivers behind
burst_attn_func / burst_attn_func_striped -- K/V rotation, the Q-bundle + dQ
ring of the backward, zigzag / striped shard views, the hierarchical ring --
run with the oracle-backed chunk operators injected (tests only) and are
compared, through autograd, with dense attention on the full sequence (the
reference's protocol, test/test_burst.py:159-219).  With grouped-query K/V
(fewer heads than Q) the reference is dense attention on K/V expanded per
group, and each forward hop must carry 1/G of the bytes of the same call with
MHA K/V."""
import os
import sys

import pytest
import torch
import torch.distributed as dist

from ring_harness import double_group, install_staged_transport, spawn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


HQ = 4
HKV_CASES = (2, 1)  # grouped-query K/V: G = 2 (GQA) and G = Hq (MQA)


def _check(ops, rank, world, case, seq_dim, hq, hkv, double_group=(None, None)):
    """One call of the ring driver on this rank, forward and backward, against dense attention."""
    from burst_attn import burst_attn_func, burst_attn_func_striped, comm
    from oracle import attention_oracle as orc

    func, causal, layout = {
        "none": (burst_attn_func, False, "contiguous"),
        "zigzag": (burst_attn_func, True, "zigzag"),
        "striped": (burst_attn_func_striped, True, "striped"),
    }[case]
    G = hq // hkv
    torch.manual_seed(1234)  # same full tensors on every rank (the reference broadcasts from rank 0)
    B, S, D = 2, 8 * 2 * world, 16
    q = torch.randn(B, S, hq, D, dtype=torch.float64)
    k, v = (torch.randn(B, S, hkv, D, dtype=torch.float64) for _ in range(2))
    do = torch.randn(B, S, hq, D, dtype=torch.float64)
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

    ops.calls.clear()
    comm.Ring.post = post
    try:
        o = func(ql, kl, vl, None, flash, causal, True, False, None, list(double_group))
    finally:
        comm.Ring.post = plain_post
    g = torch.autograd.grad(o, (ql, kl, vl), sh(do))
    tol = dict(rtol=1e-5, atol=1e-5)  # fp32 carried state / accumulators in the driver
    torch.testing.assert_close(unlay(o.detach()), orc.shard(o_ref.detach(), rank, world, layout), **tol)
    for got, ref, inp in zip(g, g_ref, (ql, kl, vl)):
        assert got.shape == inp.shape
        torch.testing.assert_close(unlay(got), orc.shard(ref, rank, world, layout), **tol)
    # user inputs must not have been clobbered (the reference reuses k, v, q, dO as receive buffers)
    torch.testing.assert_close(unlay(kl.detach()), orc.shard(k, rank, world, layout))
    # forward hops: K and V of this rank's shard, Hkv heads -- 1/G of the MHA hop with the same Hq
    assert len(posted) == world - 1, posted
    mha_hop = 2 * B * (S // world) * hq * D * q.element_size()
    for n in posted:
        assert n * G == mha_hop, (n, G, mha_hop)
    # one chunk launch per round, no copies: W forward rounds (+1 cast in the zigzag tail case)
    nf = sum(1 for c in ops.calls if c[0] == "fwd")
    nb = sum(1 for c in ops.calls if c[0] == "bwd")
    if not os.environ.get("BA_TEST_NO_LAUNCH_COUNT"):
        assert nf == world and nb == world, (nf, nb)


def _worker(rank, world, port, case, seq_dim, intra, dq_groups, gqa):
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from burst_attn import chunk_ops
    from oracle_ops import OracleOps
    ops = OracleOps()
    chunk_ops._set_ops_for_testing(ops)
    if os.environ.get("BA_TEST_DEFERRED"):
        install_staged_transport()
    dg = double_group(rank, world, intra, dq_groups) if intra else (None, None)
    if not (case != "none" and seq_dim == 2):  # reference asserts causal needs flash == "cuda"
        for hq, hkv in ([(HQ, h) for h in HKV_CASES] if gqa else [(3, 3)]):
            _check(ops, rank, world, case, seq_dim, hq, hkv, dg)
    dist.barrier()
    dist.destroy_process_group()


def _spawn(world, case, seq_dim=1, intra=0, dq_groups=False, gqa=False):
    """Run _worker on `world` gloo ranks and fail with every rank's traceback."""
    spawn(_worker, world, (case, seq_dim, intra, dq_groups, gqa), timeout=240)


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("case", ["none", "zigzag", "striped"])
def test_ring_driver_matches_dense(world, case):
    _spawn(world, case)


@pytest.mark.parametrize("world,intra,case,dq_groups", [
    (4, 2, "none", False), (4, 2, "zigzag", True), (4, 2, "striped", False),
    (6, 3, "zigzag", False), (6, 2, "none", True), (6, 2, "striped", False),
    (8, 4, "striped", True), (8, 2, "zigzag", False),
])
def test_double_ring_matches_dense(world, intra, case, dq_groups):
    """Hierarchical (double) ring, W = L*M with (L, M) in {(2,2), (3,2), (2,3), (4,2), (2,4)}: K/V and Q-bundle prefetch
    across nodes, dQ node sums chained along the inter-node ring (reference test_burst.py:239-247
    ``double_ring`` axis)."""
    _spawn(world, case, intra=intra, dq_groups=dq_groups)


@pytest.mark.parametrize("world,intra,case", [(4, 0, "none"), (4, 0, "zigzag"), (4, 0, "striped"),
                                              (4, 2, "zigzag"), (6, 2, "striped"), (6, 3, "none")])
def test_no_buffer_hazards_with_asynchronous_transport(world, intra, case, monkeypatch):
    """Flat and hierarchical rings under a transport that only moves data at ``wait`` and poisons the
    destinations at ``post`` (see ring_harness.install_staged_transport): what the side-stream transport does on GPUs."""
    monkeypatch.setenv("BA_TEST_DEFERRED", "1")
    monkeypatch.setenv("BA_RING_TRANSPORT", "ce")  # CPU tensors still travel over gloo; turns on the arena check
    _spawn(world, case, intra=intra)


def test_ring_driver_normal_layout_world2():
    _spawn(2, "none", seq_dim=2)


def test_single_process_world1_cpu():
    """W=1 through the same driver (no process group needed)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from burst_attn import burst_attn_func, chunk_ops
    from oracle import attention_oracle as orc
    from oracle_ops import OracleOps
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        torch.manual_seed(0)
        q, k, v, do = (torch.randn(1, 32, 2, 16, dtype=torch.float64) for _ in range(4))
        for causal in (False, True):
            qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
            o = burst_attn_func(qq, kk, vv, None, "cuda", causal)
            g = torch.autograd.grad(o, (qq, kk, vv), do)
            o_ref, _, dq, dk, dv = orc.dense_attention_bwd(q, k, v, do, None, causal)
            torch.testing.assert_close(o.detach(), o_ref, rtol=1e-5, atol=1e-5)
            for a, b in zip(g, (dq, dk, dv)):
                torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5)
    finally:
        chunk_ops._set_ops_for_testing(None)


def test_head_dim_padding_world1_cpu():
    """A head_dim the tile kernels are not built for (64 and 128 on the GPU; (8, 32) faked here) is zero-padded
    once per call by the driver up to the next tile width and sliced off again -- exact for O, dQ, dK, dV."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from burst_attn import burst_attn_func, burst_attn_func_striped, chunk_ops
    from oracle import attention_oracle as orc
    from oracle_ops import OracleOps
    ops = OracleOps()
    ops.tile_head_dims = (8, 32)
    chunk_ops._set_ops_for_testing(ops)
    try:
        torch.manual_seed(5)
        q, k, v, do = (torch.randn(2, 40, 3, 16, dtype=torch.float64) for _ in range(4))
        for func, causal in ((burst_attn_func, False), (burst_attn_func, True), (burst_attn_func_striped, True)):
            ops.calls.clear()
            qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
            o = func(qq, kk, vv, None, "cuda", causal)
            assert o.shape == q.shape and o.is_contiguous()
            g = torch.autograd.grad(o, (qq, kk, vv), do)
            assert all(c[1][-1] == 32 for c in ops.calls if c[0] in ("fwd", "bwd"))  # the tile saw padded heads
            o_ref, _, dq, dk, dv = orc.dense_attention_bwd(q, k, v, do, None, causal)
            torch.testing.assert_close(o.detach(), o_ref, rtol=1e-5, atol=1e-5)
            for a, b in zip(g, (dq, dk, dv)):
                assert a.shape == b.shape
                torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5)
        # normal layout [B, H, S, D]
        p = lambda t: t.permute(0, 2, 1, 3).contiguous()  # noqa: E731
        qq, kk, vv = (p(t).requires_grad_() for t in (q, k, v))
        o = burst_attn_func(qq, kk, vv, None, None, False)
        g = torch.autograd.grad(o, (qq, kk, vv), p(do))
        o_ref, _, dq, dk, dv = orc.dense_attention_bwd(q, k, v, do, None, False)
        torch.testing.assert_close(o.detach(), p(o_ref), rtol=1e-5, atol=1e-5)
        for a, b in zip(g, (dq, dk, dv)):
            torch.testing.assert_close(a, p(b), rtol=1e-5, atol=1e-5)
    finally:
        chunk_ops._set_ops_for_testing(None)


@pytest.mark.parametrize("blk", [16, 24])
def test_l2_blocking_of_rounds_matches_dense(monkeypatch, blk):
    """The driver splits a round into L2-sized sub-launches (carried state forward, row blocks backward,
    causal offsets for views); with a tiny block size every code path runs on CPU."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from burst_attn import burst_attn_func, burst_attn_func_striped, chunk_ops
    from oracle import attention_oracle as orc
    from oracle_ops import OracleOps
    monkeypatch.setenv("BA_L2_BLOCK", str(blk))
    ops = OracleOps()
    chunk_ops._set_ops_for_testing(ops)
    try:
        torch.manual_seed(3)
        S = 100  # ragged against the block size and far above 1.5 blocks
        q, k, v, do = (torch.randn(2, S, 2, 16, dtype=torch.float64) for _ in range(4))
        for func, causal in ((burst_attn_func, False), (burst_attn_func, True), (burst_attn_func_striped, True)):
            ops.calls.clear()
            qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
            o = func(qq, kk, vv, None, "cuda", causal)
            g = torch.autograd.grad(o, (qq, kk, vv), do)
            o_ref, _, dq, dk, dv = orc.dense_attention_bwd(q, k, v, do, None, causal)
            torch.testing.assert_close(o.detach(), o_ref, rtol=1e-5, atol=1e-5)
            for a, b in zip(g, (dq, dk, dv)):
                torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5)
            assert sum(1 for c in ops.calls if c[0] == "fwd") > 1 and sum(1 for c in ops.calls if c[0] == "bwd") > 1
    finally:
        chunk_ops._set_ops_for_testing(None)


def test_l2_blocking_random_shapes(monkeypatch):
    """Seeded sweep over (S, block size, batch, heads, causal flavour): the offset / view arithmetic of the
    L2-blocked rounds (row starts rounded to tile pairs, causal offsets of sub-views, ragged tails) against
    dense attention, forward and backward."""
    import random
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from burst_attn import burst_attn_func, burst_attn_func_striped, chunk_ops
    from oracle import attention_oracle as orc
    from oracle_ops import OracleOps
    ops = OracleOps()
    chunk_ops._set_ops_for_testing(ops)
    rng = random.Random(20240917)
    try:
        for case in range(24):
            S = rng.choice([17, 64, 100, 255, 256, 257, 300, 513, 640])
            blk = rng.choice([8, 16, 24, 100, 128, 256])
            Bn, Hn = rng.choice([1, 2]), rng.choice([1, 3])
            func, causal = rng.choice([(burst_attn_func, False), (burst_attn_func, True),
                                       (burst_attn_func_striped, True)])
            if causal and func is burst_attn_func and S % 2:
                S += 1  # zigzag halves
            monkeypatch.setenv("BA_L2_BLOCK", str(blk))
            torch.manual_seed(case)
            q, k, v, do = (torch.randn(Bn, S, Hn, 8, dtype=torch.float64) for _ in range(4))
            qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
            o = func(qq, kk, vv, None, "cuda", causal)
            g = torch.autograd.grad(o, (qq, kk, vv), do)
            o_ref, _, dq, dk, dv = orc.dense_attention_bwd(q, k, v, do, None, causal)
            msg = f"case {case}: S={S} blk={blk} B={Bn} H={Hn} {func.__name__} causal={causal}"
            torch.testing.assert_close(o.detach(), o_ref, rtol=1e-5, atol=1e-5, msg=lambda m: f"{msg}: {m}")
            for a, b in zip(g, (dq, dk, dv)):
                torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5, msg=lambda m: f"{msg}: {m}")
    finally:
        chunk_ops._set_ops_for_testing(None)


@pytest.mark.parametrize("case", ["none", "zigzag", "striped"])
def test_ring_driver_with_l2_blocking_world2(case, monkeypatch):
    """Ring rounds + L2 blocking together (blocks of 8 rows/keys, S_local = 16): half views of the
    zigzag rounds and the causal offsets compose."""
    monkeypatch.setenv("BA_L2_BLOCK", "8")
    monkeypatch.setenv("BA_TEST_NO_LAUNCH_COUNT", "1")
    _spawn(2, case)


@pytest.mark.parametrize("blk", [16, 1000])
def test_single_gpu_wrappers_packed_bias_blocked_cpu(monkeypatch, blk):
    """burst_attn.flash_triton (flash_attn_func / _kvpacked_func / _qkvpacked_func): strided views of the packed
    tensors, bottom-right-aligned causal with Sq != Sk, per-key bias narrowed per L2 block -- the Python logic,
    on CPU with oracle-backed chunk operators, against dense attention."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from burst_attn import chunk_ops
    from burst_attn.flash_triton import flash_attn_func, flash_attn_kvpacked_func, flash_attn_qkvpacked_func
    from oracle import attention_oracle as orc
    from oracle_ops import OracleOps
    monkeypatch.setenv("BA_L2_BLOCK", str(blk))
    ops = OracleOps()
    ops.tile_head_dims = (16,)
    chunk_ops._set_ops_for_testing(ops)
    try:
        torch.manual_seed(11)
        B, S, H, D = 2, 70, 2, 16
        qkv = torch.randn(B, S, 3, H, D, dtype=torch.float64)
        do = torch.randn(B, S, H, D, dtype=torch.float64)
        bias = torch.randn(1, H, 1, S, dtype=torch.float64)
        bias[..., 3::5] = float("-inf")
        q, k, v = (qkv[:, :, i].contiguous() for i in range(3))
        for causal in (False, True):
            o_ref, _, dq, dk, dv = orc.dense_attention_bwd(q, k, v, do, None, causal, bias=bias)
            p = qkv.clone().requires_grad_()
            o = flash_attn_qkvpacked_func(p, bias, causal)
            (dqkv,) = torch.autograd.grad(o, (p,), do)
            torch.testing.assert_close(o.detach(), o_ref, rtol=1e-5, atol=1e-5)
            for i, r in enumerate((dq, dk, dv)):
                torch.testing.assert_close(dqkv[:, :, i], r, rtol=1e-5, atol=1e-5)
            qq, kv = q.clone().requires_grad_(), qkv[:, :, 1:].clone().requires_grad_()
            o = flash_attn_kvpacked_func(qq, kv, bias, causal)
            gq, gkv = torch.autograd.grad(o, (qq, kv), do)
            torch.testing.assert_close(gq, dq, rtol=1e-5, atol=1e-5)
            torch.testing.assert_close(gkv[:, :, 0], dk, rtol=1e-5, atol=1e-5)
            torch.testing.assert_close(gkv[:, :, 1], dv, rtol=1e-5, atol=1e-5)
        # Sq != Sk, causal aligned bottom-right (the last query sees every key), no bias
        qs, dos = q[:, 30:].contiguous(), do[:, 30:].contiguous()
        o_ref, _, dq, dk, dv = orc.dense_attention_bwd(qs, k, v, dos, None, True)
        qq, kk, vv = (t.clone().requires_grad_() for t in (qs, k, v))
        o = flash_attn_func(qq, kk, vv, None, True)
        g = torch.autograd.grad(o, (qq, kk, vv), dos)
        torch.testing.assert_close(o.detach(), o_ref, rtol=1e-5, atol=1e-5)
        for a, r in zip(g, (dq, dk, dv)):
            torch.testing.assert_close(a, r, rtol=1e-5, atol=1e-5)
        with pytest.raises(NotImplementedError):
            flash_attn_func(qq, kk, vv, torch.zeros(1, H, 40, S), False)
    finally:
        chunk_ops._set_ops_for_testing(None)


@pytest.mark.parametrize("case,seq_dim", [("none", 1), ("zigzag", 1), ("striped", 1), ("none", 2)])
def test_gqa_world1(case, seq_dim):
    """Grouped-query K/V (Hkv < Hq) through the driver at W = 1, in-process."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from burst_attn import chunk_ops
    from oracle_ops import OracleOps
    ops = OracleOps()
    chunk_ops._set_ops_for_testing(ops)
    try:
        for hkv in HKV_CASES:
            _check(ops, 0, 1, case, seq_dim, HQ, hkv)
    finally:
        chunk_ops._set_ops_for_testing(None)


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("case,seq_dim", [("none", 1), ("zigzag", 1), ("striped", 1), ("none", 2)])
def test_gqa_ring_matches_dense(world, case, seq_dim):
    _spawn(world, case, seq_dim, gqa=True)


@pytest.mark.parametrize("case", ["none", "zigzag", "striped"])
def test_gqa_double_ring_matches_dense(case):
    """Hierarchical ring, W = 4 as 2 nodes of 2: K/V (Hkv heads) hop inside the node and prefetch across nodes."""
    _spawn(4, case, intra=2, gqa=True)


@pytest.mark.parametrize("seq_dim", [1, 2])
def test_q_heads_not_a_multiple_of_kv_heads_raises(seq_dim):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from burst_attn import burst_attn_func, chunk_ops
    from oracle_ops import OracleOps
    chunk_ops._set_ops_for_testing(OracleOps())
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
    head, L2 blocking on and off: the Python logic on CPU with the oracle operators; gradients come back with the
    shapes of the inputs."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from burst_attn import chunk_ops
    from burst_attn.flash_triton import flash_attn_func, flash_attn_kvpacked_func
    from oracle import attention_oracle as orc
    from oracle_ops import OracleOps
    monkeypatch.setenv("BA_L2_BLOCK", str(blk))
    ops = OracleOps()
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
