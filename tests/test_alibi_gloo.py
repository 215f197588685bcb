"""ALiBi without a GPU: the ring drivers' per-launch distances under gloo with fp64 oracle chunk operators
(``oracle_ops``), each run reassembled and compared with the fp64 ALiBi oracle over the full sequence; the flash_attn_*
wrappers' bottom-right positions; argument checks of the public API and of the C-ABI."""
import os

import pytest
import torch
import torch.distributed as dist

import mask_oracle as mo
from ring_harness import double_group, spawn

# window_size values: none, narrower than a shard, two-sided
WINDOWS = [(-1, -1), (5, -1), (7, 4)]


def _slopes(B, H, per_batch):
    """Slopes large enough that a distance one off moves every output well past the tolerance."""
    g = torch.Generator().manual_seed(5)
    if per_batch:
        return 0.2 + 0.6 * torch.rand(B, H, generator=g)
    return 0.2 + 0.6 * torch.rand(H, generator=g)


def _check(rank, world, layout, window, dg=(None, None), S_local=12, Hkv=2, per_batch=False, seq_dim=1):
    from burst_attn import burst_attn_func, burst_attn_func_striped
    from oracle import attention_oracle as orc
    func = burst_attn_func_striped if layout.startswith("striped") else burst_attn_func
    causal = layout in ("zigzag", "striped")
    shard = {"contiguous": "contiguous", "zigzag": "zigzag", "striped": "striped", "striped_nc": "striped"}[layout]
    torch.manual_seed(77)
    B, S, H, D = 2, S_local * world, 4, 8
    q, do = (torch.randn(B, S, H, D, dtype=torch.float64) for _ in range(2))
    k, v = (torch.randn(B, S, Hkv, D, dtype=torch.float64) for _ in range(2))
    slopes = _slopes(B, H, per_batch)
    G = H // Hkv
    o_ref, _, dq_ref, dk_ref, dv_ref = mo.dense_attention_bwd(q, k.repeat_interleave(G, 2), v.repeat_interleave(G, 2),
                                                              do, 0.3, causal, window, mo.as_bh(slopes, B))
    dk_ref, dv_ref = (t.unflatten(2, (Hkv, G)).sum(3) for t in (dk_ref, dv_ref))
    lay = (lambda t: t) if seq_dim == 1 else (lambda t: t.transpose(1, 2).contiguous())
    unlay = (lambda t: t) if seq_dim == 1 else (lambda t: t.transpose(1, 2))
    sh = lambda t: orc.shard(t, rank, world, shard)  # noqa: E731
    ql, kl, vl = (lay(sh(t)).requires_grad_() for t in (q, k, v))
    o = func(ql, kl, vl, 0.3, "cuda" if seq_dim == 1 else None, causal, False, False, None, list(dg), window, slopes)
    g = torch.autograd.grad(o, (ql, kl, vl), lay(sh(do)))
    tol = dict(rtol=1e-5, atol=1e-5)  # fp32 carried state / accumulators in the driver
    name = f"{layout} W={world} window={window} rank={rank}"
    torch.testing.assert_close(unlay(o.detach()), sh(o_ref), **tol, msg=lambda m: f"o {name}: {m}")
    for n, got, ref in zip(("dq", "dk", "dv"), g, (dq_ref, dk_ref, dv_ref)):
        torch.testing.assert_close(unlay(got), sh(ref), **tol, msg=lambda m: f"{n} {name}: {m}")


def _worker(rank, world, port, intra):
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from burst_attn import chunk_ops
    from oracle_ops import OracleOps
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        dg = double_group(rank, world, intra, False) if intra else (None, None)
        for layout in ("contiguous", "zigzag", "striped", "striped_nc"):
            for i, window in enumerate(WINDOWS):
                _check(rank, world, layout, window, dg, Hkv=2 if i % 2 else 4, per_batch=i == 1)
        _check(rank, world, "contiguous", (-1, -1), dg, seq_dim=2)  # [B, H, S, D]
        dist.barrier()
    finally:
        chunk_ops._set_ops_for_testing(None)
        dist.destroy_process_group()


@pytest.mark.parametrize("world,intra", [(2, 0), (4, 0), (4, 2)])
def test_alibi_ring_matches_dense(world, intra):
    """burst_attn_func (contiguous and zigzag shards) and burst_attn_func_striped (causal and not) on flat rings of 2
    and 4 ranks and the 2 x 2 hierarchical ring, with and without a window, GQA and (B, H) slopes, against the fp64
    ALiBi oracle over the full sequence."""
    spawn(_worker, world, (intra,), timeout=300)


@pytest.mark.parametrize("blk", [None, "16"])
def test_alibi_world1_and_l2_blocks(monkeypatch, blk):
    """One rank, with and without L2 blocking (BA_L2_BLOCK = 16: sub-launches whose rows and keys start inside the
    shard, so their distance offsets shift)."""
    from burst_attn import chunk_ops
    from oracle_ops import OracleOps
    if blk:
        monkeypatch.setenv("BA_L2_BLOCK", blk)
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        for layout in ("contiguous", "zigzag", "striped", "striped_nc"):
            for i, window in enumerate(WINDOWS + [(40, 3)]):
                _check(0, 1, layout, window, S_local=70, Hkv=2 if i % 2 else 4, per_batch=i == 1)
    finally:
        chunk_ops._set_ops_for_testing(None)


@pytest.mark.parametrize("blk", [None, "32"])
def test_flash_wrappers_alibi_cpu(monkeypatch, blk):
    """Bottom-right positions (Sq != Sk), windows, GQA and (B, H) slopes through the three wrappers."""
    from burst_attn import chunk_ops
    from burst_attn.flash_triton import flash_attn_func, flash_attn_kvpacked_func, flash_attn_qkvpacked_func
    from oracle_ops import OracleOps
    if blk:
        monkeypatch.setenv("BA_L2_BLOCK", blk)
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        torch.manual_seed(9)
        tol = dict(rtol=1e-5, atol=1e-5)
        for sq, sk in [(70, 70), (50, 110), (110, 45)]:
            q, do = (torch.randn(2, sq, 4, 16, dtype=torch.float64) for _ in range(2))
            k, v = (torch.randn(2, sk, 2, 16, dtype=torch.float64) for _ in range(2))
            for causal in (False, True):
                for per_batch, window in ((False, (-1, -1)), (True, (5, -1)), (False, (30, 50))):
                    slopes = _slopes(2, 4, per_batch)
                    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
                    o = flash_attn_func(qq, kk, vv, None, causal, 0.25, window, slopes)
                    g = torch.autograd.grad(o, (qq, kk, vv), do)
                    ke, ve = k.repeat_interleave(2, 2), v.repeat_interleave(2, 2)
                    o_ref, _, dq, dk, dv = mo.dense_attention_bwd(q, ke, ve, do, 0.25, causal, window,
                                                                  mo.as_bh(slopes, 2))
                    torch.testing.assert_close(o.detach(), o_ref, **tol)
                    torch.testing.assert_close(g[0], dq, **tol)
                    torch.testing.assert_close(g[1], dk.unflatten(2, (2, 2)).sum(3), **tol)
                    torch.testing.assert_close(g[2], dv.unflatten(2, (2, 2)).sum(3), **tol)
                    o2 = flash_attn_kvpacked_func(q, torch.stack([k, v], 2), None, causal, 0.25, window, slopes)
                    torch.testing.assert_close(o2, o_ref, **tol)
            if sq == sk:
                slopes = _slopes(2, 4, False)
                o3 = flash_attn_qkvpacked_func(torch.stack([q, q, q], 2), None, True, 0.25, (9, -1), slopes)
                ref = mo.dense_attention_bwd(q, q, q, do, 0.25, True, (9, -1), mo.as_bh(slopes, 2))[0]
                torch.testing.assert_close(o3, ref, **tol)
    finally:
        chunk_ops._set_ops_for_testing(None)


def _calls_worker(rank, world, port, outdir):
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from burst_attn import burst_attn_func, burst_attn_func_striped, chunk_ops
    from oracle import attention_oracle as orc
    from oracle_ops import OracleOps
    ops = OracleOps()
    chunk_ops._set_ops_for_testing(ops)
    try:
        torch.manual_seed(1)
        q, k, v = (torch.randn(1, 8 * world, 1, 8, dtype=torch.float64) for _ in range(3))
        res = {}
        for name, func, causal, shard in (("contiguous", burst_attn_func, False, "contiguous"),
                                          ("zigzag", burst_attn_func, True, "zigzag"),
                                          ("striped", burst_attn_func_striped, True, "striped")):
            ql, kl, vl = (orc.shard(t, rank, world, shard).requires_grad_() for t in (q, k, v))
            for tag, extra in (("omitted", ()), ("none", ((-1, -1), None))):
                ops.calls.clear()
                o = func(ql, kl, vl, None, "cuda", causal, False, False, None, [None, None], *extra)
                torch.autograd.grad(o.sum(), (ql, kl, vl))
                res[(name, tag)] = list(ops.calls)
        torch.save(res, os.path.join(outdir, f"calls{rank}.pt"))
        dist.barrier()
    finally:
        chunk_ops._set_ops_for_testing(None)
        dist.destroy_process_group()


def test_alibi_none_makes_todays_calls(tmp_path):
    """alibi_slopes=None records exactly the chunk calls of a call without the argument, in every layout (W = 4)."""
    spawn(_calls_worker, 4, (str(tmp_path),), timeout=300)
    for rank in range(4):
        res = torch.load(os.path.join(tmp_path, f"calls{rank}.pt"), weights_only=False)  # oracle_ops.Call records
        for name in ("contiguous", "zigzag", "striped"):
            assert res[(name, "omitted")] == res[(name, "none")], name
            assert all(c.alibi is None for c in res[(name, "none")])


@pytest.mark.parametrize("bad,exc", [(torch.tensor([0.5, 0.25], dtype=torch.float64), TypeError),
                                     ([0.5, 0.25], TypeError),
                                     (torch.tensor([0.5, 0.25, 0.1]), ValueError),
                                     (torch.tensor([[[0.5, 0.25]]]), ValueError),
                                     (torch.tensor([[0.5, 0.25]] * 3), ValueError),
                                     (torch.tensor([0.5, float("inf")]), ValueError),
                                     (torch.tensor([float("nan"), 0.5]), ValueError)])
def test_bad_slopes_raise(bad, exc):
    from burst_attn import burst_attn_func, burst_attn_func_striped, chunk_ops
    from burst_attn.flash_triton import flash_attn_func
    from oracle_ops import OracleOps
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        q = torch.randn(2, 8, 2, 8, dtype=torch.float64)
        for call in (lambda: burst_attn_func(q, q, q, None, "cuda", False, False, False, None, [None, None], (-1, -1),
                                             bad),
                     lambda: burst_attn_func_striped(q, q, q, None, "cuda", True, False, False, None, [None, None],
                                                     (-1, -1), bad),
                     lambda: flash_attn_func(q, q, q, None, False, None, (-1, -1), bad)):
            with pytest.raises(exc, match="alibi_slopes"):
                call()
    finally:
        chunk_ops._set_ops_for_testing(None)


def test_alibi_with_key_bias_raises():
    from burst_attn import chunk_ops
    from burst_attn.flash_triton import flash_attn_func
    from oracle_ops import OracleOps
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        q = torch.randn(1, 8, 2, 8, dtype=torch.float64)
        with pytest.raises(NotImplementedError, match="alibi_slopes"):
            flash_attn_func(q, q, q, torch.zeros(1, 2, 1, 8), False, None, (-1, -1), torch.tensor([0.5, 0.25]))
    finally:
        chunk_ops._set_ops_for_testing(None)


@pytest.fixture(scope="module")
def nat():
    from burst_attn import native
    if not os.path.exists(native.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return native


def test_alibi_entry_points_reject_bad_arguments(nat):
    L = nat.lib()
    assert L.ba_version() >= 203
    z4 = nat.ba_tensor4(None, 0, 0, 0)
    zr = nat.ba_rowstat(None, 0, 0)
    slopes = (nat.ctypes.c_float * 4)(0.5, 0.25, 0.125, 0.0625)
    sp = nat.ctypes.cast(slopes, nat.ctypes.c_void_p)
    fwd = lambda mm, s, sb, ps: L.ba_fwd_chunk_alibi(z4, z4, z4, z4, zr, z4, 1, 128, 128, 4, 2, 128, 1.0, mm, 0, 0,  # noqa
                                                     s, sb, 5, ps, 3, 1, None)
    bwd = lambda mm, s, sb, ps: L.ba_bwd_chunk_alibi(z4, z4, z4, z4, zr, zr, z4, z4, z4, 1, 128, 128, 4, 2, 128, 1.0,  # noqa
                                                     mm, 0, 0, s, sb, 5, ps, 0, 1, None)
    for call in (fwd, bwd):
        assert call(0, None, 0, 1) != 0 and b"slopes" in L.ba_last_error()
        assert call(0, sp, -4, 1) != 0 and b"stride" in L.ba_last_error()
        for ps in (0, -3):
            assert call(0, sp, 0, ps) != 0 and b"position stride" in L.ba_last_error()
        assert call(4, sp, 0, 1) != 0 and b"mask mode" in L.ba_last_error()
        for mm in (0, 1, 3):
            assert call(mm, sp, 4, 2) != 0 and b"null" in L.ba_last_error()  # valid: reaches the operand check
