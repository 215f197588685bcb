"""Packed documents (cu_seqlens) without a GPU: the document oracle, the ring drivers under gloo with the fp64 oracle
chunk operators (oracle_ops), the planner's launches per round, the doc kernels' index arithmetic restated in Python
(doc_index: the deterministic-mode deadlock precondition), and argument checks of the public API and of the C-ABI."""
import ctypes
import os

import pytest
import torch
import torch.distributed as dist

import doc_index as di
import mask_oracle as mo
from ring_harness import double_group, spawn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = dict(rtol=1e-5, atol=1e-5)  # fp32 carried state / accumulators in the driver


def _cus(S):
    """One document; many short ones; zero-length ones; documents across shard edges; edges at 64/128 multiples +-1."""
    return [[0, S], list(range(0, S, 5)) + [S], [0, 0, 3, 3, 17, S - 1, S, S], [0, S // 3, S // 2 + 1, S],
            sorted({0, S} | {x for b in (64, 128) for x in (b - 1, b, b + 1) if 0 < x < S})]


def test_doc_oracle_matches_double_loop():
    torch.manual_seed(2)
    S, cu = 11, [0, 3, 3, 7, 11]
    q, k, v = (torch.randn(1, S, 2, 4, dtype=torch.float64) for _ in range(3))
    for causal, window in ((False, None), (True, None), (True, (2, -1)), (False, (1, 2))):
        o, lse, *_ = mo.dense_attention_bwd(q, k, v, torch.zeros_like(q), 0.5, causal, window, cu=cu)
        for a in range(S):
            d = max(i for i in range(len(cu) - 1) if cu[i] <= a)
            js = [c for c in range(cu[d], cu[d + 1]) if (not causal or c <= a) and
                  (window is None or ((window[0] < 0 or c >= a - window[0]) and (window[1] < 0 or causal or
                                                                                  c <= a + window[1])))]
            s = torch.stack([(q[0, a] * k[0, c]).sum(-1) * 0.5 for c in js])
            torch.testing.assert_close(o[0, a], torch.einsum("nh,nhd->hd", torch.softmax(s, 0), v[0, js]))
            torch.testing.assert_close(lse[0, :, a], torch.logsumexp(s, 0))
    # one document is the plain windowed oracle
    o1 = mo.dense_attention_bwd(q, k, v, q, 0.5, True, (3, -1), cu=[0, S])
    o2 = mo.dense_attention_bwd(q, k, v, q, 0.5, True, (3, -1))
    for a, b in zip(o1, o2):
        torch.testing.assert_close(a, b)


def _check(rank, world, layout, cu, window=(-1, -1), causal=None, dg=(None, None), S_local=12, B=1, Hkv=2,
           seq_dim=1):
    from burst_attn import burst_attn_func, burst_attn_func_striped, chunk_ops
    from oracle import attention_oracle as orc
    func = burst_attn_func_striped if layout == "striped" else burst_attn_func
    causal = layout != "contiguous" if causal is None else causal
    torch.manual_seed(77)
    S, H, D = S_local * world, 4, 8
    q, do = (torch.randn(B, S, H, D, dtype=torch.float64) for _ in range(2))
    k, v = (torch.randn(B, S, Hkv, D, dtype=torch.float64) for _ in range(2))
    G = H // Hkv
    o_ref, _, dq_ref, dk_ref, dv_ref = mo.dense_attention_bwd(q, k.repeat_interleave(G, 2), v.repeat_interleave(G, 2),
                                                              do, 0.3, causal, window, cu=cu)
    dk_ref, dv_ref = (t.unflatten(2, (Hkv, G)).sum(3) for t in (dk_ref, dv_ref))
    lay = (lambda t: t) if seq_dim == 1 else (lambda t: t.permute(0, 2, 1, 3).contiguous())
    sh = lambda t: lay(orc.shard(t, rank, world, layout))  # noqa: E731
    ql, kl, vl = (sh(t).requires_grad_() for t in (q, k, v))
    ops = chunk_ops.get_ops()
    ops.pairs.clear()
    o = func(ql, kl, vl, 0.3, "cuda" if seq_dim == 1 else None, causal, False, False, None, list(dg), window, None,
             torch.tensor(cu, dtype=torch.int32))
    g = torch.autograd.grad(o, (ql, kl, vl), sh(do))
    torch.testing.assert_close(o.detach(), sh(o_ref), **TOL)
    for got, ref in zip(g, (dq_ref, dk_ref, dv_ref)):
        torch.testing.assert_close(got, sh(ref), **TOL)
    # the forward's launches attend exactly this rank's visible (query, key) position pairs, each once
    pos = orc.shard(torch.arange(S).view(1, S, 1, 1), rank, world, layout).view(-1).tolist()
    vis = mo.same_doc(torch.arange(S), torch.arange(S), cu)
    w = mo.window_mask(S, S, window, causal)
    vis = vis if w is None else vis & w
    want = {(a, c) for a in pos for c in vis[a].nonzero().view(-1).tolist()}
    assert ops.pairs == want


def _worker(rank, world, port, intra):
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from burst_attn import chunk_ops
    from oracle_ops import OracleOps
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        dg = double_group(rank, world, intra, False) if intra else (None, None)
        S = 12 * world
        for layout in ("contiguous", "zigzag", "striped"):
            for cu in _cus(S):
                _check(rank, world, layout, cu, dg=dg)
            _check(rank, world, layout, _cus(S)[3], window=(5, -1), dg=dg)
            # burst_attn_func's shards follow causal (zigzag iff causal); striped shards run either way
            _check(rank, world, layout, _cus(S)[2], causal=False if layout == "striped" else None, dg=dg, B=2, Hkv=4)
            if layout == "contiguous":
                _check(rank, world, layout, _cus(S)[1], window=(3, 2), dg=dg, seq_dim=2)
        dist.barrier()
    finally:
        chunk_ops._set_ops_for_testing(None)
        dist.destroy_process_group()


@pytest.mark.parametrize("world,intra", [(2, 0), (4, 0), (4, 2)])
def test_doc_ring_matches_dense(world, intra):
    """burst_attn_func (contiguous and zigzag shards) and burst_attn_func_striped with cu_seqlens on flat rings of 2
    and 4 ranks and the 2 x 2 hierarchical ring, against the fp64 document oracle, causal and not, with windows, GQA,
    B = 2 and both sequence axes."""
    spawn(_worker, world, (intra,), timeout=600)


@pytest.mark.parametrize("blk", [None, "16"])
def test_doc_world1_and_l2_blocks(monkeypatch, blk):
    from burst_attn import chunk_ops
    from oracle_ops import OracleOps
    if blk:
        monkeypatch.setenv("BA_L2_BLOCK", blk)
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        for layout in ("contiguous", "zigzag", "striped"):
            for cu in _cus(70):
                _check(0, 1, layout, cu, S_local=70)
                _check(0, 1, layout, cu, window=(9, -1), S_local=70)
    finally:
        chunk_ops._set_ops_for_testing(None)


@pytest.mark.parametrize("blk", [None, "32"])
def test_flash_attn_varlen_func_cpu(monkeypatch, blk):
    from burst_attn import chunk_ops
    from burst_attn.flash_triton import flash_attn_varlen_func
    from oracle_ops import OracleOps
    if blk:
        monkeypatch.setenv("BA_L2_BLOCK", blk)
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        torch.manual_seed(4)
        T = 90
        q, do = (torch.randn(T, 4, 16, dtype=torch.float64) for _ in range(2))
        k, v = (torch.randn(T, 2, 16, dtype=torch.float64) for _ in range(2))
        for cu in _cus(T):
            cut = torch.tensor(cu, dtype=torch.int32)
            longest = max(b - a for a, b in zip(cu, cu[1:]))
            for causal, window in ((False, (-1, -1)), (True, (-1, -1)), (True, (7, -1)), (False, (4, 9))):
                chunk_ops.get_ops().pairs.clear()
                qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
                o = flash_attn_varlen_func(qq, kk, vv, cut, cut, longest, longest, 0.0, 0.25, causal, window)
                g = torch.autograd.grad(o, (qq, kk, vv), do)
                o_r, _, dq, dk, dv = mo.dense_attention_bwd(q[None], k[None].repeat_interleave(2, 2),
                                                            v[None].repeat_interleave(2, 2), do[None], 0.25, causal,
                                                            window, cu=cu)
                torch.testing.assert_close(o.detach(), o_r[0], **TOL)
                torch.testing.assert_close(g[0], dq[0], **TOL)
                torch.testing.assert_close(g[1], dk[0].unflatten(1, (2, 2)).sum(2), **TOL)
                torch.testing.assert_close(g[2], dv[0].unflatten(1, (2, 2)).sum(2), **TOL)
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
        S_local = 8
        S = S_local * world
        torch.manual_seed(1)
        q, k, v = (torch.randn(1, S, 1, 8, dtype=torch.float64) for _ in range(3))
        inside = torch.tensor([0] + [x for r in range(world) for x in (r * S_local + 3, (r + 1) * S_local)],
                              dtype=torch.int32)
        res = {}
        for name, func, causal, shard in (("contiguous", burst_attn_func, False, "contiguous"),
                                          ("zigzag", burst_attn_func, True, "zigzag"),
                                          ("striped", burst_attn_func_striped, True, "striped")):
            ql, kl, vl = (orc.shard(t, rank, world, shard).requires_grad_() for t in (q, k, v))
            for tag, extra in (("inside", ((-1, -1), None, inside)),):
                ops.calls.clear()
                ops.pairs.clear()
                o = func(ql, kl, vl, None, "cuda", causal, False, False, None, [None, None], *extra)
                torch.autograd.grad(o.sum(), (ql, kl, vl))
                res[(name, tag)] = list(ops.calls)
        torch.save(res, os.path.join(outdir, f"calls{rank}.pt"))
        dist.barrier()
    finally:
        chunk_ops._set_ops_for_testing(None)
        dist.destroy_process_group()


def test_rounds_without_a_shared_document_launch_nothing(tmp_path):
    """W = 4, contiguous shards, documents inside single shards: only the own round launches (one forward and one
    backward kernel over the own shard, whose two documents the kernels mask apart).  (That calls without cu_seqlens
    plan exactly as before is pinned by tests/test_launch_plans.py against tests/golden/plans.json.)"""
    world = 4
    spawn(_calls_worker, world, (str(tmp_path),), timeout=300)
    for rank in range(world):
        res = torch.load(os.path.join(tmp_path, f"calls{rank}.pt"), weights_only=False)  # oracle_ops.Call records
        calls = res[("contiguous", "inside")]
        fwd = [c for c in calls if c[0] == "fwd"]
        bwd = [c for c in calls if c[0] == "bwd"]
        assert len(fwd) == 1 and len(bwd) == 1, calls  # one launch over the own shard's two documents
        for c in fwd + bwd:
            assert c[1][1] == 8 and c[2][1] == 8 and c[-1][1:3] == (8 * rank, 8 * rank), c


def _plan_launches(layout, world, S_local, cu, band):
    """Every (rank, round) launch of the planner with its positions, as doc_index launches."""
    from burst_attn.burst_attn_interface import _fwd_band_launches, _bwd_band_launches, _positions, _round_pieces
    out = []
    for iq in range(world):
        for jk in range(world):
            pieces = _round_pieces(layout, world, iq, jk, S_local, S_local, band, False, cu)
            pos_q, ps = _positions(layout, world, iq, S_local)
            pos_k, _ = _positions(layout, world, jk, S_local)
            for q0, qn, k0, kn, lo, hi in _fwd_band_launches(pieces) + _bwd_band_launches(pieces):
                out.append(di.Launch(qn, kn, hi is not None, 0 if hi is None else hi, lo, cu, pos_q(q0), pos_k(k0),
                                     ps))
    return out


def test_doc_kernel_index_arithmetic_sweep():
    """doc_index.check_launch on the sweep: the forward's row limits and tile ranges, the backward's Q-block ranges and
    staged offsets, and the deterministic mode's "x visits i iff x_min(i) <= x <= x_max(i)"."""
    for case in di.sweep():
        di.check_launch(di.Launch(*case))


def test_doc_kernel_index_arithmetic_on_ring_launches(monkeypatch):
    """The same on every launch the planner makes for rings of W = 2, 4 and 8 in all three layouts (L2 blocks of 128
    rows / keys, so sub-launches are checked too)."""
    monkeypatch.setenv("BA_L2_BLOCK", "128")
    n = 0
    for world in (2, 4, 8):
        S_local = 192
        S = S_local * world
        for cu in ([0, 127, 128, 129, 300, 301, S - 1, S], list(range(0, S, 170)) + [S]):
            for layout, band in (("contiguous", (None, None)), ("zigzag", (None, 0)), ("striped", (None, 0)),
                                 ("striped", (150, None)), ("contiguous", (200, 0))):
                for L in _plan_launches(layout, world, S_local, cu, band):
                    di.check_launch(L)
                    n += 1
    assert n > 100


@pytest.mark.parametrize("mutant", di.MUTANTS)
def test_index_check_rejects_mutants(mutant):
    """Each deliberate fault of the restated arithmetic fails check_launch on some sweep case."""
    for case in di.sweep():
        try:
            di.check_launch(di.Launch(*case), mutant)
        except AssertionError:
            return
    pytest.fail(f"{mutant} passed every sweep case")


@pytest.mark.parametrize("bad,err,match", [
    ([1, 24], ValueError, "start at 0"), ([0, 23], ValueError, "end at"), ([0, 13, 12, 24], ValueError,
                                                                           "non-decreasing"),
    ([[0, 24]], ValueError, "1-D"), ([0], ValueError, "1-D"), ("int64", TypeError, "int32"), ("list", TypeError,
                                                                                                "torch.Tensor")])
def test_bad_cu_seqlens_raise(bad, err, match):
    from burst_attn import burst_attn_func, burst_attn_func_striped, chunk_ops
    from burst_attn.flash_triton import flash_attn_varlen_func
    from oracle_ops import OracleOps
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        q = torch.randn(1, 24, 2, 8, dtype=torch.float64)
        cu = {"int64": torch.tensor([0, 24]), "list": [0, 24]}.get(bad) if isinstance(bad, str) else \
            torch.tensor(bad, dtype=torch.int32)
        for f in (burst_attn_func, burst_attn_func_striped):
            with pytest.raises(err, match=match):
                f(q, q, q, None, "cuda", False, False, False, None, [None, None], (-1, -1), None, cu)
        with pytest.raises(err, match=match):
            flash_attn_varlen_func(q[0], q[0], q[0], cu, cu, 24, 24)
    finally:
        chunk_ops._set_ops_for_testing(None)


def test_unsupported_combinations_raise():
    from burst_attn import burst_attn_func, chunk_ops
    from burst_attn.flash_triton import flash_attn_varlen_func
    from oracle_ops import OracleOps
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        q = torch.randn(24, 2, 8, dtype=torch.float64)
        cu = torch.tensor([0, 10, 24], dtype=torch.int32)
        with pytest.raises(NotImplementedError, match="alibi_slopes"):
            burst_attn_func(q[None], q[None], q[None], None, "cuda", False, False, False, None, [None, None], (-1, -1),
                            torch.ones(2), cu)
        for kw, match in ((dict(dropout_p=0.1), "dropout"), (dict(softcap=5.0), "softcap"),
                          (dict(alibi_slopes=torch.ones(2)), "alibi"), (dict(return_attn_probs=True), "attn_probs")):
            with pytest.raises(NotImplementedError, match=match):
                flash_attn_varlen_func(q, q, q, cu, cu, 14, 14, **kw)
        with pytest.raises(NotImplementedError, match="cu_seqlens_q must equal"):
            flash_attn_varlen_func(q, q, q, cu, torch.tensor([0, 12, 24], dtype=torch.int32), 14, 14)
        with pytest.raises(ValueError, match="max_seqlen_q"):
            flash_attn_varlen_func(q, q, q, cu, cu, 13, 14)
    finally:
        chunk_ops._set_ops_for_testing(None)


@pytest.fixture(scope="module")
def nat():
    from burst_attn import native
    if not os.path.exists(native.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return native


def test_doc_entry_points_check_arguments(nat):
    L = nat.lib()
    assert L.ba_version() >= 204
    z4 = nat.ba_tensor4(None, 0, 0, 0)
    zr = nat.ba_rowstat(None, 0, 0)
    cu = ctypes.c_void_p(16)  # an aligned, non-null address: the checks never read it
    fwd = lambda cu, n, qp, kp, ps: L.ba_fwd_chunk_doc(z4, z4, z4, z4, zr, z4, 1, 128, 128, 4, 2, 128, 1.0, 1, 0,  # noqa
                                                       0, cu, n, qp, kp, ps, 3, 1, None)
    bwd = lambda cu, n, qp, kp, ps: L.ba_bwd_chunk_doc(z4, z4, z4, z4, zr, zr, z4, z4, z4, 1, 128, 128, 4, 2, 128,  # noqa
                                                       1.0, 1, 0, 0, cu, n, qp, kp, ps, 0, 1, None)
    for call in (fwd, bwd):
        assert call(None, 1, 0, 0, 1) != 0 and b"null cu_seqlens" in L.ba_last_error()
        assert call(cu, 0, 0, 0, 1) != 0 and b"n_docs" in L.ba_last_error()
        assert call(cu, 1, 0, 0, 0) != 0 and b"stride" in L.ba_last_error()
        assert call(cu, 1, -1, 0, 1) != 0 and b"q_pos0" in L.ba_last_error()
        assert call(cu, 1, 2 ** 31 - 100, 0, 1) != 0 and b"int32" in L.ba_last_error()
        assert call(cu, 1, 0, 0, 1) != 0 and b"null" in L.ba_last_error()  # valid: reaches the operand check
    for name in ("ba_fwd_chunk_doc", "ba_bwd_chunk_doc"):
        assert hasattr(ctypes.CDLL(nat.LIB_PATH), name) and name in nat.exported_symbols()

