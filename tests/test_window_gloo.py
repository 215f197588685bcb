"""Sliding-window attention without a GPU: the windowed oracle, the ring drivers' per-round bands under gloo with the
fp64 oracle chunk operators, the launches they skip, argument checks of the public API and of the C-ABI."""
import ctypes
import os
import sys

import pytest
import torch
import torch.distributed as dist

import mask_oracle as mo
from ring_harness import double_group, spawn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (left, right): narrower than a shard, spanning several shards, two-sided, the diagonal only
WINDOWS = [(5, -1), (23, -1), (7, 4), (0, 0), (-1, 6)]


def test_window_mask_matches_double_loop():
    for sq, sk in [(7, 7), (5, 11), (9, 4)]:
        for causal in (False, True):
            for left, right in WINDOWS + [(-1, -1), (2, 0), (30, 30)]:
                m = mo.window_mask(sq, sk, (left, right), causal)
                r = 0 if causal else right
                for i in range(sq):
                    for j in range(sk):
                        p = i + sk - sq
                        want = (left < 0 or j >= p - left) and (r < 0 or j <= p + r)
                        assert (True if m is None else bool(m[i, j])) == want, (sq, sk, causal, left, right, i, j)


def test_windowed_oracle_matches_double_loop_and_causal():
    from oracle import attention_oracle as orc
    torch.manual_seed(3)
    q, k, v = (torch.randn(1, n, 2, 8, dtype=torch.float64) for n in (6, 9, 9))
    o, lse = mo.dense_attention(q, k, v, 0.5, False, (2, 1))
    for i in range(6):
        p = i + 3
        js = [j for j in range(9) if p - 2 <= j <= p + 1]
        s = torch.stack([(q[0, i] * k[0, j]).sum(-1) * 0.5 for j in js])  # [n, H]
        w = torch.softmax(s, 0)
        torch.testing.assert_close(o[0, i], torch.einsum("nh,nhd->hd", w, v[0, js]))
        torch.testing.assert_close(lse[0, :, i], torch.logsumexp(s, 0))
    o1, l1 = mo.dense_attention(q, k, v, 0.5, False, (-1, 0))
    o2, l2 = orc.dense_attention(q, k, v, 0.5, True)
    torch.testing.assert_close(o1, o2)
    torch.testing.assert_close(l1, l2)
    do = torch.randn_like(q)
    for a, b in zip(mo.dense_attention_bwd(q, k, v, do, 0.5, True, (-1, -1)), orc.dense_attention_bwd(q, k, v, do, 0.5, True)):
        torch.testing.assert_close(a, b)


def _check(ops, rank, world, layout, window, dg=(None, None), S_local=12):
    from burst_attn import burst_attn_func, burst_attn_func_striped
    from oracle import attention_oracle as orc
    func = burst_attn_func_striped if layout.startswith("striped") else burst_attn_func
    causal = layout in ("zigzag", "striped")
    shard = {"contiguous": "contiguous", "zigzag": "zigzag", "striped": "striped", "striped_nc": "striped"}[layout]
    torch.manual_seed(77)
    B, S, H, D = 1, S_local * world, 2, 8
    q, k, v, do = (torch.randn(B, S, H, D, dtype=torch.float64) for _ in range(4))
    o_ref, _, dq_ref, dk_ref, dv_ref = mo.dense_attention_bwd(q, k, v, do, 0.3, causal, window)
    sh = lambda t: orc.shard(t, rank, world, shard)  # noqa: E731
    ql, kl, vl = (sh(t).requires_grad_() for t in (q, k, v))
    o = func(ql, kl, vl, 0.3, "cuda", causal, False, False, None, list(dg), window)
    g = torch.autograd.grad(o, (ql, kl, vl), sh(do))
    tol = dict(rtol=1e-5, atol=1e-5)  # fp32 carried state / accumulators in the driver
    torch.testing.assert_close(o.detach(), sh(o_ref), **tol)
    for got, ref in zip(g, (dq_ref, dk_ref, dv_ref)):
        torch.testing.assert_close(got, sh(ref), **tol)


def _worker(rank, world, port, intra):
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from burst_attn import chunk_ops
    from oracle_ops import OracleOps
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        dg = double_group(rank, world, intra, False) if intra else (None, None)
        for layout in ("contiguous", "zigzag", "striped", "striped_nc"):
            for window in WINDOWS:
                _check(chunk_ops.get_ops(), rank, world, layout, window, dg)
        dist.barrier()
    finally:
        chunk_ops._set_ops_for_testing(None)
        dist.destroy_process_group()


@pytest.mark.parametrize("world,intra", [(2, 0), (4, 0), (4, 2)])
def test_windowed_ring_matches_dense(world, intra):
    """burst_attn_func (contiguous and zigzag shards) and burst_attn_func_striped (causal and not) on flat rings of 2
    and 4 ranks and the 2 x 2 hierarchical ring, against the windowed dense oracle."""
    spawn(_worker, world, (intra,), timeout=300)


def test_windowed_world1_and_l2_blocks(monkeypatch):
    """One rank, with and without L2 blocking of the rounds (BA_L2_BLOCK = 16: rows whose first visible key block is
    not block 0, and rows the last launch does not visit)."""
    from burst_attn import chunk_ops
    from oracle_ops import OracleOps
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        for blk in (None, "16"):
            if blk:
                monkeypatch.setenv("BA_L2_BLOCK", blk)
            for layout in ("contiguous", "zigzag", "striped", "striped_nc"):
                for window in WINDOWS + [(40, 3)]:
                    _check(chunk_ops.get_ops(), 0, 1, layout, window, S_local=70)
    finally:
        chunk_ops._set_ops_for_testing(None)


@pytest.mark.parametrize("blk", [None, "32"])
def test_flash_wrappers_window_cpu(monkeypatch, blk):
    from burst_attn import chunk_ops
    from burst_attn.flash_triton import flash_attn_func, flash_attn_kvpacked_func, flash_attn_qkvpacked_func
    from oracle_ops import OracleOps
    if blk:
        monkeypatch.setenv("BA_L2_BLOCK", blk)
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        torch.manual_seed(9)
        for sq, sk in [(70, 70), (50, 110), (110, 45)]:
            q, do = (torch.randn(2, sq, 4, 16, dtype=torch.float64) for _ in range(2))
            k, v = (torch.randn(2, sk, 2, 16, dtype=torch.float64) for _ in range(2))
            for causal in (False, True):
                for window in WINDOWS + [(30, 50)]:
                    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
                    o = flash_attn_func(qq, kk, vv, None, causal, 0.25, window)
                    g = torch.autograd.grad(o, (qq, kk, vv), do)
                    ke, ve = k.repeat_interleave(2, 2), v.repeat_interleave(2, 2)
                    o_ref, _, dq, dk, dv = mo.dense_attention_bwd(q, ke, ve, do, 0.25, causal, window)
                    tol = dict(rtol=1e-5, atol=1e-5)  # fp32 accumulators in the driver
                    torch.testing.assert_close(o.detach(), o_ref, **tol)
                    torch.testing.assert_close(g[0], dq, **tol)
                    torch.testing.assert_close(g[1], dk.unflatten(2, (2, 2)).sum(3), **tol)
                    torch.testing.assert_close(g[2], dv.unflatten(2, (2, 2)).sum(3), **tol)
                    kv = torch.stack([k, v], 2)
                    o2 = flash_attn_kvpacked_func(q, kv, None, causal, 0.25, window)
                    torch.testing.assert_close(o2, o_ref, **tol)
            if sq == sk:
                qkv = torch.stack([q, q, q], 2).requires_grad_()
                o3 = flash_attn_qkvpacked_func(qkv, None, True, 0.25, (9, -1))
                torch.testing.assert_close(o3.detach(), mo.dense_attention(q, q, q, 0.25, True, (9, -1))[0], rtol=1e-5,
                                           atol=1e-5)
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
        torch.manual_seed(1)
        q, k, v = (torch.randn(1, S_local * world, 1, 8, dtype=torch.float64) for _ in range(3))
        res = {}
        for name, func, causal, shard in (("contiguous", burst_attn_func, False, "contiguous"),
                                          ("zigzag", burst_attn_func, True, "zigzag"),
                                          ("striped", burst_attn_func_striped, True, "striped")):
            ql, kl, vl = (orc.shard(t, rank, world, shard).requires_grad_() for t in (q, k, v))
            for tag, extra in (("omitted", ()), ("minus1", ((-1, -1),)), ("half", ((S_local // 2, S_local // 2),))):
                ops.calls.clear()
                o = func(ql, kl, vl, None, "cuda", causal, False, False, None, [None, None], *extra)
                torch.autograd.grad(o.sum(), (ql, kl, vl))
                res[(name, tag)] = list(ops.calls)
        torch.save(res, os.path.join(outdir, f"calls{rank}.pt"))
        dist.barrier()
    finally:
        chunk_ops._set_ops_for_testing(None)
        dist.destroy_process_group()


def test_rounds_outside_the_window_launch_nothing(tmp_path):
    """W = 8, contiguous shards of S rows, window (S/2, S/2): only the shards of ranks i-1, i, i+1 launch a forward
    kernel on rank i, and only the bundles of those ranks a backward kernel.  window_size=(-1, -1) records exactly the
    calls of a call without the argument, in every layout."""
    world, S = 8, 8
    spawn(_calls_worker, world, (str(tmp_path),), timeout=300)
    for rank in range(world):
        res = torch.load(os.path.join(tmp_path, f"calls{rank}.pt"), weights_only=False)  # oracle_ops.Call records
        for name in ("contiguous", "zigzag", "striped"):
            assert res[(name, "omitted")] == res[(name, "minus1")], name
        calls = res[("contiguous", "half")]
        n_neighbours = len({j for j in (rank - 1, rank, rank + 1) if 0 <= j < world})
        fwd = [c for c in calls if c[0] == "fwd"]
        bwd = [c for c in calls if c[0] == "bwd"]
        assert len(fwd) == n_neighbours and len(bwd) == n_neighbours, (rank, fwd, bwd)
        for c in fwd + bwd:
            assert c[1][1] == S and c[2][1] == S  # whole shards: no L2 split at this size
        # the own shard: the window's two sides; the neighbours: one side each (the other masks nothing)
        assert sorted((c.causal, c.causal_offset, c.lower) for c in fwd) == sorted(
            [(True, S // 2, -S // 2)] + ([(False, 0, S // 2)] if rank > 0 else []) +
            ([(True, -S // 2, None)] if rank < world - 1 else []))


@pytest.mark.parametrize("window", [(-2, 0), (0, -5), (3,), "ab", (1.5, None)])
def test_bad_window_raises(window):
    from burst_attn import burst_attn_func, chunk_ops
    from burst_attn.flash_triton import flash_attn_func
    from oracle_ops import OracleOps
    chunk_ops._set_ops_for_testing(OracleOps())
    try:
        q = torch.randn(1, 8, 1, 8, dtype=torch.float64)
        with pytest.raises(ValueError, match="window_size"):
            burst_attn_func(q, q, q, None, "cuda", False, False, False, None, [None, None], window)
        with pytest.raises(ValueError, match="window_size"):
            flash_attn_func(q, q, q, None, False, None, window)
    finally:
        chunk_ops._set_ops_for_testing(None)


@pytest.fixture(scope="module")
def nat():
    from burst_attn import native
    if not os.path.exists(native.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return native


def test_band_entry_points_reject_bad_masks_and_bands(nat):
    L = nat.lib()
    assert L.ba_version() >= 202
    z4 = nat.ba_tensor4(None, 0, 0, 0)
    zr = nat.ba_rowstat(None, 0, 0)
    fwd = lambda mm, hi, lo: L.ba_fwd_chunk_band(z4, z4, z4, zr, z4, zr, z4, 1, 128, 128, 4, 2, 128, 1.0, mm, hi, lo,  # noqa
                                                 3, 1, None)
    bwd = lambda mm, hi, lo: L.ba_bwd_chunk_band(z4, z4, z4, z4, zr, zr, zr, z4, z4, z4, 1, 128, 128, 4, 2, 128, 1.0,  # noqa
                                                 mm, hi, lo, 0, 1, None)
    for call in (fwd, bwd):
        for mm in (4, 5, -1, 8):
            assert call(mm, 0, 0) != 0 and b"mask mode" in L.ba_last_error()
        assert call(3, 0, 1) != 0 and b"lower_offset" in L.ba_last_error()  # lower edge above the upper one
        for mm, hi, lo in ((3, 5, -5), (2, 0, 7), (3, 0, 0), (1, 0, 0), (0, 0, 0)):
            assert call(mm, hi, lo) != 0 and b"null" in L.ba_last_error()  # valid: reaches the operand check
        # causal offsets anywhere in the int range are valid; the band check compares the caller's values
        for mm, hi, lo in ((1, 2 ** 31 - 1, 0), (1, -2 ** 31, 0), (3, 2 ** 31 - 1, 2 ** 31 - 1), (3, -2 ** 31, -2 ** 31)):
            assert call(mm, hi, lo) != 0 and b"null" in L.ba_last_error()
        assert call(3, -2 ** 31, -2 ** 31 + 1) != 0 and b"-2147483648" in L.ba_last_error()
    # the existing entry points keep rejecting the lower-edge bit
    rc = L.ba_fwd_chunk_gqa(z4, z4, z4, zr, z4, zr, z4, 1, 128, 128, 4, 2, 128, 1.0, 2, 0, 3, 1, None)
    assert rc != 0 and b"mask mode" in L.ba_last_error()
    rc = L.ba_bwd_chunk_gqa(z4, z4, z4, z4, zr, zr, zr, z4, z4, z4, 1, 128, 128, 4, 2, 128, 1.0, 3, 0, 0, 1, None)
    assert rc != 0 and b"mask mode" in L.ba_last_error()


def test_band_symbols_bound(nat):
    L = ctypes.CDLL(nat.LIB_PATH)
    for name in ("ba_fwd_chunk_band", "ba_bwd_chunk_band"):
        assert hasattr(L, name) and name in nat.exported_symbols()


def test_band_mutants_rejected_by_the_model_cpu():
    """The 16-bit comparator rejects the faults of lowp_band.BAND_MUTANTS this case reaches (model against model, on
    the CPU); tests/test_lowp_band.py rejects every one of them on sweep cases of both dtypes."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import lowp_band
    import lowp_model as lm
    case = lm._case(257, [(257, None)], 64, torch.bfloat16, tag="band_mutant_cpu_")
    x = lm.make_inputs(case)
    x["masks"] = [("band", -70, 10)]
    args = (x["q"], x["ks"], x["vs"], x["do"], x["scale"], x["masks"], x["biases"])
    model, ref = lm.lowp_chain(*args), lm.oracle_chain(*args)
    absmax = [lm.scores_absmax(x["q"], x["ks"], x["scale"], x["masks"])]
    lm.assert_chain_within_model("band", model, ref, model, torch.bfloat16, absmax)
    vis = lm.visible(257, 257, x["masks"][0])
    live = [m for m in lowp_band.BAND_MUTANTS
            if any(not torch.equal(lm._vis_for(257, 257, x["masks"][0], None, m, side), vis)
                   for side in ("fwd", "bwd"))]
    assert {"band_lo_plus1_fwd", "band_lo_plus1_bwd", "band_i_end_short"} <= set(live), live
    for mutant in live:
        with pytest.raises(AssertionError):
            lm.assert_chain_within_model(mutant, lm.lowp_chain(*args, mutant=mutant), ref, model, torch.bfloat16,
                                         absmax)
