"""Launch plans of the band planner, which plans every call, against summaries of the plans recorded from the commit
before it (``tests/golden/plans.json``, written by ``tests/golden/make_plans.py``), when causal and mask-free calls
still had a planner of their own; and the bottom-right causal call with at least 256 more queries than keys, whose first rows
that planner left unwritten once the keys were split over L2 blocks."""
import importlib.util
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _make_plans():
    spec = importlib.util.spec_from_file_location("make_plans", os.path.join(GOLDEN, "make_plans.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


MP = _make_plans()
with open(os.path.join(GOLDEN, "plans.json")) as _f:
    PARENT = json.load(_f)


def _check_duties(cfg, fwd):
    """The first launch starts the state only if it covers every row, the last launch writes its own rows in 16 bit
    and the casts cover exactly the other rows."""
    S = MP.rows_of(cfg)
    launches = [e for e in fwd if e[0] == "fwd"]
    for n, e in enumerate(launches):
        assert e[6] == (n == 0 and e[1] == [0, S]), (n, e)
        assert e[7] == (n == len(launches) - 1), (n, e)
        assert e[8] == (e[1] if e[7] else None), e
    q0, qn = launches[-1][1] if launches else (0, 0)
    casts = sorted(tuple(e[1]) for e in fwd if e[0] == "cast")
    assert casts == [c for c in ((0, q0), (q0 + qn, S - q0 - qn)) if c[1] > 0], casts


@pytest.mark.parametrize("cfg", MP.CONFIGS, ids=MP.key)
def test_launch_plan_matches_parent(cfg):
    """Without window or ALiBi: the same launches in the same order, and no more rows cast.  With one: exact merges
    and forward row starts rounded down to 256 only, so the same keys per row and round and never more launches."""
    sys.path.insert(0, os.path.join(ROOT, "burst-attention_b200"))
    plan = MP.record(cfg)
    _check_duties(cfg, plan["fwd"])
    old, new = PARENT[MP.key(cfg)], MP.summary(cfg, plan)
    if MP.plain(cfg):
        assert new[:2] == old[:2] and new[2] <= old[2], (new, old)
    else:
        assert new[0] == old[0] and new[1] <= old[1] and new[2] <= old[2], (new, old)


@pytest.mark.parametrize("packed", [False, True])
def test_causal_more_queries_than_keys_blocked_cpu(monkeypatch, packed):
    """flash_attn_func / flash_attn_kvpacked_func, causal (bottom-right), Sq - Sk >= 256 and K/V split over small L2
    blocks: the first key block's launch starts at a multiple of 256 rows > 0.  The rows before it see no key and
    must come back 0 with no gradient, with every scratch allocation starting as NaN."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from burst_attn import chunk_ops
    from burst_attn.flash_triton import flash_attn_func, flash_attn_kvpacked_func
    from oracle import attention_oracle as orc
    from oracle_ops import OracleOps
    monkeypatch.setenv("BA_L2_BLOCK", "16")
    torch.manual_seed(5)
    B, Sq, Sk, H, D = 1, 600, 40, 2, 16
    q, do = torch.randn(B, Sq, H, D, dtype=torch.float64), torch.randn(B, Sq, H, D, dtype=torch.float64)
    kv = torch.randn(B, Sk, 2, H, D, dtype=torch.float64)
    k, v = kv[:, :, 0].contiguous(), kv[:, :, 1].contiguous()
    n = Sq - Sk  # rows that see no key: 0 out, no gradient (the dense oracle has no softmax over no key)
    zero = torch.zeros(B, n, H, D, dtype=torch.float64)
    o_ref, _, dq, dk, dv = orc.dense_attention_bwd(q[:, n:], k, v, do[:, n:], None, True)
    o_ref, dq = torch.cat([zero, o_ref], 1), torch.cat([zero, dq], 1)
    empty, empty_like = torch.empty, torch.empty_like
    monkeypatch.setattr(torch, "empty", lambda *a, **kw: empty(*a, **kw).fill_(float("nan")))
    monkeypatch.setattr(torch, "empty_like", lambda *a, **kw: empty_like(*a, **kw).fill_(float("nan")))
    ops = OracleOps()
    ops.tile_head_dims = (D,)
    chunk_ops._set_ops_for_testing(ops)
    try:
        qq = q.clone().requires_grad_()
        if packed:
            pkv = kv.clone().requires_grad_()
            o = flash_attn_kvpacked_func(qq, pkv, None, True)
            gq, gkv = torch.autograd.grad(o, (qq, pkv), do)
            g = (gq, gkv[:, :, 0], gkv[:, :, 1])
        else:
            kk, vv = k.clone().requires_grad_(), v.clone().requires_grad_()
            o = flash_attn_func(qq, kk, vv, None, True)
            g = torch.autograd.grad(o, (qq, kk, vv), do)
    finally:
        chunk_ops._set_ops_for_testing(None)
    assert any(c[0] == "fwd" and c[1][1] < Sq for c in ops.calls)  # the forward was split over key blocks
    torch.testing.assert_close(o.detach(), o_ref, rtol=1e-5, atol=1e-5)
    for a, r in zip(g, (dq, dk, dv)):
        torch.testing.assert_close(a, r, rtol=1e-5, atol=1e-5)
