"""The code path the headline bench runs at N=1/2/4: every ring round goes through the L2-blocked
sub-launches of the launch planner ``_fwd_band_launches`` / ``_bwd_band_launches`` (burst_attn_interface.py) -- K/V
blocks with carried state forward, Q-row blocks backward, views trimmed to the rows / keys each block sees.
Here with the NATIVE kernels (tests/test_ring_gloo.py covers the same drivers with oracle ops on CPU):

* public API, W=1, tiny ``BA_L2_BLOCK`` so that S ~ 1-2k already splits into many sub-launches,
  non-causal / causal (zigzag r=1) / striped, fwd + bwd against the fp64 oracle;
* ``ba_fwd_chunk`` / ``ba_bwd_chunk`` directly with the causal offsets those views produce
  (negative non-multiples of the tile, large positive, Sq != Sk), incl. the state-passthrough case
  of a Q tile pair whose first tile sees nothing while the second does.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from burst_attn import burst_attn_func, burst_attn_func_striped  # noqa: E402
from burst_attn.chunk_ops import NativeOps  # noqa: E402
from gpu_util import TOL  # noqa: E402
from oracle import attention_oracle as orc  # noqa: E402

SCALE = 128 ** -0.5


def _mk(shape, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, device="cuda", generator=g).to(dtype)


@pytest.mark.parametrize("blk", [256, 512])
@pytest.mark.parametrize("S", [1024, 1536 + 200])
@pytest.mark.parametrize("mode", ["none", "causal", "striped"])
def test_public_api_l2_blocked_w1(monkeypatch, blk, S, mode):
    monkeypatch.setenv("BA_L2_BLOCK", str(blk))
    dtype = torch.bfloat16
    b, n = 1, 3
    q, k, v, do = (_mk((b, S, n, 128), dtype, s) for s in (1, 2, 3, 4))
    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
    func = burst_attn_func_striped if mode == "striped" else burst_attn_func
    causal = mode != "none"
    from burst_attn import chunk_ops  # count launches to prove the blocked path ran
    n0 = chunk_ops.get_ops().launches
    o = func(qq, kk, vv, None, "cuda", causal, True, False, None)
    dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
    torch.cuda.synchronize()
    assert chunk_ops.get_ops().launches - n0 >= 2 * ((S + blk - 1) // blk), "L2-blocked sub-launch path did not run"
    o_ref, _, dq_ref, dk_ref, dv_ref = orc.dense_attention_bwd(q.cpu(), k.cpu(), v.cpu(), do.cpu(), None, causal)
    torch.testing.assert_close(o.double().cpu(), o_ref, **TOL[dtype])
    for g, r in ((dv, dv_ref), (dk, dk_ref), (dq, dq_ref)):
        torch.testing.assert_close(g.double().cpu(), r, **TOL[dtype])


def test_public_api_l2_blocked_fp16_reference_tolerance(monkeypatch):
    """Same path at the reference's own fp16 tolerance (test/checker.py:6-10)."""
    monkeypatch.setenv("BA_L2_BLOCK", "256")
    dtype = torch.float16
    q, k, v, do = (_mk((2, 1280, 2, 128), dtype, s) for s in (5, 6, 7, 8))
    for causal in (False, True):
        qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
        o = burst_attn_func(qq, kk, vv, None, "cuda", causal)
        dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
        o_ref, _, dq_ref, dk_ref, dv_ref = orc.dense_attention_bwd(q.cpu(), k.cpu(), v.cpu(), do.cpu(), None, causal)
        for g, r in ((o, o_ref), (dv, dv_ref), (dk, dk_ref), (dq, dq_ref)):
            torch.testing.assert_close(g.double().cpu(), r, **TOL[dtype])


# ---- direct kernel calls with the offsets the views produce ------------------------------------
OFFSETS = [(-200, 512, 512), (-129, 640, 384), (-1, 300, 300), (384, 256, 1000), (1000, 384, 640), (-255, 512, 256),
           (100, 200, 333), (-256, 768, 512)]


@pytest.mark.parametrize("off,Sq,Sk", OFFSETS)
@pytest.mark.parametrize("first", [True, False])
def test_fwd_chunk_causal_offsets(off, Sq, Sk, first):
    """key b visible to row a iff b <= a + off.  Rows with a + off < 0 see nothing: with carried
    state they must pass it through unchanged, on a first call they produce (O=0, lse=-inf)."""
    dtype = torch.bfloat16
    B, H = 1, 2
    q, k, v = _mk((B, Sq, H, 128), dtype, 11), _mk((B, Sk, H, 128), dtype, 12), _mk((B, Sk, H, 128), dtype, 13)
    ops = NativeOps()
    lse = torch.empty(B, H, Sq, device="cuda", dtype=torch.float32)
    o_acc = torch.empty(B, Sq, H, 128, device="cuda", dtype=torch.float32)
    o0 = l0 = None
    if not first:  # a previous non-causal chunk provides the carried state
        k0, v0 = _mk((B, 256, H, 128), dtype, 14), _mk((B, 256, H, 128), dtype, 15)
        ops.fwd_chunk(q, k0, v0, o_acc, lse, None, SCALE, False, 0, True, False, 1)
        o0, l0 = orc.chunk_forward(q.cpu(), k0.cpu(), v0.cpu(), None, None, SCALE, "none")
    ops.fwd_chunk(q, k, v, o_acc, lse, None, SCALE, True, off, first, False, 1)
    torch.cuda.synchronize()
    o_ref, l_ref = orc.chunk_forward(q.cpu(), k.cpu(), v.cpu(), o0, l0, SCALE, ("causal_offset", off))
    dead = torch.isinf(l_ref)  # [B,H,Sq]
    got_l = lse.double().cpu()
    assert torch.equal(torch.isinf(got_l) & (got_l < 0), dead)
    torch.testing.assert_close(got_l[~dead], l_ref[~dead], rtol=1e-3, atol=2e-3)
    alive = (~dead).permute(0, 2, 1).unsqueeze(-1).expand_as(o_ref)
    torch.testing.assert_close(o_acc.double().cpu()[alive], o_ref[alive], **TOL[dtype])


@pytest.mark.parametrize("off,Sq,Sk", OFFSETS)
def test_bwd_chunk_causal_offsets(off, Sq, Sk):
    dtype = torch.bfloat16
    B, H = 1, 2
    q, do = _mk((B, Sq, H, 128), dtype, 21), _mk((B, Sq, H, 128), dtype, 22)
    k, v = _mk((B, Sk, H, 128), dtype, 23), _mk((B, Sk, H, 128), dtype, 24)
    mode = ("causal_offset", off)
    o_ref, lse_ref = orc.chunk_forward(q.cpu(), k.cpu(), v.cpu(), None, None, SCALE, mode)
    dead = torch.isinf(lse_ref)
    ops = NativeOps()
    o_dev = o_ref.to(dtype).cuda()
    delta = torch.empty(B, H, Sq, device="cuda", dtype=torch.float32)
    ops.delta(o_dev, do, delta, 1)
    acc = [torch.zeros(t.shape, device="cuda", dtype=torch.float32) for t in (q, k, v)]
    ops.bwd_chunk(do, q, k, v, delta, lse_ref.float().cuda().contiguous(), acc[0], acc[1], acc[2], SCALE, True, off, 1)
    torch.cuda.synchronize()
    delta_ref = orc.compute_delta(o_dev.cpu(), do.cpu())
    lse_for_ref = torch.where(dead, torch.full_like(lse_ref, 1e30), lse_ref)  # dead rows: p = 0
    ref = orc.chunk_backward(do.cpu(), q.cpu(), k.cpu(), v.cpu(), delta_ref, lse_for_ref, SCALE, mode)
    for g, r in zip(acc, ref):
        assert not torch.isnan(g).any()
        torch.testing.assert_close(g.double().cpu(), r, **TOL[dtype])


def test_blocked_equals_unblocked_bitwise_forward_lse(monkeypatch):
    """The blocked forward is the same arithmetic as a ring of K/V chunks: lse of the blocked run must
    agree with the single-launch run to fp32 round-off, O to the 16-bit output precision."""
    dtype = torch.bfloat16
    q, k, v = (_mk((1, 2048, 2, 128), dtype, s) for s in (31, 32, 33))
    outs = []
    for blk in ("100000", "512"):
        monkeypatch.setenv("BA_L2_BLOCK", blk)
        with torch.no_grad():
            outs.append(burst_attn_func(q, k, v, None, "cuda", True))
    torch.cuda.synchronize()
    torch.testing.assert_close(outs[0].float(), outs[1].float(), rtol=1e-2, atol=1e-2)
