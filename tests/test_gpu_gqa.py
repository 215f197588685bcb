"""Grouped-query attention (K/V with Hkv < Hq heads) on one H100.

* chunk level, against the library's own MHA path on K/V repeated to Hq heads (same inputs): O and lse are bitwise
  equal (each query head does identical arithmetic), dQ is bitwise equal with deterministic=True (same per-key-block
  contributions in the same key-block order), dK / dV agree to fp32 summation order (the GQA kernel sums the G heads
  in registers, the reference sums G separate fp32 results);
* against the fp64 oracle on expanded K/V with gpu_util.TOL: chunk level (causal offsets, ragged S, key bias, both
  layouts) and the public API (fp16 / bf16, head dims 64, 128 and 96 (padded), G in {2, 4, Hq}, L2-blocked
  sub-launches, deterministic on and off);
* the reference protocol shapes at W = 1 with Hq = 32, Hkv = 8; the single-GPU flash_attn wrappers; host-resident
  operands; and one sampled case at S = 65536 (Hq = 32, Hkv = 8), above the L2-block threshold.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from burst_attn import burst_attn_func, burst_attn_func_striped  # noqa: E402
from burst_attn.chunk_ops import NativeOps  # noqa: E402
from gpu_util import TOL  # noqa: E402
import scale_model as sm  # noqa: E402
from oracle import attention_oracle as orc  # noqa: E402

HQ = 8


def _rand(shape, dtype, seed, device="cuda"):
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randn(*shape, device=device, generator=g, dtype=torch.float32).to(dtype)


def _expand(t, G, hd):
    return t.repeat_interleave(G, dim=hd)


def _group_sum(t, G, hd):
    return t.unflatten(hd, (t.shape[hd] // G, G)).sum(hd + 1)


def _chunk_fwd_bwd(q, k, v, do, scale, causal, off, bias, det, seq_dim):
    """One forward (FIRST|LAST) and one backward chunk call through NativeOps; fp32 gradient accumulators."""
    ops = NativeOps()
    B, Sq, H = q.shape[0], q.shape[seq_dim], q.shape[3 - seq_dim]
    out = torch.empty_like(q)
    lse = torch.empty(B, H, Sq, device="cuda", dtype=torch.float32)
    kw = {} if bias is None else {"bias": bias}
    ops.fwd_chunk(q, k, v, None, lse, out, scale, causal, off, True, True, seq_dim, **kw)
    delta = torch.empty(B, H, Sq, device="cuda", dtype=torch.float32)
    ops.delta(out, do, delta, seq_dim)
    acc = [torch.zeros(t.shape, device="cuda", dtype=torch.float32) for t in (q, k, v)]
    ops.bwd_chunk(do, q, k, v, delta, lse, *acc, scale, causal, off, seq_dim, deterministic=det, **kw)
    torch.cuda.synchronize()
    return out, lse, acc


# (Sq, Sk, causal, causal offset, key bias, layout, deterministic)
_CHUNK_CASES = [
    (384, 384, False, 0, False, 1, False),
    (300, 333, True, 33, True, 2, True),   # ragged, bottom-right causal, bias, normal layout
    (256, 512, True, 256, False, 1, True),
    (200, 333, False, 0, True, 1, False),
]


@pytest.mark.parametrize("hkv", [4, 2, 1])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_chunk_gqa_matches_mha_on_expanded_kv_and_oracle(dtype, D, hkv):
    G = HQ // hkv
    scale = D ** -0.5
    for n, (Sq, Sk, causal, off, with_bias, seq_dim, det) in enumerate(_CHUNK_CASES):
        hd = 3 - seq_dim
        B = 2

        def mk(S, H, seed):
            t = _rand((B, S, H, D), dtype, seed)
            return t if seq_dim == 1 else t.permute(0, 2, 1, 3).contiguous()

        q, do = mk(Sq, HQ, 10 * n + 1), mk(Sq, HQ, 10 * n + 2)
        k, v = mk(Sk, hkv, 10 * n + 3), mk(Sk, hkv, 10 * n + 4)
        bias = _rand((1, HQ, Sk), torch.float32, 10 * n + 5).expand(B, HQ, Sk) if with_bias else None
        msg = f"case {n}: Sq={Sq} Sk={Sk} causal={causal} off={off} bias={with_bias} seq_dim={seq_dim} det={det}"

        o, lse, (dq, dk, dv) = _chunk_fwd_bwd(q, k, v, do, scale, causal, off, bias, det, seq_dim)
        ke, ve = _expand(k, G, hd).contiguous(), _expand(v, G, hd).contiguous()
        o_m, lse_m, (dq_m, dk_m, dv_m) = _chunk_fwd_bwd(q, ke, ve, do, scale, causal, off, bias, det, seq_dim)
        assert dk.shape == k.shape and dv.shape == v.shape
        assert torch.equal(o, o_m), msg
        assert torch.equal(lse, lse_m), msg
        if det:
            assert torch.equal(dq, dq_m), msg
        else:
            torch.testing.assert_close(dq, dq_m, rtol=0, atol=1e-5 * dq_m.abs().max().item(), msg=msg)
        for got, ref in ((dk, _group_sum(dk_m, G, hd)), (dv, _group_sum(dv_m, G, hd))):
            torch.testing.assert_close(got, ref, rtol=0, atol=1e-5 * ref.abs().max().item(), msg=msg)

        # fp64 oracle on expanded K/V ([B, S, H, D] layout)
        lay = (lambda t: t) if seq_dim == 1 else (lambda t: t.permute(0, 2, 1, 3))
        qc, kc, vc, doc = (lay(t).cpu() for t in (q, ke, ve, do))
        mode = ("causal_offset", off) if causal else "none"
        bc = None if bias is None else bias.cpu()
        o_ref, lse_ref = orc.chunk_forward(qc, kc, vc, None, None, scale, mode, key_bias=bc)
        torch.testing.assert_close(lay(o).double().cpu(), o_ref, **TOL[dtype], msg=msg)
        delta_ref = orc.compute_delta(lay(o).cpu(), doc)
        rdq, rdk, rdv = orc.chunk_backward(doc, qc, kc, vc, delta_ref, lse_ref, scale, mode, key_bias=bc)
        torch.testing.assert_close(lay(dq).double().cpu(), rdq, **TOL[dtype], msg=msg)
        torch.testing.assert_close(lay(dk).double().cpu(), _group_sum(rdk, G, 2), **TOL[dtype], msg=msg)
        torch.testing.assert_close(lay(dv).double().cpu(), _group_sum(rdv, G, 2), **TOL[dtype], msg=msg)


def _api_vs_oracle(func, q, k, v, do, causal, seq_dim, det, tol):
    """Public API call (autograd) against the fp64 oracle on K/V expanded to Hq heads."""
    G = q.shape[3 - seq_dim] // k.shape[3 - seq_dim]
    flash = "cuda" if seq_dim == 1 else None
    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
    o = func(qq, kk, vv, None, flash, causal, True, det, None)
    dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
    torch.cuda.synchronize()
    assert dq.shape == q.shape and dk.shape == k.shape and dv.shape == v.shape
    assert o.dtype == q.dtype and dk.dtype == k.dtype
    lay = (lambda t: t) if seq_dim == 1 else (lambda t: t.permute(0, 2, 1, 3))
    qc, kc, vc, doc = (lay(t).cpu().double() for t in (q, k, v, do))
    qr, kr, vr = (t.clone().requires_grad_() for t in (qc, kc, vc))
    # (at W = 1 the striped driver owns every token: its mask is plain causal as well)
    o_ref, _ =orc.dense_attention(qr, _expand(kr, G, 2), _expand(vr, G, 2), None, causal)
    refs = torch.autograd.grad(o_ref, (qr, kr, vr), doc)
    torch.testing.assert_close(lay(o).double().cpu(), o_ref.detach(), **tol)
    for got, ref in zip((dq, dk, dv), refs):
        torch.testing.assert_close(lay(got).double().cpu(), ref, **tol)


@pytest.mark.parametrize("hkv", [4, 2, 1])
@pytest.mark.parametrize("D", [64, 128, 96])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_public_api_gqa_l2_blocked_against_oracle(monkeypatch, dtype, D, hkv):
    """BA_L2_BLOCK=256 at S=600: every round is split into sub-launches (carried state forward, row blocks
    backward, causal offsets of sub-views), with K/V of Hkv heads."""
    monkeypatch.setenv("BA_L2_BLOCK", "256")
    S, B = 600, 1
    cases = [(burst_attn_func, False, 1, False), (burst_attn_func, True, 1, True),
             (burst_attn_func_striped, True, 1, False), (burst_attn_func, False, 2, True)]
    for n, (func, causal, seq_dim, det) in enumerate(cases):
        q, do = (_rand((B, S, HQ, D), dtype, 100 * n + s) for s in (1, 2))
        k, v = (_rand((B, S, hkv, D), dtype, 100 * n + s) for s in (3, 4))
        if seq_dim == 2:
            q, k, v, do = (t.permute(0, 2, 1, 3).contiguous() for t in (q, k, v, do))
        _api_vs_oracle(func, q, k, v, do, causal, seq_dim, det, TOL[dtype])


@pytest.mark.parametrize("func", [burst_attn_func, burst_attn_func_striped])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_reference_protocol_w1_gqa(func, causal, dtype):
    """The reference's protocol shapes (b=2, s=256, d=128) with Hq=32 query heads and Hkv=8 K/V heads."""
    torch.manual_seed(0)
    b, s, d = 2, 256, 128
    q, do = (torch.randn(b, s, 32, d, device="cuda", dtype=dtype) for _ in range(2))
    k, v = (torch.randn(b, s, 8, d, device="cuda", dtype=dtype) for _ in range(2))
    _api_vs_oracle(func, q, k, v, do, causal, 1, False, TOL[dtype])


@pytest.mark.parametrize("causal", [False, True])
def test_flash_wrappers_gqa(monkeypatch, causal):
    """flash_attn_func / flash_attn_kvpacked_func with nheads_k | nheads, per-key bias per query head,
    Sq != Sk (bottom-right causal), L2-blocked; gradients have the shapes of the inputs."""
    from burst_attn.flash_triton import flash_attn_func, flash_attn_kvpacked_func
    monkeypatch.setenv("BA_L2_BLOCK", "256")
    dtype, D, hkv, Sq, Sk = torch.bfloat16, 128, 2, 300, 700
    G = HQ // hkv
    q, do = (_rand((2, Sq, HQ, D), dtype, s) for s in (41, 42))
    kv = _rand((2, Sk, 2, hkv, D), dtype, 43)
    bias = _rand((1, HQ, 1, Sk), torch.float32, 44)
    bias[..., 5::9] = float("-inf")
    k, v = kv[:, :, 0], kv[:, :, 1]
    qr, kr, vr = (t.cpu().double().requires_grad_() for t in (q, k, v))
    o_ref, _ = orc.dense_attention(qr, _expand(kr, G, 2), _expand(vr, G, 2), None, causal, bias=bias.cpu())
    refs = torch.autograd.grad(o_ref, (qr, kr, vr), do.cpu().double())
    tol = TOL[dtype]

    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
    o = flash_attn_func(qq, kk, vv, bias, causal)
    g = torch.autograd.grad(o, (qq, kk, vv), do)
    torch.testing.assert_close(o.double().cpu(), o_ref.detach(), **tol)
    for got, ref, inp in zip(g, refs, (qq, kk, vv)):
        assert got.shape == inp.shape
        torch.testing.assert_close(got.double().cpu(), ref, **tol)

    qq, pkv = q.clone().requires_grad_(), kv.clone().requires_grad_()
    o = flash_attn_kvpacked_func(qq, pkv, bias, causal)
    gq, gkv = torch.autograd.grad(o, (qq, pkv), do)
    assert gkv.shape == pkv.shape
    torch.testing.assert_close(gq.double().cpu(), refs[0], **tol)
    torch.testing.assert_close(gkv[:, :, 0].double().cpu(), refs[1], **tol)
    torch.testing.assert_close(gkv[:, :, 1].double().cpu(), refs[2], **tol)


@pytest.mark.parametrize("causal", [False, True])
def test_host_resident_gqa(monkeypatch, causal):
    """Pinned host operands with K/V of Hkv heads: streamed up and down under the L2-blocked sub-launches."""
    monkeypatch.setenv("BA_L2_BLOCK", "256")
    dtype, S, hkv = torch.bfloat16, 1024 + 100, 2
    torch.manual_seed(0)
    q, do = (torch.randn(1, S, HQ, 128).to(dtype).pin_memory() for _ in range(2))
    k, v = (torch.randn(1, S, hkv, 128).to(dtype).pin_memory() for _ in range(2))
    qq, kk, vv = (t.clone().pin_memory().requires_grad_() for t in (q, k, v))
    o = burst_attn_func(qq, kk, vv, None, "cuda", causal)
    dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
    torch.cuda.synchronize()
    assert all(t.device.type == "cpu" and t.dtype == dtype for t in (o, dq, dk, dv))
    assert dk.shape == k.shape and dv.shape == v.shape
    G = HQ // hkv
    qr, kr, vr = (t.double().requires_grad_() for t in (q, k, v))
    o_ref, _ = orc.dense_attention(qr, _expand(kr, G, 2), _expand(vr, G, 2), None, causal)
    refs = torch.autograd.grad(o_ref, (qr, kr, vr), do.double())
    torch.testing.assert_close(o.double(), o_ref.detach(), **TOL[dtype])
    for got, ref in zip((dq, dk, dv), refs):
        torch.testing.assert_close(got.double(), ref, **TOL[dtype])


@pytest.mark.parametrize("causal", [False, True])
def test_sampled_rows_gqa_at_65536(causal):
    """S = 65536, Hq = 32, Hkv = 8, bf16 through the public API (L2-blocked sub-launches, as in bench.py): one whole
    K/V group -- O and dQ of its G query heads, dK and dV of its K/V head -- against the row-blocked fp64 oracle within
    the 16-bit error model (``scale_model``)."""
    S, H, HKV, D = 65536, 32, 8, 128
    G = H // HKV
    q, do = (_rand((1, S, H, D), torch.bfloat16, s) for s in (201, 202))
    k, v = (_rand((1, S, HKV, D), torch.bfloat16, s) for s in (203, 204))
    qq, kk, vv = (t.detach().requires_grad_() for t in (q, k, v))
    o = burst_attn_func(qq, kk, vv, None, "cuda", causal, True, False, None)
    dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
    torch.cuda.synchronize()
    assert not any(torch.isnan(t).any().item() for t in (o, dq, dk, dv))
    assert dk.shape == k.shape
    hk = 3
    sm.check_api(f"gqa_S{S}{'_causal' if causal else ''}", (o.detach(), dq, dk, dv), q, k, v, do,
                 ("causal_offset", 0) if causal else None, heads=range(hk * G, hk * G + G), block=1024,
                 seams=(32768,))
