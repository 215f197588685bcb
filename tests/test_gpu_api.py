"""Public API (burst_attn_func / burst_attn_func_striped) on one GPU (W=1),
through autograd, against the oracle -- the reference's own test protocol
(test/test_burst.py:159-219: b=2, s=256*W, n=32, d=128, fp16, rtol=1e-3/atol=1e-2)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from burst_attn import burst_attn_func, burst_attn_func_striped  # noqa: E402
from gpu_util import TOL  # noqa: E402
from oracle import attention_oracle as orc  # noqa: E402


@pytest.mark.parametrize("func", [burst_attn_func, burst_attn_func_striped])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_reference_protocol_w1(func, causal, dtype):
    torch.manual_seed(0)
    b, s, n, d = 2, 256, 32, 128
    q, k, v, do = (torch.randn(b, s, n, d, device="cuda", dtype=dtype) for _ in range(4))
    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
    o = func(qq, kk, vv, None, "cuda", causal, True, False, None)
    dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
    o_ref, _, dq_ref, dk_ref, dv_ref = orc.dense_attention_bwd(q.cpu(), k.cpu(), v.cpu(), do.cpu(), None, causal)
    assert o.dtype == dtype and dq.dtype == dtype
    # gradients of a 16-bit O: the oracle differentiates the exact O, allow the dtype's tolerance
    torch.testing.assert_close(o.double().cpu(), o_ref, **TOL[dtype])
    for g, r in ((dv, dv_ref), (dk, dk_ref), (dq, dq_ref)):
        torch.testing.assert_close(g.double().cpu(), r, **TOL[torch.bfloat16] if dtype == torch.bfloat16 else
                                   dict(rtol=1e-3, atol=1e-2))


def test_normal_layout_flash_none():
    torch.manual_seed(1)
    q, k, v, do = (torch.randn(1, 4, 384, 128, device="cuda", dtype=torch.bfloat16) for _ in range(4))
    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
    o = burst_attn_func(qq, kk, vv, None, None, False)
    dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
    p = lambda t: t.permute(0, 2, 1, 3).cpu()
    o_ref, _, dq_ref, dk_ref, dv_ref = orc.dense_attention_bwd(p(q), p(k), p(v), p(do))
    torch.testing.assert_close(p(o).double(), o_ref, **TOL[torch.bfloat16])
    for g, r in ((dv, dv_ref), (dk, dk_ref), (dq, dq_ref)):
        torch.testing.assert_close(p(g).double(), r, **TOL[torch.bfloat16])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_flash_triton_noncausal(dtype):
    """flash="triton" (reference: inter_flash_attn_triton / _backward_triton, burst_utils.py:103-146) selects the
    same sm_90a tile kernels in the flash layout [B,S,N,H]; non-causal is the only mode the reference allows."""
    torch.manual_seed(2)
    b, s, n, d = 2, 384, 4, 128
    q, k, v, do = (torch.randn(b, s, n, d, device="cuda", dtype=dtype) for _ in range(4))
    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
    o = burst_attn_func(qq, kk, vv, None, "triton", False, True)
    dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
    o_ref, _, dq_ref, dk_ref, dv_ref = orc.dense_attention_bwd(q.cpu(), k.cpu(), v.cpu(), do.cpu())
    for g, r in ((o, o_ref), (dv, dv_ref), (dk, dk_ref), (dq, dq_ref)):
        torch.testing.assert_close(g.double().cpu(), r, **TOL[dtype])


def test_causal_requires_cuda_flash_like_reference():
    q = torch.randn(1, 128, 1, 128, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(AssertionError):
        burst_attn_func(q, q, q, None, "triton", True)


@pytest.mark.parametrize("causal", [False, True])
def test_packed_qkv_wrappers_match_oracle(causal):
    """flash_attn_func / _kvpacked_func / _qkvpacked_func (reference flash_triton.py:1013-1160): single-GPU entry
    points over the same tile kernels, operands read through strided views of the packed tensors."""
    from burst_attn.flash_triton import flash_attn_func, flash_attn_kvpacked_func, flash_attn_qkvpacked_func
    torch.manual_seed(4)
    dtype = torch.bfloat16
    b, s, n, d = 2, 384, 3, 128
    qkv = torch.randn(b, s, 3, n, d, device="cuda", dtype=dtype)
    do = torch.randn(b, s, n, d, device="cuda", dtype=dtype)
    q, k, v = (qkv[:, :, i].contiguous() for i in range(3))
    o_ref, _, dq_ref, dk_ref, dv_ref = orc.dense_attention_bwd(q.cpu(), k.cpu(), v.cpu(), do.cpu(), None, causal)

    p = qkv.clone().requires_grad_()
    o = flash_attn_qkvpacked_func(p, None, causal)
    (dqkv,) = torch.autograd.grad(o, (p,), do)
    torch.testing.assert_close(o.double().cpu(), o_ref, **TOL[dtype])
    for i, r in enumerate((dq_ref, dk_ref, dv_ref)):
        torch.testing.assert_close(dqkv[:, :, i].double().cpu(), r, **TOL[dtype])

    qq, kv = q.clone().requires_grad_(), qkv[:, :, 1:].clone().requires_grad_()
    o = flash_attn_kvpacked_func(qq, kv, None, causal)
    dq, dkv = torch.autograd.grad(o, (qq, kv), do)
    torch.testing.assert_close(dq.double().cpu(), dq_ref, **TOL[dtype])
    torch.testing.assert_close(dkv[:, :, 0].double().cpu(), dk_ref, **TOL[dtype])
    torch.testing.assert_close(dkv[:, :, 1].double().cpu(), dv_ref, **TOL[dtype])

    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
    o = flash_attn_func(qq, kk, vv, None, causal)
    torch.testing.assert_close(o.double().cpu(), o_ref, **TOL[dtype])
    with pytest.raises(NotImplementedError):
        flash_attn_func(qq, kk, vv, torch.zeros(1, n, s, s, device="cuda"), causal)


@pytest.mark.parametrize("D", [128, 64])
@pytest.mark.parametrize("causal", [False, True])
def test_key_vector_bias(monkeypatch, D, causal):
    """The "vector" bias of the reference's LAO tile (lao.py:102-105,155-173): scores = q k^T * scale + bias[b,h,key],
    incl. -inf entries (key-padding mask) and a batch-broadcast bias, through L2-blocked sub-launches."""
    from burst_attn.flash_triton import flash_attn_func
    monkeypatch.setenv("BA_L2_BLOCK", "256")
    torch.manual_seed(6)
    dtype = torch.bfloat16
    b, s, n = 2, 700, 3
    q, k, v, do = (torch.randn(b, s, n, D, device="cuda", dtype=dtype) for _ in range(4))
    for bias in (torch.randn(b, n, 1, s, device="cuda") * 2.0, torch.randn(1, n, 1, s, device="cuda")):
        bias[:, :, :, 5::7] = float("-inf")  # masked keys
        bias[:, 0, :, 1] = 30.0              # one dominant key
        qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
        o = flash_attn_func(qq, kk, vv, bias, causal)
        dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
        o_ref, _, dq_ref, dk_ref, dv_ref = orc.dense_attention_bwd(q.cpu(), k.cpu(), v.cpu(), do.cpu(), None, causal,
                                                                   bias=bias.cpu())
        if causal:  # row 0 sees only key 0 (finite bias); rows whose visible keys are all masked do not exist here
            assert not torch.isnan(o_ref).any()
        # a bias of a few units makes the softmax peaky (gradients of O(1..10)): the stated bf16 tolerance with a wider
        # absolute floor, plus the size-independent yardstick "not worse than 2x a plain bf16 PyTorch implementation"
        qp, kp, vp = (t.detach().permute(0, 2, 1, 3).clone().requires_grad_() for t in (q, k, v))
        sc = (qp @ kp.transpose(-1, -2)) * D ** -0.5 + bias
        if causal:
            sc = sc.masked_fill(~torch.ones(s, s, dtype=torch.bool, device="cuda").tril(), float("-inf"))
        op = torch.softmax(sc.float(), -1).to(dtype) @ vp
        plain = [t.permute(0, 2, 1, 3) for t in (op, *torch.autograd.grad(op, (qp, kp, vp), do.permute(0, 2, 1, 3)))]
        for got, ref, pl in zip((o, dq, dk, dv), (o_ref, dq_ref, dk_ref, dv_ref), plain):
            assert not torch.isnan(got).any()
            torch.testing.assert_close(got.double().cpu(), ref, rtol=1.6e-2, atol=6e-2)
            e_ours, e_plain = (got.double().cpu() - ref).abs().max().item(), (pl.double().cpu() - ref).abs().max().item()
            assert e_ours <= 2 * e_plain + 1e-3, (e_ours, e_plain)
        assert torch.all(dk[:, 5::7] == 0) and torch.all(dv[:, 5::7] == 0)  # masked keys get no gradient
