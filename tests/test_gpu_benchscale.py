"""Parity AT THE SIZES THE BENCH TIMES (BASELINE.json configs C2/C3/C4 per-GPU shapes: S_local = 32768 and
65536, H = 32, d = 128, bf16), where a dense oracle over the whole problem does not finish:

* whole heads: O, dQ, dK and dV of two heads against the fp64 oracle within the 16-bit error model, computed in
  row blocks (``scale_model``), non-causal and causal;
* one whole head of dK / dV against fp32 dense attention with autograd on the GPU at S = 32768;
* the FA-style bf16 criterion of SURVEY.md 8(c): max-abs error against the fp64 oracle <= 2x the error
  of a plain bf16 PyTorch implementation of the same op (+ the hard cap of gpu_util.TOL).

Everything goes through the public API (so the L2-blocked sub-launch drivers run exactly as in bench.py).
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from burst_attn import burst_attn_func  # noqa: E402
from gpu_util import TOL  # noqa: E402
from burst_attn.burst_attn_interface import _l2_block  # noqa: E402
import scale_model as sm  # noqa: E402
from oracle import attention_oracle as orc  # noqa: E402

H, D = 32, 128


def _mk(S, seed, heads=H):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(1, S, heads, D, device="cuda", generator=g, dtype=torch.float32).to(torch.bfloat16)


def _run(q, k, v, do, causal):
    qq, kk, vv = (t.detach().requires_grad_() for t in (q, k, v))
    o = burst_attn_func(qq, kk, vv, None, "cuda", causal, True, False, None)
    dq, dk, dv = torch.autograd.grad(o, (qq, kk, vv), do)
    torch.cuda.synchronize()
    return o, dq, dk, dv


@pytest.mark.parametrize("S,causal", [(32768, False), (65536, False), (65536, True)])
def test_sampled_rows_at_bench_scale(S, causal):
    """Whole heads (the first and a seeded one) of O, dQ, dK and dV against the row-blocked fp64 oracle within the
    16-bit error model (``scale_model``): at this size a fixed tolerance misses a dropped key tile."""
    q, k, v, do = (_mk(S, s) for s in (101, 102, 103, 104))
    out = _run(q, k, v, do, causal)
    assert not any(torch.isnan(t).any().item() for t in out)
    h = int(torch.randint(1, H, (1,), generator=torch.Generator().manual_seed(S + int(causal))))
    blk = _l2_block()
    sm.check_api(f"benchscale_S{S}{'_causal' if causal else ''}", out, q, k, v, do,
                 ("causal_offset", 0) if causal else None, heads=[0, h], block=1024,
                 seams=(blk,) if S > blk + blk // 2 else ())


def test_one_head_dk_dv_against_fp32_dense_at_32768():
    """dK / dV of every key need every Q row: check one whole head against fp32 dense attention with autograd
    on the GPU (torch matmul + softmax in fp32, TF32 off), same 16-bit inputs."""
    S = 32768
    q, k, v, do = (_mk(S, s) for s in (111, 112, 113, 114))
    o, dq, dk, dv = _run(q, k, v, do, False)
    h = 5
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        qq, kk, vv = (t[0, :, h].float().clone().requires_grad_() for t in (q, k, v))
        # row blocks keep the fp32 score matrix at 4096 x 32768
        o_ref = torch.empty(S, D, device="cuda")
        for r0 in range(0, S, 4096):
            s = (qq[r0:r0 + 4096] @ kk.T) / math.sqrt(D)
            p = torch.softmax(s, dim=-1)
            (p @ vv).backward(do[0, r0:r0 + 4096, h].float())
            with torch.no_grad():
                o_ref[r0:r0 + 4096] = p @ vv
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    tol = TOL[torch.bfloat16]
    torch.testing.assert_close(o[0, :, h].float(), o_ref, **tol)
    torch.testing.assert_close(dq[0, :, h].float(), qq.grad, **tol)
    torch.testing.assert_close(dk[0, :, h].float(), kk.grad, **tol)
    torch.testing.assert_close(dv[0, :, h].float(), vv.grad, **tol)


def _plain_lowp_attention(q, k, v, do, causal):
    """A plain PyTorch implementation in the INPUT dtype (16-bit matmuls, fp32 softmax) with autograd -- the
    yardstick of the FA-style criterion."""
    qq, kk, vv = (t.detach().permute(0, 2, 1, 3).clone().requires_grad_() for t in (q, k, v))
    s = (qq @ kk.transpose(-1, -2)) * (D ** -0.5)
    if causal:
        S = s.shape[-1]
        s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool, device=s.device).tril(), float("-inf"))
    p = torch.softmax(s.float(), dim=-1).to(q.dtype)
    o = p @ vv
    g = torch.autograd.grad(o, (qq, kk, vv), do.permute(0, 2, 1, 3))
    return [t.permute(0, 2, 1, 3) for t in (o, *g)]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("causal", [False, True])
def test_error_not_worse_than_twice_plain_lowp_pytorch(dtype, causal):
    """max|ours - fp64| <= 2 * max|plain 16-bit PyTorch - fp64| + small floor, for O, dQ, dK, dV."""
    torch.manual_seed(3)
    b, s, n = 2, 1024, 8
    q, k, v, do = (torch.randn(b, s, n, D, device="cuda", dtype=dtype) for _ in range(4))
    ours = _run(q, k, v, do, causal)
    plain = _plain_lowp_attention(q, k, v, do, causal)
    o_ref, _, dq_ref, dk_ref, dv_ref = orc.dense_attention_bwd(q.cpu(), k.cpu(), v.cpu(), do.cpu(), None, causal)
    for name, a, p, r in zip(("o", "dq", "dk", "dv"), ours, plain, (o_ref, dq_ref, dk_ref, dv_ref)):
        e_ours = (a.double().cpu() - r).abs().max().item()
        e_plain = (p.double().cpu() - r).abs().max().item()
        assert e_ours <= 2 * e_plain + 1e-4, f"{name}: ours {e_ours:.3e} vs plain {dtype} PyTorch {e_plain:.3e}"
