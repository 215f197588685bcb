"""sm_90a building blocks (TMA box/swizzle, wgmma descriptors, accumulator fragment,
register-A form of wgmma) checked one by one against torch on the GPU."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from gpu_util import selftest  # noqa: E402


@pytest.fixture(scope="module")
def ab():
    torch.manual_seed(0)
    a = torch.randn(128, 128, device="cuda").to(torch.bfloat16)
    b = torch.randn(128, 128, device="cuda").to(torch.bfloat16)
    return a, b


def test_tma_box_swizzle128(ab):
    a, b = ab
    raw = selftest(2, a, b).view(torch.bfloat16).view(128, 8, 8)  # [row][16B chunk][8 elems]
    exp = torch.empty_like(raw)
    src = a[:, :64].reshape(128, 8, 8)
    for r in range(128):
        for c in range(8):
            exp[r, c ^ (r % 8)] = src[r, c]
    assert torch.equal(raw, exp)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_ss_kmajor_gemm(ab, dtype):
    a, b = (t.to(dtype) for t in ab)
    out = selftest(0, a, b)
    torch.testing.assert_close(out, a.float() @ b.float().t(), rtol=1e-3, atol=1e-2)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_rs_gemm_p_in_registers(ab, dtype):
    a, b = (t.to(dtype) for t in ab)
    out = selftest(1, a, b)
    torch.testing.assert_close(out, a.float() @ b.float(), rtol=1e-3, atol=1e-2)


def test_ss_mnmajor_gemm(ab):
    a, b = ab
    out = selftest(3, a, b)
    torch.testing.assert_close(out, a.float().t() @ b.float(), rtol=1e-3, atol=1e-2)
