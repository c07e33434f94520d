"""The tensor-core GEMM's short epilogue loop (16-bit C, alpha and optional bias only) against an fp32 torch product,
with a partial last row tile, and with an odd N (no paired stores), which keeps the general loop."""
import pytest
import torch

from neurst_b200 import lib as L

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", [(300, 256, 256), (1000, 129, 192)])
@pytest.mark.parametrize("with_bias", [False, True])
def test_plain_16bit_epilogue(dt, M, N, K, with_bias):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(M, K, device="cuda", generator=g).to(dt)
    B = torch.randn(N, K, device="cuda", generator=g).to(dt)
    bias = torch.randn(N, device="cuda", generator=g) if with_bias else None
    C = torch.full((M, N), float("nan"), device="cuda").to(dt)
    kw = dict(alpha=0.5)
    if with_bias:
        kw["bias"] = bias
    L.gemm(A, B, C, **kw)
    ref = 0.5 * (A.float() @ B.float().t())
    if with_bias:
        ref = ref + bias
    torch.cuda.synchronize()
    tol = 2e-2 if dt == torch.float16 else 1e-1
    assert torch.isfinite(C.float()).all()
    assert float((C.float() - ref).abs().max()) < tol * float(ref.abs().max())
