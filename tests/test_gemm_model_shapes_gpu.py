"""wgmma GEMM at the model's real shapes (cfg-2: B*T = 8000 encoder rows, 2816 decoder rows, neither a multiple of the
128-row tile) with every epilogue combination the model issues, against a torch fp32 contraction of the same 16-bit
operands.  Each CTA's tiles alternate between its two consumer warpgroups, so these shapes also cover CTAs whose last
tile belongs to either warpgroup and tiles whose rows or columns run past the tensor."""
import pytest
import torch

from neurst_b200 import lib as L

pytestmark = pytest.mark.gpu

F16 = torch.float16


def _rnd(g, *shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(F16)


def _rel(x, ref):
    return float((x.float() - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("M,N,K,b_mn", [(8000, 768, 256, True), (8000, 256, 256, False), (2816, 768, 256, True),
                                        (2816, 8192, 256, False), (8000, 256, 5120, True), (8000, 200, 256, False)])
def test_bias_16bit_out(M, N, K, b_mn):
    g = torch.Generator(device="cuda").manual_seed(11)
    A = _rnd(g, M, K)
    B = _rnd(g, K, N, scale=0.1) if b_mn else _rnd(g, N, K, scale=0.1)
    bias = torch.randn(N, device="cuda", generator=g)
    C = torch.zeros(M, N, device="cuda", dtype=F16)
    L.gemm(A, B, C, b_mn=b_mn, bias=bias)
    ref = A.float() @ (B.float() if b_mn else B.float().t()) + bias
    assert _rel(C, ref) < 2e-3


def test_bias_relu_dropout():
    """FFN1-shaped product with bias, ReLU and dropout: every element is 0 or the reference scaled by 1 / (1 - p)."""
    g = torch.Generator(device="cuda").manual_seed(12)
    M, N, K, p = 8000, 1024, 256, 0.1
    A, W = _rnd(g, M, K), _rnd(g, K, N, scale=0.1)
    bias = torch.randn(N, device="cuda", generator=g)
    C = torch.zeros(M, N, device="cuda", dtype=F16)
    L.gemm(A, W, C, b_mn=True, bias=bias, relu=True, dropout=(p, 1234, 7))
    ref = torch.relu(A.float() @ W.float() + bias)
    kept = C.float() != 0
    frac = float(((ref > 0) & ~kept).sum()) / float((ref > 0).sum())
    assert abs(frac - p) < 0.01, frac
    assert float((C.float() - ref / (1 - p)).abs()[kept].max()) < 2e-3 * float(ref.abs().max()) / (1 - p)


def test_mask_fp32_out():
    """Data gradient through a ReLU: dX = alpha (dY W^T) masked by the forward activation (> 0), fp32 output."""
    g = torch.Generator(device="cuda").manual_seed(13)
    M, N, K = 8000, 256, 2048
    dY, W = _rnd(g, M, K), _rnd(g, N, K, scale=0.05)
    msk = _rnd(g, M, N)
    C = torch.zeros(M, N, device="cuda")
    L.gemm(dY, W, C, mask_src=msk, alpha=0.5)
    ref = 0.5 * (dY.float() @ W.float().t()) * (msk.float() > 0)
    assert _rel(C, ref) < 1e-5


def test_bias_dropout_fp32_residual():
    """Attention output projection: x += dropout(Y W + b), the fp32 residual added last."""
    g = torch.Generator(device="cuda").manual_seed(14)
    M, N, K, p = 8000, 256, 256, 0.1
    Y, W = _rnd(g, M, K), _rnd(g, K, N, scale=0.1)
    bias = torch.randn(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g)
    C = torch.zeros(M, N, device="cuda")
    L.gemm(Y, W, C, b_mn=True, bias=bias, dropout=(p, 99, 3), residual=res)
    lin = Y.float() @ W.float() + bias
    kept = (C - res).abs() > 1e-6
    frac = 1.0 - float(kept.float().mean())
    assert abs(frac - p) < 0.01, frac
    err = (C - (res + lin / (1 - p))).abs()[kept]
    assert float(err.max()) < 1e-5 * float(lin.abs().max()) / (1 - p) + 1e-5


@pytest.mark.parametrize("splitk", [1, 0, 4])
@pytest.mark.parametrize("M,N,K", [(256, 768, 8000), (256, 2048, 2816), (2304, 256, 20000)])
def test_fp32_accumulate_and_split_k(M, N, K, splitk):
    """Weight gradient dW += X^T dY: MN-major operands, fp32 accumulate, split-K chosen by the library (0) or fixed."""
    g = torch.Generator(device="cuda").manual_seed(15)
    X, dY = _rnd(g, K, M), _rnd(g, K, N, scale=1e-2)
    dW = torch.randn(M, N, device="cuda", generator=g)
    ref = dW + X.float().t() @ dY.float()
    L.gemm(X, dY, dW, a_mn=True, b_mn=True, accumulate=True, splitk=splitk)
    assert _rel(dW, ref) < 1e-4


def test_batched_mn_major():
    """Unfused attention: P V per (batch, head) through 4-D maps, V read MN-major, 16-bit output."""
    g = torch.Generator(device="cuda").manual_seed(16)
    B, H, T, dh = 2, 4, 1000, 64
    P = _rnd(g, B, H, T, T, scale=0.05)
    V = _rnd(g, B, H, T, dh)
    O = torch.zeros(B, H, T, dh, device="cuda", dtype=F16)
    L.gemm(P, V, O, b_mn=True)
    ref = P.float() @ V.float()
    assert _rel(O, ref) < 2e-3
    # and the backward product dP = dO V^T with both operands K-major, batched, ragged T
    dO = _rnd(g, B, H, T, dh)
    dP = torch.zeros(B, H, T, T, device="cuda")
    L.gemm(dO, V, dP)
    ref = dO.float() @ V.float().transpose(-1, -2)
    assert _rel(dP, ref) < 1e-5
