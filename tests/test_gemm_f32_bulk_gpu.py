"""GEMMs with fp32 C that leave through the tensor map (tc_gemm_f32_kernel): bulk stores of alpha * acc (+ bias), or bulk
reduce-adds for split-K and accumulate, against a torch fp32 contraction of the same 16-bit operands.  The shapes are the
model's (the logits GEMM 2816 x 8192 x 256, the encoder's 8000-row products) plus the tensor map's edges: rows past M
(8000 and 2816 are not multiples of 128), columns past N (N = 200 ends inside a 32-column box, 64 inside a 128-column tile),
and C as a column slice of a wider tensor (ldc != N), where the columns beside the slice must stay untouched."""
import pytest
import torch

from neurst_b200 import lib as L

pytestmark = pytest.mark.gpu

F16 = torch.float16


def _rnd(g, *shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(F16)


def _rel(x, ref):
    return float((x.float() - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("M,N,K,b_mn,alpha", [(2816, 8192, 256, False, 1.0), (8000, 256, 768, True, 1.0), (8000, 200, 256, False, 0.5),
                                              (1000, 64, 512, True, 1.0)])
@pytest.mark.parametrize("with_bias", [True, False])
def test_fp32_store(M, N, K, b_mn, alpha, with_bias):
    g = torch.Generator(device="cuda").manual_seed(21)
    A = _rnd(g, M, K)
    B = _rnd(g, K, N, scale=0.1) if b_mn else _rnd(g, N, K, scale=0.1)
    bias = torch.randn(N, device="cuda", generator=g) if with_bias else None
    C = torch.full((M, N), float("nan"), device="cuda")
    L.gemm(A, B, C, b_mn=b_mn, bias=bias, alpha=alpha)
    ref = alpha * (A.float() @ (B.float() if b_mn else B.float().t()))
    if with_bias:
        ref = ref + bias
    assert torch.isfinite(C).all()
    assert _rel(C, ref) < 1e-5


@pytest.mark.parametrize("splitk", [1, 0, 3])
@pytest.mark.parametrize("M,N,K", [(8000, 256, 512), (2816, 200, 8192)])
def test_fp32_accumulate_into_slice(M, N, K, splitk):
    """C += alpha A B^T into columns 8 .. 8 + N of a pre-filled [M, N + 24] tensor (ldc = N + 24)."""
    g = torch.Generator(device="cuda").manual_seed(22)
    A, B = _rnd(g, M, K), _rnd(g, N, K, scale=0.05)
    W = torch.randn(M, N + 24, device="cuda", generator=g)
    before = W.clone()
    C = W[:, 8:8 + N]
    L.gemm(A, B, C, accumulate=True, splitk=splitk, alpha=0.5)
    ref = before[:, 8:8 + N] + 0.5 * (A.float() @ B.float().t())
    assert _rel(C, ref) < 1e-4                     # fp32 sums over K = 8192 without split-K: test_gemm_model_shapes_gpu's bound
    assert torch.equal(W[:, :8], before[:, :8]) and torch.equal(W[:, 8 + N:], before[:, 8 + N:])


def test_fp32_store_slice_leaves_neighbours():
    """A stored C that is a column slice: the bulk stores are clipped at N and write nothing beside the slice."""
    g = torch.Generator(device="cuda").manual_seed(23)
    M, N, K = 2816, 200, 256
    A, B = _rnd(g, M, K), _rnd(g, N, K, scale=0.1)
    bias = torch.randn(N, device="cuda", generator=g)
    W = torch.randn(M, N + 56, device="cuda", generator=g)
    before = W.clone()
    C = W[:, 16:16 + N]
    L.gemm(A, B, C, bias=bias)
    assert _rel(C, A.float() @ B.float().t() + bias) < 1e-5
    assert torch.equal(W[:, :16], before[:, :16]) and torch.equal(W[:, 16 + N:], before[:, 16 + N:])
