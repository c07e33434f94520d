"""wgmma GEMM through the C ABI (b200st_gemm) vs a torch fp32 contraction of the same 16-bit-rounded operands:
K-major / MN-major operands, bf16 and fp16 operand formats, every output type, split-K accumulate, fused epilogues.
Mixed A/B formats are refused by the library (they fault on the hardware)."""
import pytest
import torch

from neurst_b200 import lib as L

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}


def _ref(A, B, a_mn, b_mn):
    a = A.float().transpose(-1, -2) if a_mn else A.float()
    b = B.float() if b_mn else B.float().transpose(-1, -2)
    return a @ b


@pytest.mark.parametrize("adt,bdt", [("bf16", "bf16"), ("f16", "f16")])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("cdt", ["f32", "bf16", "f16"])
def test_operand_formats(adt, bdt, a_mn, b_mn, cdt):
    g = torch.Generator(device="cuda").manual_seed(1)
    M, N, K = 304, 192, 136          # ragged tiles; MN-major rows must be 16-byte multiples for TMA (M % 8 == 0)
    A = torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g).to(DT[adt])
    B = torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g).to(DT[bdt])
    C = torch.zeros(M, N, device="cuda", dtype=DT[cdt])
    L.gemm(A, B, C, a_mn=a_mn, b_mn=b_mn)
    ref = _ref(A, B, a_mn, b_mn)
    tol = 2e-5 if cdt == "f32" else (8e-3 if cdt == "bf16" else 1e-3)
    err = float((C.float() - ref).abs().max() / ref.abs().max())
    assert err < tol, err


def test_mixed_operand_formats_are_refused():
    A = torch.randn(128, 64, device="cuda").to(torch.float16)
    B = torch.randn(64, 64, device="cuda").to(torch.bfloat16)
    C = torch.zeros(128, 64, device="cuda")
    with pytest.raises(L.B200STError):
        L.gemm(A, B, C)


def test_f16_wgrad_splitk_accumulate():
    """dW += X^T dY (both fp16, loss-scaled gradient), split-K reduce-add into the fp32 gradient arena."""
    g = torch.Generator(device="cuda").manual_seed(2)
    M, K, N = 4096, 256, 512
    X = torch.randn(M, K, device="cuda", generator=g).to(torch.float16)
    dY = (torch.randn(M, N, device="cuda", generator=g) * 1e-3).to(torch.float16)
    dW = torch.ones(K, N, device="cuda")
    L.gemm(X, dY, dW, a_mn=True, b_mn=True, accumulate=True, splitk=0)
    ref = 1.0 + X.float().t() @ dY.float()
    assert float((dW - ref).abs().max()) < 1e-4


def test_f16_epilogue_bias_relu_mask_residual():
    g = torch.Generator(device="cuda").manual_seed(3)
    M, N, K = 512, 256, 256
    A = torch.randn(M, K, device="cuda", generator=g).to(torch.float16)
    W = (torch.randn(K, N, device="cuda", generator=g) * 0.1).to(torch.float16)
    bias = torch.randn(N, device="cuda", generator=g)
    H = torch.zeros(M, N, device="cuda", dtype=torch.float16)
    L.gemm(A, W, H, b_mn=True, bias=bias, relu=True)
    ref = torch.relu(A.float() @ W.float() + bias)
    assert float((H.float() - ref).abs().max()) < 2e-2
    # dgrad-style: fp16 gradient x fp16 weight, masked by the fp16 forward activation, fp32 residual
    dY = torch.randn(M, N, device="cuda", generator=g).to(torch.float16)
    res = torch.randn(M, K, device="cuda", generator=g)
    Wt = (torch.randn(N, K, device="cuda", generator=g) * 0.1).to(torch.float16)     # [N_out=K_in...] B as K-major [n,k]
    msk = (torch.randn(M, K, device="cuda", generator=g)).to(torch.float16)
    dX = torch.zeros(M, K, device="cuda")
    L.gemm(dY, Wt.t().contiguous(), dX, mask_src=msk, residual=res, alpha=0.5)
    ref = (0.5 * (dY.float() @ Wt.float())) * (msk.float() > 0) + res
    assert float((dX - ref).abs().max()) < 1e-3 * float(ref.abs().max())
