"""The criterion's and the attention softmax's C-ABI kernels per element against fp64:

- b200st_lsce: label-smoothed cross entropy, its per-sequence sums, token counts and loss, and dlogits = loss_scale *
  d(reduce_loss)/d(logits) in fp32, bf16 or fp16 (or none).  Branches (elem_kernels.cu, lsce_fwd_bwd):
  lsce_vec_kernel<8> (V % 4 == 0, V <= 8192, 16-byte aligned logits and dlogits), lsce_vec_kernel<32> (the same up to
  V = 32768), and the scalar lsce_kernel (V % 4 != 0, V > 32768, or a logits view that is not 16-byte aligned).
  Targets outside [0, V) are clamped to 0 and V - 1: that is the library's contract for out-of-range labels, and one
  case pins it down.
- b200st_softmax_fwd (lib.softmax): P = softmax(S + bias[b, k] + causal mask) over the keys, P in fp32, bf16 or fp16.
  Branches (softmax_fwd): a warp per row holding the row in registers, 8 keys per lane per step, STEPS = 1, 2, 4, 8 for
  Tk <= 256, 512, 1024, 2048; more keys are refused on the host.  With a causal mask key k is visible from query q iff
  k <= q + Tk - Tq.

Bounds.  fp32 dlogits: coef * (p - target) with coef = loss_scale / (number of counted tokens).  p in [0, 1] carries
the relative error of the fp32 row sum of exp(z - max) (at most ~160 sequential terms per thread plus a block tree:
~1e-5 in the worst case, ~1e-6 for random rows whose largest p is a few percent) and of lse (a few units in the last
place of |lse| <= ~90, seen only where p is near 1); 4e-6 * coef covers both.  nll_sum: each row's cross entropy is
formed from lse, z[label] - lse and sum(z) - V * lse in fp32, a few units in the last place of |lse| per row; 4e-6 *
max(1, |lse|) per counted row.  Softmax P in fp32: the exponent argument's rounding (|s - max| <= 16 here, 1e-6
relative), expf's two units and the row sum (<= 64 sequential terms per lane, 5 shuffle levels: 4.1e-6 relative)
stay below 8e-6 * P.  16-bit outputs may differ from the fp64 value rounded to their type by one unit in the last place,
plus the fp32 term.  Masked rows (dlogits) and masked keys (P) are exactly zero."""
import pytest
import torch

from neurst_b200 import lib as L
from oracle import restatement as R
from tests.test_front_kernels_gpu import DT, assert_close

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------
# label-smoothed cross entropy
# ---------------------------------------------------------------------------------------------------------------------
def lsce_case(V, seed, B=4, Lq=5):
    """Logits ~ N(0, 2) with one +80 outlier, targets including 0 and V - 1, lengths 0, Lq, > Lq and in between."""
    g = torch.Generator().manual_seed(seed)
    logits = 2.0 * torch.randn(B, Lq, V, generator=g)
    logits[1, 2, (7 * V) // 11] += 80.0
    trg = torch.randint(0, V, (B, Lq), generator=g)
    trg[1, 0], trg[2, 4] = 0, V - 1
    trg_length = torch.tensor([0, Lq, Lq + 3, 2], dtype=torch.long)
    return logits, trg, trg_length


def lsce_device(logits, trg, trg_length, label_smoothing, d_dtype, loss_scale, offset=False):
    B, Lq, V = logits.shape
    buf = torch.empty(B * Lq * V + 1, device="cuda")
    z = (buf[1:] if offset else buf[:-1]).view(B, Lq, V)
    z.copy_(logits)
    trg_d, len_d = trg.cuda(), trg_length.cuda()
    nll = torch.full((B,), float("nan"), device="cuda")
    ntok = torch.full((B,), float("nan"), device="cuda")
    loss = torch.full((1,), float("nan"), device="cuda")
    dl = torch.full((B, Lq, V), float("nan"), dtype=DT[d_dtype], device="cuda") if d_dtype else None
    L.check(L.load().b200st_lsce(z.data_ptr(), trg_d.data_ptr(), len_d.data_ptr(), B, Lq, V, label_smoothing, nll.data_ptr(),
                                 ntok.data_ptr(), loss.data_ptr(), dl.data_ptr() if dl is not None else None,
                                 L._dt(dl) if dl is not None else L.F32, loss_scale, L._stream()))
    torch.cuda.synchronize()
    return nll.cpu(), ntok.cpu(), loss.cpu(), dl.cpu() if dl is not None else None


def check_lsce(logits, trg, trg_length, label_smoothing, d_dtype, loss_scale, offset=False):
    B, Lq, V = logits.shape
    nll, ntok, loss, dl = lsce_device(logits, trg, trg_length, label_smoothing, d_dtype, loss_scale, offset)
    z = logits.double().requires_grad_(True)
    label = trg.clamp(0, V - 1)
    nll_ref, _, ntok_ref = R.label_smoothed_ce(z, label, trg_length, label_smoothing)
    loss_ref = R.reduce_loss(z, label, trg_length, label_smoothing)
    (dz,) = torch.autograd.grad(loss_ref, z)
    w = R.input_length_to_nonpadding(trg_length, Lq, torch.float64)
    assert torch.equal(ntok, ntok_ref.float())
    lse = torch.logsumexp(logits.double(), -1)
    row_tol = 4e-6 * lse.abs().clamp(min=1.0) * w
    assert_close(nll, nll_ref.detach(), torch.float32, row_tol.sum(1), "nll_sum")
    assert_close(loss, loss_ref.detach().view(1), torch.float32, float(row_tol.sum()) / float(ntok_ref.sum()), "loss")
    if dl is None:
        return
    assert torch.isfinite(dl.float()).all()
    masked = w == 0
    assert bool((dl[masked] == 0).all()), "masked rows must have zero dlogits"
    coef = loss_scale / float(ntok_ref.sum())
    assert_close(dl, loss_scale * dz, DT[d_dtype], 4e-6 * coef, "dlogits")


# V -> branch: 12, 8192: lsce_vec_kernel<8>; 8196, 32768: lsce_vec_kernel<32>; 97, 8193 (V % 4 != 0), 32772, 40000
# (V > 32768) and 8192 read through a view one float into its buffer: the scalar lsce_kernel
LSCE_V = [pytest.param(V, False, id=str(V)) for V in (12, 97, 8192, 8193, 8196, 32768, 32772, 40000)] + \
         [pytest.param(8192, True, id="8192-offset")]


@pytest.mark.parametrize("d_dtype,loss_scale", [("fp32", 1.0), ("fp32", 1024.0), ("bf16", 1.0), ("bf16", 1024.0), ("fp16", 1.0),
                                                ("fp16", 1024.0), (None, 1.0)])
@pytest.mark.parametrize("label_smoothing", [0.0, 0.1])
@pytest.mark.parametrize("V,offset", LSCE_V)
def test_lsce_vs_fp64(V, offset, label_smoothing, d_dtype, loss_scale):
    logits, trg, trg_length = lsce_case(V, seed=V)
    check_lsce(logits, trg, trg_length, label_smoothing, d_dtype, loss_scale, offset)


@pytest.mark.parametrize("V", [97, 8192])         # the scalar and the vector kernel
def test_lsce_clamps_out_of_range_labels(V):
    logits, trg, trg_length = lsce_case(V, seed=5)
    trg[1, 1], trg[2, 3] = -3, V + 5
    check_lsce(logits, trg, trg_length, 0.1, "fp32", 1.0)


# ---------------------------------------------------------------------------------------------------------------------
# softmax over keys
# ---------------------------------------------------------------------------------------------------------------------
def round8(x):
    return (x + 7) // 8 * 8


# mode -> (B, H, Tq(Tk), key bias with -1e9 tails, causal, extra row stride of S, extra row stride of P)
SOFTMAX_MODES = {
    "plain": (2, 3, lambda Tk: 5, False, False, 0, 0),
    "bias-wide-rows": (2, 3, lambda Tk: 5, True, False, 24, 16),
    "causal-square": (1, 2, lambda Tk: Tk, False, True, 0, 0),
    "causal-rect-bias": (2, 2, lambda Tk: (Tk + 1) // 2, True, True, 0, 8),
}


@pytest.mark.parametrize("dtype", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("mode", list(SOFTMAX_MODES))
@pytest.mark.parametrize("Tk", [1, 7, 8, 255, 256, 257, 511, 513, 1023, 1025, 2047, 2048])
def test_softmax_fwd_vs_fp64(Tk, mode, dtype):
    B, H, tq, with_bias, causal, padS, padP = SOFTMAX_MODES[mode]
    Tq = tq(Tk)
    ldS, ldP = round8(Tk) + padS, round8(Tk) + padP
    g = torch.Generator().manual_seed(Tk * 13 + len(mode))
    S = (2.0 * torch.randn(B, H, Tq, ldS, generator=g)).cuda()[..., :Tk]
    Pbuf = torch.full((B, H, Tq, ldP), float("nan"), dtype=DT[dtype], device="cuda")
    bias = None
    hidden = torch.zeros(B, 1, Tq, Tk, dtype=torch.bool)
    if with_bias:
        lengths = [Tk] + [max(1, (Tk * (b + 1)) // (B + 2)) for b in range(1, B)]
        bias = torch.zeros(B, Tk)
        for b, n in enumerate(lengths):
            bias[b, n:] = -1e9
            hidden[b, :, :, n:] = True
        bias = bias.cuda()
    if causal:
        k, q = torch.arange(Tk), torch.arange(Tq)
        hidden |= (k[None, :] > q[:, None] + Tk - Tq).view(1, 1, Tq, Tk)
    L.softmax(S, Pbuf[..., :Tk], bias, causal)
    torch.cuda.synchronize()
    P = Pbuf[..., :Tk].cpu()
    ref = torch.softmax(S.double().cpu().masked_fill(hidden, float("-inf")), -1)
    assert torch.isfinite(P.float()).all()
    assert bool((P.expand_as(ref)[hidden.expand_as(ref)] == 0).all()), "masked keys must have P == 0"
    assert_close(P, ref, DT[dtype], 8e-6 * ref, "P Tk=%d %s" % (Tk, mode))
    if padP > 0:       # nothing is written past the padded row (round8(Tk)) into a wider stride
        assert bool(torch.isnan(Pbuf[..., round8(Tk):].float()).all())


def test_softmax_refuses_more_than_2048_keys():
    Tk = 2049
    S = torch.zeros(1, 1, 2, round8(Tk), device="cuda")[..., :Tk]
    P = torch.zeros(1, 1, 2, round8(Tk), device="cuda")[..., :Tk]
    with pytest.raises(L.B200STError, match="2048"):
        L.softmax(S, P)
