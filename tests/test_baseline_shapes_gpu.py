"""Parity at the BASELINE.json configurations (not toy shapes): speech_transformer_s (d=256, H=4, ffn=2048, 12+6 layers,
V=8192) on [B,1000,80] / L=88 (cfg-2) and [B,1500,80] / L=128 (cfg-3), speech_transformer_m (d=512, H=8) on the T=300 and
T=3000 buckets (cfg-4); ragged lengths, dropout off/on.  CUDA path through the C ABI vs the fp64 oracle: logits, loss and
EVERY gradient tensor.  Tolerances (max-abs logits on O(1) logits / relative L2 per gradient tensor):
  fp32     1e-4 / 1e-3   (reference's own TF<->PT tolerance class, SURVEY Appx A.11)
  mixed16  5e-3 / 4e-2   (= fp16: the reference's mixed_float16 — fp16 operands and activations, fp32 accumulation, dynamic
           loss scale)
  bf16     6e-2 / 1.5e-1 (8-bit significand operands everywhere; kept as the comparison point)
"""
import time

import pytest
import torch

from oracle import restatement as R
from tests import parity_utils as U

pytestmark = pytest.mark.gpu

_ORACLE_CACHE = {}     # (hp, B, T, L, dropout) -> oracle outputs (the Philox masks are identical for every precision)

TOL = {"fp32": (1e-4, 1e-4, 1e-3), "mixed16": (5e-3, 2e-3, 4e-2), "bf16": (6e-2, 3e-2, 1.5e-1)}
PRECISIONS = ["fp32", "mixed16", "bf16"]


def _run_case(hp, B, T, Lq, precision, dropout, seed=11):
    cfg = dict(R.CONFIGS[hp])
    P = R.init_params(cfg, seed=seed, random_bias=True)
    batch = U.synthetic_speech_batch(cfg, B, T, Lq, seed=seed + 1, ragged=True)
    rt = U.speech_runtime(cfg, precision, dropout=dropout, label_smoothing=0.1)
    rt.load_parameters(P)
    cb = U.to_cuda(batch)
    dseed = 987
    cb.update(training=dropout > 0, seed=dseed, want_logits=True, want_enc_out=True)
    rt.ensure_grads().zero_()
    out = rt.run(cb, backward=True)
    torch.cuda.synchronize()
    T2 = R.length_after_conv(T)
    masks = U.dropout_masks(rt, cfg, B, T2, Lq, dropout, dseed) if dropout > 0 else R.NO_DROPOUT
    t0 = time.time()
    key = (hp, B, T, Lq, dropout)
    if key not in _ORACLE_CACHE:
        _ORACLE_CACHE[key] = U.oracle_loss_and_grads(P, cfg, batch, 0.1, masks)
    logits, loss, grads = _ORACLE_CACHE[key]
    t_or = time.time() - t0
    e_logits = float((out["logits"].cpu().double() - logits).abs().max())
    e_rms = float((out["logits"].cpu().double() - logits).pow(2).mean().sqrt())
    e_loss = abs(float(out["loss"]) - float(loss))
    # fp16 precision: the gradient arena carries the dynamic loss scale (unscaled inside the optimizer step)
    S = float(rt.loss_scale_state[0]) if rt.fp16 else 1.0
    errs = sorted(((U.rel_err(rt.grad_view(k) / S, g), k) for k, g in grads.items()), reverse=True)
    print("\n[baseline-shape %s B=%d T=%d L=%d %s p=%.1f] logits max-abs %.3e rms %.3e | loss %.6f vs %.6f (%.2e) | "
          "worst grads %s | oracle %.1fs" % (hp, B, T, Lq, precision, dropout, e_logits, e_rms, float(out["loss"]), float(loss),
                                              e_loss, ", ".join("%s %.2e" % (k, e) for e, k in errs[:3]), t_or))
    tl, tloss, tg = TOL[precision]
    assert e_logits < tl, e_logits
    assert e_loss < tloss * max(1.0, abs(float(loss))), e_loss
    assert errs[0][0] < tg, errs[:5]
    assert torch.equal(out["n_tokens"].cpu(), batch["trg_length"].clamp(max=Lq).float())


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("dropout", [0.0, 0.1])
def test_cfg2_speech_transformer_s(precision, dropout):
    """BASELINE cfg-2 shape per utterance: [B,1000,80], L=88, speech_transformer_s."""
    _run_case("speech_transformer_s", 2, 1000, 88, precision, dropout)


@pytest.mark.parametrize("precision", ["mixed16"])
def test_cfg3_speech_transformer_s_T1500(precision):
    """BASELINE cfg-3 per-GPU shape: [B,1500,80], L=128 (T'=375: 3 kv blocks, ragged tiles)."""
    _run_case("speech_transformer_s", 2, 1500, 128, precision, 0.1)


@pytest.mark.parametrize("T,B,Lq", [(300, 4, 32), (3000, 1, 152)])
@pytest.mark.parametrize("precision", ["fp32", "mixed16"])
def test_cfg4_speech_transformer_m_buckets(T, B, Lq, precision):
    """BASELINE cfg-4: speech_transformer_m (d=512, H=8), shortest and longest frame buckets, ragged src_length."""
    if precision == "fp32" and T == 3000:
        pytest.skip("fp32 SIMT parity mode at T=3000 (T2 = 750 keys: softmax STEPS = 4) is covered at toy width by "
                    "test_model_gpu.py::test_row_kernel_branches_vs_oracle[T2_757-fp32]; the T=300 bucket runs STEPS = 1")
    _run_case("speech_transformer_m", B, T, Lq, precision, 0.1)
