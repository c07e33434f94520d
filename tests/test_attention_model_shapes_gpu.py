"""Fused attention at the benchmark's shapes: a full training step (forward and backward, dropout 0.1) with the fused
attention kernels against the same step on the materialised attention path, in fp16 and bf16.

speech_transformer_s dimensions at T = 1000 (T2 = 250, L = 88) give the encoder self-attention (two query tiles), the
decoder cross-attention (Tq 88, Tk 250) and the causal decoder self-attention (88 x 88).  One utterance has 480 frames
(120 subsampled keys), so its second key block holds only padding: the backward skips it and its dK / dV must be zero.
speech_transformer_m dimensions at T = 3000 give Tk = 750: six query tiles per key block, so the two-stage Q / dO ring
of the backward wraps three times."""
import pytest
import torch

from oracle import restatement as R
from tests import parity_utils as U

pytestmark = pytest.mark.gpu

SHAPES = {
    "s_T1000": (dict(model="speech", d=256, heads=4, enc_layers=2, dec_layers=2, ffn=512, channels=64, feat=80, in_channels=1,
                     vocab=96), 4, 1000, 88, [1000, 480, 777, 1000]),
    "m_T3000": (dict(model="speech", d=512, heads=8, enc_layers=1, dec_layers=1, ffn=512, channels=64, feat=80, in_channels=1,
                     vocab=96), 2, 3000, 40, [3000, 2201]),
}


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_fused_attention_step_matches_materialised_path(shape, precision):
    from neurst_b200 import lib as L
    from neurst_b200.runtime import Runtime, make_config
    cfg, B, T, Lq, lengths = SHAPES[shape]
    P = R.init_params(cfg, seed=11, random_bias=True)
    batch = U.synthetic_speech_batch(cfg, B, T, Lq, seed=5)
    batch["src_length"] = torch.tensor(lengths, dtype=batch["src_length"].dtype)
    for b, n in enumerate(lengths):
        batch["src"][b, n:] = 0.0
    batch = U.to_cuda(batch)
    res = []
    for disable in (False, True):
        c = make_config(L.MODEL_SPEECH, cfg["d"], cfg["heads"], cfg["ffn"], cfg["enc_layers"], cfg["dec_layers"], cfg["vocab"],
                        channels=cfg["channels"], precision=precision, attention_dropout=0.1, ffn_dropout=0.1,
                        postprocess_dropout=0.1, label_smoothing=0.1, disable_fused_attention=disable)
        rt = Runtime(c)
        rt.load_parameters(P)
        rt.ensure_grads().zero_()
        b = dict(batch); b.update(training=True, seed=5, want_logits=True)
        out = rt.run(b, backward=True)
        torch.cuda.synchronize()
        res.append((out["logits"].float().clone(), rt.grads.float().clone()))
        del rt
    assert torch.isfinite(res[0][1]).all()
    assert float((res[0][0] - res[1][0]).abs().max()) < 3e-2
    assert U.rel_err(res[0][1], res[1][1]) < 3e-2
