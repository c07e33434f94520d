"""The fused FFN kernel adds each CTA's output rows into x_out with TMA bulk reductions from shared memory.  In the
deterministic mode a slice issues its reductions only after the slices before it have completed theirs (tickets), so at
the benchmark's decoder shape (M = 2816: 22 row tiles x 4 slices on 132 SMs) and at an encoder shape with a partial last
row tile (M = 1600: 13 tiles x 8 slices, the last tile 64 rows), two runs of the same step give bit-identical logits, and
the step matches the GEMM chain."""
import torch

from oracle import restatement as R
from tests import parity_utils as U
import pytest

pytestmark = pytest.mark.gpu


def test_deterministic_bulk_reductions_at_decoder_shape():
    from neurst_b200 import lib as L
    from neurst_b200.runtime import Runtime, make_config
    cfg = dict(model="speech", d=256, heads=4, enc_layers=2, dec_layers=1, ffn=2048, channels=64, feat=80, in_channels=1, vocab=96)
    P = R.init_params(cfg, seed=11, random_bias=True)
    batch = U.to_cuda(U.synthetic_speech_batch(cfg, 32, 200, 88, seed=5, ragged=False))
    res = []
    for disable in (False, False, True):
        c = make_config(L.MODEL_SPEECH, cfg["d"], cfg["heads"], cfg["ffn"], cfg["enc_layers"], cfg["dec_layers"], cfg["vocab"],
                        channels=cfg["channels"], precision="fp16", attention_dropout=0.1, ffn_dropout=0.1,
                        postprocess_dropout=0.1, label_smoothing=0.1, disable_fused_attention=disable, deterministic=True)
        rt = Runtime(c)
        rt.load_parameters(P)
        rt.ensure_grads().zero_()
        b = dict(batch); b.update(training=True, seed=5, want_logits=True)
        out = rt.run(b, backward=True)
        torch.cuda.synchronize()
        res.append((out["logits"].float().clone(), rt.grads.float().clone()))
        del rt
    (lg0, g0), (lg1, g1), (lgc, gc) = res
    assert torch.equal(lg0, lg1)
    assert U.rel_err(g1, g0) < 1e-6           # the split-K weight gradients still add in arrival order
    assert torch.isfinite(g0).all()
    assert float((lg0 - lgc).abs().max()) < 3e-2
    assert U.rel_err(g0, gc) < 3e-2
