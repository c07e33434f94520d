"""Fused FFN at the benchmark's shapes: a full training step (forward and backward, dropout 0.1) with the fused FFN kernel
against the same step on the GEMM chain (`disable_fused_attention` selects both reference paths), in fp16 and bf16.

speech_transformer_s dimensions (d 256, ffn 2048) at B = 32, T = 1000, L = 88 give the encoder's M = 8000 rows (63 row
tiles, 2 hidden slices per tile) and the decoder's M = 2816 (22 tiles, 4 slices).  B = 4 with ragged lengths gives
M = 1000, a partial last row tile and 16 slices of one 128-column chunk each.  d = 128 runs the other accumulator width
(M = 1200, again a partial row tile)."""
import pytest
import torch

from oracle import restatement as R
from tests import parity_utils as U

pytestmark = pytest.mark.gpu

S_DIMS = dict(model="speech", d=256, heads=4, enc_layers=2, dec_layers=1, ffn=2048, channels=64, feat=80, in_channels=1, vocab=96)
SHAPES = {
    "s_M8000_M2816": (S_DIMS, 32, 1000, 88, None),
    "s_M1000_ragged": (S_DIMS, 4, 1000, 40, [1000, 480, 777, 913]),
    "d128_M1200": (dict(S_DIMS, d=128, heads=2, ffn=1024), 8, 600, 30, [600, 600, 411, 599, 256, 600, 533, 97]),
}


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_fused_ffn_step_matches_gemm_chain(shape, precision):
    from neurst_b200 import lib as L
    from neurst_b200.runtime import Runtime, make_config
    cfg, B, T, Lq, lengths = SHAPES[shape]
    P = R.init_params(cfg, seed=11, random_bias=True)
    batch = U.synthetic_speech_batch(cfg, B, T, Lq, seed=5)
    if lengths is not None:
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
