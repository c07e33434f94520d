"""The training step adds its gradients into the fp32 arena (include/b200st.h: "gradients are ACCUMULATED"): the grouped
weight-gradient kernel and the fused FFN kernel leave their tiles as TMA bulk reduce-adds, never as stores.  A step on an
arena pre-filled with a seeded random G0 must leave G0 + G, where G is the same step's gradient on a zeroed arena.

The speech config takes the implicit front-end (channels 256, one input channel, F2 = 20: the conv2 filter gradient is a
one-product group) and has cross-attention, so the step runs groups of 1 (conv2), 2 (self-attention out + qkv, FFN w2 + w1)
and 3 (cross-attention q, out, kv) products, the split-K and accumulate GEMMs, and the tied target embedding, whose gradient
the logits' weight gradient (side stream) and the embedding backward (main stream) both add to.

G0 is scaled per tensor to 4 max |G|: a tile stored instead of added is off by about |G0| there.  The checks allow the
rounding of the add (a few ulps of |G0| + |G|) and 5e-2 max |G| for the run-to-run spread of the step itself: its fp32
atomic sums land in a different order each run and flip roundings of the 16-bit data gradients, which the front-end
filter gradients sum over every position (measured up to 1e-3 of max |G| in fp16 and 5e-3 in bf16)."""
import pytest
import torch

from oracle import restatement as R
from tests import parity_utils as U

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
def test_step_adds_into_prefilled_gradients(precision):
    from neurst_b200 import lib as L
    from neurst_b200.runtime import Runtime, make_config
    cfg = dict(model="speech", d=256, heads=4, enc_layers=2, dec_layers=2, ffn=1024, channels=256, feat=80, in_channels=1, vocab=512)
    P = R.init_params(cfg, seed=21, random_bias=True)
    batch = U.to_cuda(U.synthetic_speech_batch(cfg, 8, 240, 40, seed=6))

    def step(prefill):
        c = make_config(L.MODEL_SPEECH, cfg["d"], cfg["heads"], cfg["ffn"], cfg["enc_layers"], cfg["dec_layers"], cfg["vocab"],
                        feat=cfg["feat"], in_channels=cfg["in_channels"], channels=cfg["channels"], precision=precision,
                        attention_dropout=0.1, ffn_dropout=0.1, postprocess_dropout=0.1, label_smoothing=0.1)
        rt = Runtime(c)
        rt.load_parameters(P)
        rt.ensure_grads().zero_()
        for k, g0 in prefill.items():
            rt.grad_view(k).copy_(g0)
        b = dict(batch)
        b.update(training=True, seed=9)
        rt.run(b, backward=True)
        torch.cuda.synchronize()
        out = {k: rt.grad_view(k).clone() for k in rt.table}
        del rt
        return out

    G = step({})
    gen = torch.Generator(device="cuda").manual_seed(1234)
    G0 = {k: torch.randn(g.shape, device="cuda", generator=gen) * (4.0 * float(g.abs().max()) or 1.0) for k, g in G.items()}
    G1 = step(G0)
    eps = torch.finfo(torch.float32).eps
    bad = []
    for k, g in G.items():
        d = (G1[k] - G0[k] - g).abs()
        tol = 8 * eps * (G0[k].abs() + g.abs()) + 5e-2 * float(g.abs().max())
        if not bool((d <= tol).all()):
            bad.append((k, float(d.max()), float(g.abs().max()), float((d > tol).float().mean())))
    assert not bad, bad
    assert all(bool(torch.isfinite(g).all()) for g in G.values())
