"""CUDA path (through the C ABI) vs the oracle and the committed golden fixtures — SpeechTransformer
forward, loss and every gradient.  fp32 precision is held to the reference's own tolerances; bf16 (wgmma)
to the stated looser bounds."""
import numpy as np
import pytest
import torch

from oracle import restatement as R
from tests import golden_utils as G
from tests import parity_utils as U

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["refpt_speech_toy", "refpt_speech_small"])
def test_forward_matches_reference_pt_fixture_fp32(name):
    """logits of the UNMODIFIED reference neurst_pt model (committed fixture) vs CUDA fp32 path."""
    z, P, cfg = G.refpt_case(name)
    rt = U.speech_runtime(cfg, "fp32")
    rt.load_parameters(P)
    out = rt.run(U.to_cuda(dict(src=G.t(z["src"]), src_length=torch.tensor(z["src_length"]),
                                trg_input=torch.tensor(z["trg_input"]), want_enc_out=True)), backward=False)
    err = float((out["logits"].cpu() - G.t(z["logits"])).abs().max())
    assert err < 1e-4, err          # north_star: logits within 1e-3 of the reference


def test_forward_bf16_vs_reference_fixture():
    z, P, cfg = G.refpt_case("refpt_speech_small")
    rt = U.speech_runtime(cfg, "bf16")
    rt.load_parameters(P)
    out = rt.run(U.to_cuda(dict(src=G.t(z["src"]), src_length=torch.tensor(z["src_length"]),
                                trg_input=torch.tensor(z["trg_input"]))), backward=False)
    ref = G.t(z["logits"])
    err = float((out["logits"].cpu() - ref).abs().max())
    # bf16 tensor-core operands (8-bit mantissa) through 2+2 layers: stated tolerance 5e-2 abs on O(1) logits
    assert err < 5e-2, err


TOL = {"fp32": (1e-4, 2e-4), "fp16": (8e-3, 5e-2), "bf16": (6e-2, 1e-1)}     # logits max-abs, gradient relative L2


def check_step_vs_oracle(cfg, precision, dropout, B, T, Lq, tol_logits, tol_grad):
    """One training step (forward, label-smoothed loss, backward) through the C ABI against the fp64 oracle with the
    library's own dropout masks: logits, loss, token counts and every gradient tensor."""
    P = R.init_params(cfg, seed=7, random_bias=True)
    batch = U.synthetic_speech_batch(cfg, B, T, Lq, seed=3)
    rt = U.speech_runtime(cfg, precision, dropout=dropout, label_smoothing=0.1)
    rt.load_parameters(P)
    seed = 4242
    cb = U.to_cuda(batch)
    cb.update(training=dropout > 0, seed=seed, want_logits=True)
    rt.ensure_grads().zero_()
    out = rt.run(cb, backward=True)
    T2 = R.length_after_conv(T)
    masks = U.dropout_masks(rt, cfg, B, T2, Lq, dropout, seed) if dropout > 0 else R.NO_DROPOUT
    logits, loss, grads = U.oracle_loss_and_grads(P, cfg, batch, 0.1, masks)
    e_logits = float((out["logits"].cpu().double() - logits).abs().max())
    worst = ("", 0.0)
    S = float(rt.loss_scale_state[0]) if rt.fp16 else 1.0      # fp16: gradients carry the dynamic loss scale
    for k, g in grads.items():
        e = U.rel_err(rt.grad_view(k) / S, g)
        if e > worst[1]:
            worst = (k, e)
    print("\n[%s d=%d H=%d ffn=%d V=%d B=%d T=%d (T2=%d) L=%d p=%.1f] logits max-abs %.3e | loss %.6f vs %.6f | worst grad %s %.2e"
          % (precision, cfg["d"], cfg["heads"], cfg["ffn"], cfg["vocab"], B, T, T2, Lq, dropout, e_logits, float(out["loss"]),
             float(loss), worst[0], worst[1]))
    assert e_logits < tol_logits
    assert abs(float(out["loss"]) - float(loss)) < tol_logits * max(1.0, abs(float(loss)))
    nt = batch["trg_length"].clamp(max=Lq).float()
    assert torch.equal(out["n_tokens"].cpu(), nt)
    assert worst[1] < tol_grad, worst


@pytest.mark.parametrize("precision,tol_logits,tol_grad", [(p,) + TOL[p] for p in ("fp32", "fp16", "bf16")])
@pytest.mark.parametrize("dropout", [0.0, 0.1])
@pytest.mark.parametrize("channels", [64, 256])      # 256 = the production front-end kernels (normalised-save conv1 path)
def test_forward_backward_vs_oracle(precision, tol_logits, tol_grad, dropout, channels):
    cfg = dict(model="speech", d=64, heads=4, enc_layers=2, dec_layers=2, ffn=128, channels=channels, feat=80, in_channels=1, vocab=96)
    check_step_vs_oracle(cfg, precision, dropout, 3, 61, 9, tol_logits, tol_grad)


def speech_cfg(d, heads, ffn, vocab, channels=8):
    return dict(model="speech", d=d, heads=heads, enc_layers=2, dec_layers=2, ffn=ffn, channels=channels, feat=80, in_channels=1,
                vocab=vocab)


# Shapes that select the row kernels' other branches (neurst_b200/csrc/elem_kernels.cu).  The unfused attention path (fp32, or
# 16-bit with head dim != 64) runs softmax_fwd/bwd with STEPS = ceil(Tk / 256) rounded up to 1, 2, 4 or 8; T2 is the key
# length after the two stride-2 convolutions, R.length_after_conv(T): T = 1204 -> 301, 3028 -> 757, 4804 -> 1201.
BRANCH_CASES = [
    # d % 8 == 4: ln_bwd_vec_kernel hands dY to the next backward block through the dropout bitmap at rows whose first
    # element is not on a byte boundary; V = 97: the scalar lsce_kernel (V % 4 != 0) and scalar colsum_kernel (V % 8 != 0)
    pytest.param(speech_cfg(12, 3, 20, 97), "fp32", 0.1, 3, 61, 9, id="d12-fp32-p0.1"),
    pytest.param(speech_cfg(12, 3, 20, 97), "fp32", 0.0, 3, 61, 9, id="d12-fp32-p0"),
    # d % 4 != 0: ln_fwd_kernel and ln_bwd_kernel, then the separate cast_dropout for the next block's dY
    pytest.param(speech_cfg(10, 2, 14, 96), "fp32", 0.1, 3, 61, 9, id="d10-fp32-p0.1"),
    # long keys on the unfused path: encoder self-attention and cross-attention at Tk = T2 (STEPS 2, 4, 8, Tk % 8 != 0),
    # decoder self-attention at Tk = Lq = 261 (causal, STEPS 2)
    pytest.param(speech_cfg(16, 2, 24, 96), "fp32", 0.1, 2, 1204, 261, id="T2_301-L261-fp32"),
    pytest.param(speech_cfg(16, 2, 24, 96), "fp32", 0.1, 2, 3028, 9, id="T2_757-fp32"),
    pytest.param(speech_cfg(16, 2, 24, 96), "fp32", 0.1, 2, 4804, 9, id="T2_1201-fp32"),
    # 16-bit P (dropout on the rounded probabilities), head dim 32: not the fused kernel
    pytest.param(speech_cfg(64, 2, 128, 96), "bf16", 0.1, 2, 1204, 9, id="T2_301-bf16"),
    pytest.param(speech_cfg(64, 2, 128, 96), "fp16", 0.1, 2, 1204, 9, id="T2_301-fp16"),
    pytest.param(speech_cfg(64, 2, 128, 96), "bf16", 0.1, 2, 3028, 9, id="T2_757-bf16"),
    pytest.param(speech_cfg(64, 2, 128, 96), "fp16", 0.1, 2, 3028, 9, id="T2_757-fp16"),
    # vocabulary: 8200 -> lsce_vec_kernel<32> and the vector colsum; above 32768 -> the scalar lsce_kernel (bf16: 16-bit
    # dlogits)
    pytest.param(speech_cfg(16, 2, 24, 8200), "fp32", 0.1, 2, 61, 9, id="V8200-fp32"),
    pytest.param(speech_cfg(16, 2, 24, 8200), "bf16", 0.1, 2, 61, 9, id="V8200-bf16"),
    pytest.param(speech_cfg(16, 2, 24, 32776), "bf16", 0.1, 2, 61, 9, id="V32776-bf16"),
    pytest.param(speech_cfg(16, 2, 24, 40000), "fp32", 0.1, 2, 61, 9, id="V40000-fp32"),
]


@pytest.mark.parametrize("cfg,precision,dropout,B,T,Lq", BRANCH_CASES)
def test_row_kernel_branches_vs_oracle(cfg, precision, dropout, B, T, Lq):
    check_step_vs_oracle(cfg, precision, dropout, B, T, Lq, *TOL[precision])


def test_kat_text_transformer_toy_fp32():
    """tests/neurst/models/transformer_test.py:23-665 — TF-generated logits of the 2+2-layer toy Transformer."""
    from tests.test_oracle import transformer_toy_params
    from neurst_b200 import lib as L
    k = G.load("kat_transformer")
    cfg, P = transformer_toy_params(k)
    rt = U.text_runtime(cfg, "fp32")
    rt.load_parameters(P)
    out = rt.run(U.to_cuda(dict(src=torch.tensor(k["dict:src"], dtype=torch.long), src_padding=G.t(k["dict:src_padding"]),
                                trg_input=torch.tensor(k["dict:trg_input"], dtype=torch.long))), backward=False)
    assert float(((out["logits"].cpu().double() - torch.tensor(k["expect:0"])) ** 2).sum()) < 1e-9


def test_adam_step_matches_oracle():
    cfg = dict(R.CONFIGS["speech_transformer_toy"])
    P = R.init_params(cfg, seed=1, random_bias=True)
    rt = U.speech_runtime(cfg, "fp32")
    rt.load_parameters(P)
    g = torch.Generator().manual_seed(0)
    grad = torch.randn(rt.numel, generator=g)
    p0 = rt.params.clone().cpu()
    m = torch.zeros_like(p0); v = torch.zeros_like(p0); p = p0.clone()
    for t in (1, 2, 3):
        rt.ensure_grads().copy_(grad.cuda() * t)
        lr = R.noam_lr(t - 1, 256, 4000, 3.5)
        rt.adam_step(lr, t, grad_scale=0.5, zero_grad=True)
        p, m, v = R.adam_update(p, grad * t * 0.5, m, v, lr, t)
        assert float(rt.grads.abs().max()) == 0.0
    assert float((rt.params.cpu() - p).abs().max()) < 1e-6


def test_cuda_graph_step_matches_eager():
    """A CUDA-graph replay of forward+backward (device-resident dropout seed) gives the same loss and gradients as the
    eager launch sequence with the same seed, and different seeds give different dropout draws."""
    from neurst_b200.runtime import GraphedTrainStep
    cfg = dict(model="speech", d=64, heads=4, enc_layers=2, dec_layers=2, ffn=128, channels=64, feat=80, in_channels=1, vocab=96)
    P = R.init_params(cfg, seed=7, random_bias=True)
    B, T, Lq = 3, 61, 9
    batch = U.to_cuda(U.synthetic_speech_batch(cfg, B, T, Lq, seed=3))
    rt = U.speech_runtime(cfg, "bf16", dropout=0.1, label_smoothing=0.1)
    rt.load_parameters(P)
    rt.ensure_grads().zero_()
    eb = dict(batch); eb.update(training=True, seed=77, want_logits=False)
    out = rt.run(eb, backward=True)
    g_eager, loss_eager = rt.grads.clone(), float(out["loss"])
    step = GraphedTrainStep(rt, B, T, Lq).capture()
    rt.grads.zero_()
    loss_graph = float(step(batch, 77)["loss"])
    torch.cuda.synchronize()
    assert abs(loss_graph - loss_eager) < 1e-6
    # split-K wgrads accumulate with fp32 atomics: order-dependent rounding only
    assert U.rel_err(rt.grads, g_eager) < 1e-4
    rt.grads.zero_()
    assert abs(float(step(batch, 78)["loss"]) - loss_eager) > 1e-7


FUSED_CFG = dict(model="speech", d=128, heads=2, enc_layers=2, dec_layers=2, ffn=128, channels=64, feat=80, in_channels=1, vocab=96)


@pytest.mark.parametrize("T,dropout", [(600, 0.0), (600, 0.1), (1100, 0.1)])
def test_fused_attention_path_vs_oracle(T, dropout):
    """head dim 64 => the fused wgmma flash-attention kernels (forward + backward): multiple q tiles / kv blocks,
    ragged key lengths (additive -1e9 key bias), causal decoder self-attention, cross-attention, Philox dropout."""
    cfg = FUSED_CFG
    P = R.init_params(cfg, seed=11, random_bias=True)
    B, Lq = 2, 9
    batch = U.synthetic_speech_batch(cfg, B, T, Lq, seed=5)
    rt = U.speech_runtime(cfg, "bf16", dropout=dropout, label_smoothing=0.1)
    rt.load_parameters(P)
    seed = 99
    cb = U.to_cuda(batch)
    cb.update(training=dropout > 0, seed=seed, want_logits=True)
    rt.ensure_grads().zero_()
    out = rt.run(cb, backward=True)
    T2 = R.length_after_conv(T)
    masks = U.dropout_masks(rt, cfg, B, T2, Lq, dropout, seed) if dropout > 0 else R.NO_DROPOUT
    logits, loss, grads = U.oracle_loss_and_grads(P, cfg, batch, 0.1, masks)
    assert float((out["logits"].cpu().double() - logits).abs().max()) < 6e-2
    assert abs(float(out["loss"]) - float(loss)) < 3e-2
    worst = max((U.rel_err(rt.grad_view(k), g), k) for k, g in grads.items())
    assert worst[0] < 1e-1, worst


def test_fused_attention_matches_materialised_path():
    from neurst_b200 import lib as L
    from neurst_b200.runtime import Runtime, make_config
    cfg = FUSED_CFG
    P = R.init_params(cfg, seed=11, random_bias=True)
    batch = U.to_cuda(U.synthetic_speech_batch(cfg, 2, 600, 9, seed=5))
    res = []
    for disable in (False, True):
        c = make_config(L.MODEL_SPEECH, cfg["d"], cfg["heads"], cfg["ffn"], 2, 2, cfg["vocab"], channels=cfg["channels"],
                        precision="bf16", attention_dropout=0.1, ffn_dropout=0.1, postprocess_dropout=0.1, label_smoothing=0.1,
                        disable_fused_attention=disable)
        rt = Runtime(c)
        rt.load_parameters(P)
        rt.ensure_grads().zero_()
        b = dict(batch); b.update(training=True, seed=5, want_logits=True)
        out = rt.run(b, backward=True)
        res.append((out["logits"].clone(), rt.grads.clone()))
    assert float((res[0][0] - res[1][0]).abs().max()) < 3e-2
    assert U.rel_err(res[0][1], res[1][1]) < 3e-2


@pytest.mark.parametrize("graph", [False, True])
def test_host_pipeline_matches_plain_loop(graph):
    """trainer.HostPipeline (H2D prefetch on a copy stream + one-step-late loss read) produces exactly the losses of the
    plain `train_step` loop on the same batches / seeds (parameters updated by Adam in between)."""
    from neurst_b200.trainer import build_speech_transformer_trainer, synthetic_batch, HostPipeline
    def make():
        tr, _ = build_speech_transformer_trainer("speech_transformer_s", vocab_size=96, precision="bf16", label_smoothing=0.1,
                                                 seed=5, use_cuda_graph=graph)
        return tr
    hbs = [synthetic_batch(2, 120, 7, 96, seed=20 + i, pin=True) for i in range(3)]
    a = make()
    plain = [float(a.train_step({k: v.cuda() for k, v in hbs[i % 3].items()}, seed=100 + i)) for i in range(5)]
    b = make()
    pipe = HostPipeline(b)
    got = [v for v in pipe.run([hbs[i % 3] for i in range(5)], seed0=100) if v is not None]
    assert len(got) == 5
    for x, y in zip(plain, got):
        assert abs(x - y) < 2e-3 * max(1.0, abs(x)), (plain, got)
    assert pipe.h2d_bytes == sum(v.numel() * v.element_size() for v in hbs[0].values())


def test_two_graph_buckets_keep_their_own_workspace():
    """ADVICE r1 (high): a second, larger shape bucket must not invalidate the pointers baked into an earlier graph.
    Capture a small bucket, then a larger one and a bigger eager call (both grow the runtime's shared workspace), then
    replay the small graph and compare with the eager result of the same batch / seed."""
    from neurst_b200.runtime import GraphedTrainStep
    cfg = dict(model="speech", d=64, heads=4, enc_layers=2, dec_layers=2, ffn=128, channels=64, feat=80, in_channels=1, vocab=96)
    P = R.init_params(cfg, seed=7, random_bias=True)
    rt = U.speech_runtime(cfg, "bf16", dropout=0.1, label_smoothing=0.1)
    rt.load_parameters(P)
    rt.ensure_grads().zero_()
    small = U.to_cuda(U.synthetic_speech_batch(cfg, 2, 41, 7, seed=3))
    big = U.to_cuda(U.synthetic_speech_batch(cfg, 6, 203, 19, seed=4))
    g_small = GraphedTrainStep(rt, 2, 41, 7).capture()
    g_big = GraphedTrainStep(rt, 6, 203, 19).capture()
    eb = dict(big); eb.update(training=True, seed=5, want_logits=True)
    rt.run(eb, backward=True)                      # eager call that reallocates the shared workspace
    torch.cuda.empty_cache()
    junk = torch.full((64 << 20,), 7, dtype=torch.uint8, device="cuda")   # whatever was freed gets reused
    rt.grads.zero_()
    es = dict(small); es.update(training=True, seed=77, want_logits=False)
    loss_eager = float(rt.run(es, backward=True)["loss"]); g_eager = rt.grads.clone()
    rt.grads.zero_()
    loss_graph = float(g_small(small, 77)["loss"])
    torch.cuda.synchronize()
    assert abs(loss_graph - loss_eager) < 1e-6
    assert U.rel_err(rt.grads, g_eager) < 1e-4
    rt.grads.zero_()
    float(g_big(big, 5)["loss"])
    del junk


def test_deterministic_mode_is_reproducible():
    """b200st_config.deterministic: the hidden slices of the fused FFN kernel reduce in slice order, so two runs of the
    same step give bit-identical logits (and gradients equal up to the fp32 atomics of the split-K weight gradients);
    the default mode differs run to run at the level of 16-bit roundings (fp32 sums in arrival order)."""
    from neurst_b200 import lib as L
    from neurst_b200.runtime import Runtime, make_config
    cfg = dict(model="speech", d=256, heads=4, enc_layers=2, dec_layers=2, ffn=1024, channels=64, feat=80, in_channels=1, vocab=96)
    P = R.init_params(cfg, seed=3, random_bias=True)
    batch = U.to_cuda(U.synthetic_speech_batch(cfg, 4, 300, 16, seed=5))
    c = make_config(L.MODEL_SPEECH, cfg["d"], cfg["heads"], cfg["ffn"], 2, 2, cfg["vocab"], channels=cfg["channels"], precision="fp16",
                    attention_dropout=0.1, ffn_dropout=0.1, postprocess_dropout=0.1, label_smoothing=0.1, deterministic=True)
    rt = Runtime(c)
    rt.load_parameters(P)
    res = []
    for _ in range(3):
        rt.ensure_grads().zero_()
        b = dict(batch); b.update(training=True, seed=9, want_logits=True)
        out = rt.run(b, backward=True)
        torch.cuda.synchronize()
        res.append((out["logits"].clone(), rt.grads.clone()))
    for lg, g in res[1:]:
        assert torch.equal(lg, res[0][0])
        assert U.rel_err(g, res[0][1]) < 1e-6
