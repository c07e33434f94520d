"""Whole-step parity of the speech front-end (conv1 + LN + ReLU, conv2 + LN + ReLU, dense) against the fp64 oracle, per
gradient tensor, across the geometries that select different kernels:

- C == 256, Cin == 1 (normalised-save conv1): in 16 bits with F2 <= 128 the implicit conv2 data gradient (four parity-class
  GEMMs writing class-major tiles of tu = 128 // F2 time rows) read back by conv1's backward; in fp32, and in 16 bits with
  F2 > 128, the explicit data gradient and the col2im gather.
- any other width or input-channel count: the generic conv1 forward and fused backward (VEC x CPL 8/16 x Cin 1/>1).

A relative L2 over every position dilutes a bug at one border, so besides a random fbank (`random`) the source is also
non-zero only in a band of 3 frames or bins at one edge (`t_end`, `f_end`, `start`).  conv1's filter gradient is
col1^T dz1 and col1 is zero outside the band, so src.conv1.kernel is then built from the border positions alone and a wrong
border row is an O(1) error in it.

16-bit runs load weights already rounded to their 16-bit type and give the oracle the same values: the shadow then equals
the fp32 master copy (conv1's affine parameters are read from the shadow) and only activation rounding is left."""
import pytest
import torch

from neurst_b200 import lib as L
from oracle import restatement as R
from tests import parity_utils as U

pytestmark = pytest.mark.gpu

DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
FRONT = ("src.conv1.kernel", "src.conv1.bias", "src.ln1.gamma", "src.ln1.beta", "src.conv2.kernel", "src.conv2.bias",
         "src.ln2.gamma", "src.ln2.beta", "src.dense.kernel", "src.dense.bias")
B, LQ = 3, 5

# Bounds: logits max-abs, loss abs, per-front-end-tensor relative L2, and the worst relative L2 over the rest of the
# model.  fp32 is held to the bound of the existing whole-model fp32 test (the largest error measured here is 5e-6 front,
# 3e-5 rest).  The 16-bit bounds are about 3x the largest error of the correct build over seeds 0..2 at every geometry and
# probe below, measured on an H100 SXM (700 W):
#              logits   loss     front    rest
#   fp16       1.8e-3   3.6e-4   4.1e-2   1.0e-1
#   bf16       1.5e-2   2.8e-3   1.5e-1   1.5e-1
# At this model size the 16-bit error of every gradient is set by the 16-bit backward of the whole model, not by the
# front-end (dense.bias is as far off as conv1.kernel), so a border bug is resolved by the fp32 runs and, through the
# edge probes, by the fp16 runs; the bf16 bounds catch gross errors only.
TOL = {
    "fp32": dict(logits=1e-4, loss=1e-4, front=2e-4, rest=2e-4),
    "fp16": dict(logits=6e-3, loss=1.2e-3, front=1.2e-1, rest=3e-1),
    "bf16": dict(logits=5e-2, loss=1e-2, front=4.5e-1, rest=4.5e-1),
}


def small_cfg(F, C, Cin):
    return dict(model="speech", d=64, heads=4, enc_layers=1, dec_layers=1, ffn=128, channels=C, feat=F, in_channels=Cin,
                vocab=96)


def probe_batch(cfg, T, probe, seed):
    """Synthetic batch (ragged lengths, utterance 0 at full length) with the fbank kept only where `probe` says."""
    batch = U.synthetic_speech_batch(cfg, B, T, LQ, seed=seed)
    src, lengths, F = batch["src"], batch["src_length"], cfg["feat"]
    keep = torch.zeros(B, T, F, 1, dtype=torch.bool)
    t = torch.arange(T).view(1, T, 1, 1)
    f = torch.arange(F).view(1, 1, F, 1)
    n = lengths.view(B, 1, 1, 1)
    if probe == "random":
        keep[:] = True
    elif probe == "t_end":          # last 3 valid frames: the tensor's edge for utterance 0, interior for the others
        keep = (t >= n - 3) & (t < n)
    elif probe == "f_end":
        keep = (f >= F - 3).expand(B, T, F, 1).clone()
    elif probe == "start":
        keep = ((t < 3) | (f < 3)).expand(B, T, F, 1).clone()
    else:
        raise ValueError(probe)
    batch["src"] = src * keep.to(src.dtype)
    return batch


def front_errors(F, C, Cin, T, precision, probe, seed=0):
    """Runs one forward + backward step on the device and on the fp64 oracle; returns the errors the tests bound."""
    cfg = small_cfg(F, C, Cin)
    P = R.init_params(cfg, seed=100 + seed, random_bias=True)
    if precision in DTYPES:
        P = {k: v.to(DTYPES[precision]).to(torch.float32) for k, v in P.items()}
    batch = probe_batch(cfg, T, probe, seed)
    rt = U.speech_runtime(cfg, precision, dropout=0.0, label_smoothing=0.1)
    rt.load_parameters(P)
    rt.ensure_grads().zero_()
    cb = U.to_cuda(batch)
    cb.update(training=False, want_logits=True)
    out = rt.run(cb, backward=True)
    torch.cuda.synchronize()
    logits, loss, grads = U.oracle_loss_and_grads(P, cfg, batch, 0.1)
    S = float(rt.loss_scale_state[0]) if rt.fp16 else 1.0      # fp16: gradients carry the dynamic loss scale
    errs = {k: U.rel_err(rt.grad_view(k) / S, g) for k, g in grads.items()}
    return dict(logits=float((out["logits"].cpu().double() - logits).abs().max()),
                loss=abs(float(out["loss"]) - float(loss)),
                front={k: errs[k] for k in FRONT},
                rest=max(e for k, e in errs.items() if k not in FRONT))


def check(e, precision):
    tol = TOL[precision]
    assert e["logits"] < tol["logits"], e
    assert e["loss"] < tol["loss"], e
    bad = {k: v for k, v in e["front"].items() if not v < tol["front"]}
    assert not bad, (bad, e)
    assert e["rest"] < tol["rest"], e


# --- C = 256, Cin = 1 -------------------------------------------------------------------------------------------------
# F=80 (production, F2 = 20, tu = 6): every probe at T = 9 (T1 = 5, T2 = 3 < tu), 47 (T1 = 24 even, T2 = 12 a multiple of
# tu) and 61 (T1 = 31 odd, T2 = 16 not a multiple).
PRODUCTION = [(80, T, probe) for T in (9, 47, 61) for probe in ("random", "t_end", "f_end", "start")]
# other feature sizes, each at one odd and one even T1:
#   F=83: F2 = 21, tu = 6 (odd F: 80 fbank + 3 pitch)      T=45: T1 = 23, T2 = 12 = 2 tu;   T=52: T1 = 26, T2 = 13
#   F=64: F2 = 16, tu = 8 (tile exactly full)              T=61: T1 = 31, T2 = 16 = 2 tu;   T=40: T1 = 20, T2 = 10
#   F=40: F2 = 10, tu = 12                                 T=9:  T1 = 5,  T2 = 3 < tu;      T=47: T1 = 24, T2 = 12 = tu
#   F=3:  F2 = 1,  tu = 128 (one frequency column)         T=9:  T1 = 5,  T2 = 3;           T=520: T1 = 260, T2 = 130 (2 tiles)
#   F=512: F2 = 128, tu = 1 (largest implicit F2)          T=9:  T1 = 5,  T2 = 3;           T=12: T1 = 6, T2 = 3
#   F=513: F2 = 129 (16-bit explicit-dgrad fallback)       T=9, T=12
FEATS = {83: (45, 52), 64: (61, 40), 40: (9, 47), 3: (9, 520), 512: (9, 12), 513: (9, 12)}
SWEEP = [(F, T, probe) for F, (ta, tb) in FEATS.items()
         for T, probe in ((ta, "random"), (tb, "random"), (ta, "t_end"), (tb, "t_end"), (ta, "f_end"), (tb, "f_end"))]


@pytest.mark.parametrize("precision", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("F,T,probe", PRODUCTION + SWEEP)
def test_front_c256_vs_oracle(F, T, probe, precision):
    check(front_errors(F, 256, 1, T, precision, probe), precision)


# --- other widths and input channels (generic conv1 kernels); C = 5 is fp32 only (16-bit modes need C % 8 == 0) ----
WIDTHS = [(1, 5), (1, 64), (2, 64), (1, 320), (3, 256), (4, 256)]


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("probe", ["random", "t_end", "f_end"])
@pytest.mark.parametrize("Cin,C", WIDTHS)
def test_front_widths_vs_oracle(Cin, C, probe, precision):
    if precision != "fp32" and C % 8:
        with pytest.raises(L.B200STError, match="channels % 8"):
            U.speech_runtime(small_cfg(83, C, Cin), precision)
        return
    check(front_errors(83, C, Cin, 47, precision, probe), precision)


def test_front_out_of_envelope_is_refused():
    """Cin = 3, C = 512: the conv1 filter (28 x 512 floats) does not fit 48 KB of shared memory; the library says so
    before launching anything."""
    cfg = small_cfg(80, 512, 3)
    P = R.init_params(cfg, seed=1, random_bias=True)
    rt = U.speech_runtime(cfg, "fp32")
    rt.load_parameters(P)
    rt.ensure_grads().zero_()
    cb = U.to_cuda(U.synthetic_speech_batch(cfg, 2, 21, LQ, seed=1))
    cb.update(training=False, want_logits=True)
    with pytest.raises(L.B200STError, match="shared memory"):
        rt.run(cb, backward=True)
    torch.cuda.synchronize()
