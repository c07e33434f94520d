"""Speech front-end gradients against the fp64 oracle at geometries where the 16-bit front-end backward wraps its grid.

The other front-end tests run B = 3 at small T: conv2's data gradient then has fewer work units than CTAs and conv1's
backward gives each warp a phase or two, so neither schedule ever wraps.  Here:

- conv2's data gradient (one launch over the four parity classes) has units = B * ub * 2 (row tiles of tu = 128 // F2 time
  rows times two 128-column n tiles), each of 36 k-blocks (9 taps x 4 channel blocks), statically cut into 132 runs (one
  per CTA of an H100) within one class tile (<= 16 k-blocks) of the mean:
    F = 80,  T = 1000:  F2 = 20, tu = 6, T2 = 250, ub = 42:  units = 3 * 42 * 2 = 252 (not a multiple of 132),
                        9072 k-blocks, 68.7 per CTA: every CTA runs tiles of about two units, cut mid-unit
    F = 127, T = 360:   F2 = 32, tu = 4, T2 = 90,  ub = 23:  units = 3 * 23 * 2 = 138, 4968 k-blocks, 37.6 per CTA
- conv1's backward (264 CTAs of 8 warps, 4 positions per warp and phase) has B * T1 * F1 positions:
    F = 80,  T = 1000:  3 * 500 * 40 = 60000, 28.4 per warp: 8 phases, the last one partly past the end
    F = 127, T = 360:   3 * 180 * 64 = 34560, 16.4 per warp: 5 phases

The fp16 runs take the four probes of test_speech_front_gpu (random fbank, or one non-zero band at an edge, so that a wrong
border row is an O(1) error in conv1's filter gradient); bf16 takes the random fbank.  Bounds: test_speech_front_gpu.TOL."""
import pytest
import torch

from oracle import restatement as R
from tests import parity_utils as U
from tests.test_speech_front_gpu import DTYPES, FRONT, LQ, check, small_cfg

pytestmark = pytest.mark.gpu

B = 3


def probe_batch(cfg, T, probe, seed):
    batch = U.synthetic_speech_batch(cfg, B, T, LQ, seed=seed)
    src, lengths, F = batch["src"], batch["src_length"], cfg["feat"]
    t = torch.arange(T).view(1, T, 1, 1)
    f = torch.arange(F).view(1, 1, F, 1)
    n = lengths.view(B, 1, 1, 1)
    if probe == "random":
        keep = torch.ones(B, T, F, 1, dtype=torch.bool)
    elif probe == "t_end":
        keep = (t >= n - 3) & (t < n)
    elif probe == "f_end":
        keep = (f >= F - 3).expand(B, T, F, 1)
    else:       # "start"
        keep = ((t < 3) | (f < 3)).expand(B, T, F, 1)
    batch["src"] = src * keep.to(src.dtype)
    return batch


def front_errors(F, T, precision, probe, seed=0):
    cfg = small_cfg(F, 256, 1)
    P = R.init_params(cfg, seed=100 + seed, random_bias=True)
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
    S = float(rt.loss_scale_state[0]) if rt.fp16 else 1.0
    errs = {k: U.rel_err(rt.grad_view(k) / S, g) for k, g in grads.items()}
    return dict(logits=float((out["logits"].cpu().double() - logits).abs().max()),
                loss=abs(float(out["loss"]) - float(loss)),
                front={k: errs[k] for k in FRONT},
                rest=max(e for k, e in errs.items() if k not in FRONT))


CASES = ([(80, 1000, "fp16", probe) for probe in ("random", "t_end", "f_end", "start")] +
         [(80, 1000, "bf16", "random"), (127, 360, "fp16", "random"), (127, 360, "fp16", "f_end")])


@pytest.mark.parametrize("F,T,precision,probe", CASES)
def test_front_backward_wrapping_grid_vs_oracle(F, T, precision, probe):
    check(front_errors(F, T, precision, probe), precision)
