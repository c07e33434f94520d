"""b200st_optimizer_step vs plain torch: Keras Adam, tf.clip_by_value / tf.clip_by_norm per gradient tensor
(neurst/training/gradaccum_keras_model.py:228-233) and the dynamic loss scale state machine
(neurst/training/revised_dynamic_loss_scale.py:60-107).

The parity tests compare the step with its fp64 restatement (oracle.restatement.optimizer_step and loss_scale_update) at
the toy table (80 tensors, 13 of them followed by alignment padding) and the speech_transformer_s table (280 tensors,
29.3 M parameters), computed with torch float64 on the device from the fp32 values the kernels read: p, m, v, the
gradients and the hyper-parameters as float32 numbers.  What differs is then the kernels' own fp32 rounding, bounded per
element to first order (u = 2^-24, the unit roundoff of fp32; `_adam_bound` and `_sumsq_depth` evaluate these):

  sum of squares of an n-element tensor (grad_stats_kernel, fp32 atomics): every term goes through at most
      d(n) = 40 + min(n / 4 + 2, n / 1024 + 514) additions of non-negative terms (a lane's 32 squares and sums, 5 warp
      shuffles, then one atomicAdd per 1024-element warp range inside the tensor, or per 4-element vector for the two warp
      ranges that straddle its ends; a tensor under 1024 elements takes per-vector atomics only):  |dS| <= d(n) u S.
      The total sums the n_tensors partial sums in sequence: d_total = max d(n) + n_tensors; ctl[5] = sqrtf(total) *
      grad_scale / S has relative error d_total u / 2 + 3u.
  gradient Adam sees, g' = g * grad_scale / S (* c / max(||g'||, c)): relative error e_g = 3u, + d(n) u / 2 + 5u with
      clip_norm (the tensor's norm: sqrtf of its sum of squares, two products; the quotient: two roundings).  Clipping by
      value is 1-Lipschitz and adds nothing.
  m = b1 m0 + (1 - b1) g' (1 - b1 is exact in fp32):     |dm| <= 3u (b1 |m0| + (1 - b1) |g'|) + (1 - b1) |g'| e_g
  v = b2 v0 + (1 - b2) g'^2 (every term >= 0):          |dv| <= (4u + 2 e_g) v
  lr_t = lr sqrtf(1 - powf(b2, t)) / (1 - powf(b1, t)), powf within 8 ulp: 1 - b^t has relative error
      e(b) = 8u b^t / (1 - b^t) + u, and e_lr = e(b1) + e(b2) / 2 + 4u.
  s = lr_t m / (sqrtf(v) + eps):                         |ds| <= lr_t |dm| / (sqrt(v) + eps) + |s| (|dv| / 2v + 3u + e_lr)
  p = p0 - s:                                            |dp| <= u |p| + |ds|
Each bound is doubled for the second-order terms.  At the 6 updates below the step size of Adam's t and t + 1 differ by
3.5 % and more, so a wrong t in the bias correction exceeds every bound by orders of magnitude; so does a vector of the
gradient counted against the neighbouring tensor, as neighbouring tensors' gradients differ by a factor 2 or 2^20 in
magnitude (`_magnitudes`)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from neurst_b200 import checkpoints as CK
from neurst_b200 import lib as L
from oracle import restatement as R
from tests import parity_utils as U

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24


def f32(x):
    return float(np.float32(x))


HP = dict(beta1=f32(0.9), beta2=f32(0.98), eps=f32(1e-9))     # the kernel's hyper-parameters, as float32 numbers


def _toy_rt(precision="fp32"):
    cfg = dict(R.CONFIGS["speech_transformer_toy"])
    if precision != "fp32":      # the tensor-core precisions need 8-element aligned dims
        cfg = dict(model="speech", d=64, heads=4, enc_layers=1, dec_layers=1, ffn=64, channels=64, feat=80, in_channels=1, vocab=96)
    rt = U.speech_runtime(cfg, precision)
    rt.load_parameters(R.init_params(cfg, seed=1, random_bias=True))
    return rt


@pytest.mark.parametrize("mode", ["value", "norm"])
def test_clipping_matches_tf_semantics(mode):
    rt = _toy_rt()
    g = torch.Generator().manual_seed(0)
    grad = torch.randn(rt.numel, generator=g) * 3.0
    # zero the alignment padding between tensors (the library never writes gradients there)
    keep = torch.zeros(rt.numel, dtype=torch.bool)
    for off, shp in rt.table.values():
        n = 1
        for s_ in shp:
            n *= s_
        keep[off:off + n] = True
    grad = grad * keep
    p0 = rt.params.clone().cpu()
    rt.ensure_grads().copy_(grad.cuda())
    clip = 0.7 if mode == "value" else 2.5
    lr = 1e-2
    rt.adam_step(lr, 1, grad_scale=0.5, zero_grad=True, clip_value=clip if mode == "value" else None,
                 clip_norm=clip if mode == "norm" else None)
    ge = grad * 0.5
    if mode == "value":
        ge = ge.clamp(-clip, clip)
    else:
        for off, shp in rt.table.values():
            n = 1
            for s_ in shp:
                n *= s_
            t = ge[off:off + n]
            ge[off:off + n] = t * clip / max(float(t.norm()), clip)       # tf.clip_by_norm
    p, _, _ = R.adam_update(p0, ge, torch.zeros_like(p0), torch.zeros_like(p0), lr, 1)
    assert float(((rt.params.cpu() - p) * keep).abs().max()) < 1e-6
    assert float(rt.grads.abs().max()) == 0.0


def test_dynamic_loss_scale_skips_and_recovers():
    rt = _toy_rt("fp16")
    st = rt.loss_scale_state
    assert float(st[0]) == 2.0 ** 15
    p0 = rt.params.clone()
    g = torch.randn(rt.numel, device="cuda") * 2.0 ** 15            # "scaled" gradients
    # 1) non-finite gradient: step skipped, scale halved, gradients zeroed, parameters and shadow untouched
    rt.ensure_grads().copy_(g)
    rt.grads[5] = float("inf")
    rt.adam_step(1e-2, 1, growth_steps=2)
    torch.cuda.synchronize()
    assert torch.equal(rt.params, p0) and float(rt.grads.abs().max()) == 0.0
    assert float(st[0]) == 2.0 ** 14 and float(st[2]) == 1.0 and float(st[3]) == 1.0 and float(st[4]) == 0.0
    # 2) finite gradients under the (new) scale: applied with Adam t = 1 and unscaled by 1/S
    S = float(st[0])
    rt.grads.copy_(g)
    rt.adam_step(1e-2, 999, growth_steps=2)       # host step_t is ignored when the device state counts
    torch.cuda.synchronize()
    pe, _, _ = R.adam_update(p0.cpu(), (g / S).cpu(), torch.zeros(rt.numel), torch.zeros(rt.numel), 1e-2, 1)
    assert float((rt.params.cpu() - pe).abs().max()) < 1e-6
    assert float(st[2]) == 0.0 and float(st[4]) == 1.0 and float(st[1]) == 1.0
    assert abs(float(st[5]) - float((g / S).norm())) < 1e-3 * float((g / S).norm())
    # the fp16 shadow follows the master weights
    assert float((rt.shadow.float() - rt.params).abs().max()) < 1e-3 * float(rt.params.abs().max())
    # 3) second finite step reaches growth_steps = 2: scale doubles
    rt.grads.copy_(g)
    rt.adam_step(1e-2, 999, growth_steps=2)
    torch.cuda.synchronize()
    assert float(st[0]) == 2.0 ** 15 and float(st[1]) == 0.0 and float(st[4]) == 2.0


# ---- fp64 parity of the whole step ----------------------------------------------------------------------------------
CASES = {"fp32-toy": ("speech_transformer_toy", "fp32"), "bf16-s": ("speech_transformer_s", "bf16"),
         "fp16-s": ("speech_transformer_s", "fp16")}


def _slots(rt):
    """(offset, numel) of every parameter tensor, in b200st_param_info order (the order of tensor_sumsq)."""
    return [(off, math.prod(shp)) for off, shp in rt.table.values()]


def _tensor_ids(rt):
    """Per element: its tensor's index, n_tensors in the alignment padding."""
    slots = _slots(rt)
    tid = torch.full((rt.numel,), len(slots), dtype=torch.int64, device=rt.device)
    for i, (off, n) in enumerate(slots):
        tid[off:off + n] = i
    return tid


def _magnitudes(rt):
    """Tensor i's gradients have magnitude 2^((i mod 21) - 10); 0 in the alignment padding (the library never writes
    gradients there)."""
    mag = torch.zeros(rt.numel, dtype=torch.float32, device=rt.device)
    for i, (off, n) in enumerate(_slots(rt)):
        mag[off:off + n] = 2.0 ** ((i % 21) - 10)
    return mag


def _grads(rt, seed, mag=None):
    gen = torch.Generator(device=rt.device).manual_seed(seed)
    return torch.randn(rt.numel, generator=gen, device=rt.device) * (_magnitudes(rt) if mag is None else mag)


def _sumsq(g, tid, n_tensors):
    return torch.zeros(n_tensors + 1, dtype=torch.float64, device=g.device).index_add_(0, tid, g.double() ** 2)[:n_tensors]


def _sumsq_depth(n):
    """The longest chain of fp32 additions a term of an n-element tensor's sum of squares goes through (module docstring)."""
    return 40 + min(n / 4 + 2, n / 1024 + 514)


def _e_pow(b, t):
    return 8 * U32 * b ** t / (1 - b ** t) + U32


def _adam_bound(p, m0, m, v, g, e_g, lr, t, beta1, beta2, eps):
    """Per-element bounds on |dp|, |dm|, |dv| of the fp32 step against the fp64 one (module docstring); p, m, v, g are
    the fp64 results and the fp64 gradient Adam saw, e_g the relative error of the kernel's gradient."""
    u = U32
    ag = g.abs()
    dm = 3 * u * (beta1 * m0.double().abs() + (1 - beta1) * ag) + (1 - beta1) * ag * e_g
    dv_rel = 4 * u + 2 * e_g
    dv = dv_rel * v
    lr_t = lr * math.sqrt(1 - beta2 ** t) / (1 - beta1 ** t)
    e_lr = _e_pow(beta1, t) + _e_pow(beta2, t) / 2 + 4 * u
    den = torch.sqrt(v) + eps
    s = lr_t * m.abs() / den
    ds = lr_t * dm / den + s * (dv_rel / 2 + 3 * u + e_lr)
    dp = u * p.abs() + ds
    return 2 * dp, 2 * dm, 2 * dv


def _assert_within(name, got, ref, bound):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = int(bad.nonzero()[0])
        raise AssertionError("%s: %d elements beyond the bound, e.g. [%d] got %r ref %r bound %r (worst err/bound %.3g)" % (
            name, int(bad.sum()), i, float(got[i]), float(ref[i]), float(bound[i]), float((err / bound.clamp_min(1e-300)).max())))


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _reset(rt, seed):
    """Fresh optimizer state and seeded weights (the shadow their rounding), as a run starts."""
    gen = torch.Generator(device=rt.device).manual_seed(seed)
    rt.params.copy_(torch.randn(rt.numel, generator=gen, device=rt.device) * 0.05)
    rt.refresh_shadow()
    rt.adam_m = rt.adam_v = None
    rt.ensure_grads().zero_()
    if rt.loss_scale_state is not None:
        rt.loss_scale_state.zero_()
        rt.loss_scale_state[0] = 2.0 ** 15
    return rt


@pytest.fixture(scope="module")
def runtimes():
    cache = {}

    def get(case):
        if case not in cache:
            name, precision = CASES[case]
            cache[case] = U.speech_runtime(R.CONFIGS[name], precision)
        return cache[case]
    yield get
    cache.clear()
    torch.cuda.empty_cache()


def _norm_straddling(g, rt, gs, clip_norm, tid):
    """Tensors i = 0 mod 4 get an unscaled norm 2 % below clip_norm, i = 1 mod 4 2 % above (far beyond fp32 rounding);
    the others keep the magnitude pattern, whose norms lie orders of magnitude on either side."""
    nrm = _sumsq(g, tid, len(rt.table)).sqrt() * gs
    target = torch.full_like(nrm, float("nan"))
    target[0::4], target[1::4] = 0.98 * clip_norm, 1.02 * clip_norm
    f = torch.where(torch.isnan(target), torch.ones_like(nrm), target / nrm)
    return (g.double() * torch.cat([f, f.new_ones(1)])[tid]).float()


@pytest.mark.parametrize("grad_scale", [1.0, 1.0 / 6.0])
@pytest.mark.parametrize("mode", ["plain", "value", "norm"])
@pytest.mark.parametrize("case", list(CASES))
def test_step_matches_fp64_restatement(runtimes, case, mode, grad_scale):
    """6 consecutive updates from the device's own state, each compared with the fp64 step from the same fp32 inputs:
    p, m, v within the bounds of the module docstring, the 16-bit shadow the round-to-nearest-even of p bit for bit, the
    gradients zero (bitwise unchanged on the last update, which passes zero_grad = 0).  Where the statistics pass runs
    (clip_norm, the fp16 loss scale), every tensor's sum of squares and their total; in fp16, the gradients carry the
    current scale and the state words follow the restatement exactly, ctl[5] the fp64 global norm within its bound."""
    rt = _reset(runtimes(case), seed=7)
    slots = _slots(rt)
    T = len(slots)
    if case == "fp32-toy":
        assert T == 80 and sum(1 for _, n in slots if n % 8) == 13
    else:
        assert T == 280 and rt.numel == 29264384
    tid = _tensor_ids(rt)
    mag = _magnitudes(rt)
    st = rt.loss_scale_state
    gs = f32(grad_scale)
    clip = dict(plain={}, value=dict(clip_value=0.7), norm=dict(clip_norm=1.5))[mode]
    depth = torch.tensor([_sumsq_depth(n) for _, n in slots] + [0.0], dtype=torch.float64, device=rt.device)
    e_g = 3 * U32 + ((depth[tid] * U32 / 2 + 5 * U32) if mode == "norm" else 0.0)
    stats = mode == "norm" or st is not None
    for k in range(6):
        lr = R.noam_lr(3994 + k, 256, 4000)                 # near the peak: every step is thousands of ulps of p
        S = float(st[0]) if st is not None else 1.0
        g = _grads(rt, seed=1000 * k + 17, mag=mag)
        if mode == "norm":
            g = _norm_straddling(g, rt, gs, clip["clip_norm"], tid)
        g = g * S
        rt.grads.copy_(g)
        p0 = rt.params.clone()
        m0 = rt.adam_m.clone() if rt.adam_m is not None else torch.zeros_like(p0)
        v0 = rt.adam_v.clone() if rt.adam_v is not None else torch.zeros_like(p0)
        st0 = st.clone() if st is not None else None
        zero_grad = k < 5
        rt.adam_step(lr, k + 1, grad_scale=grad_scale, zero_grad=zero_grad, **clip)
        t = k + 1
        pr, mr, vr, ge = R.optimizer_step(p0, g, m0, v0, slots, f32(lr), t, grad_scale=gs, loss_scale=S,
                                          **{c: f32(x) for c, x in clip.items()}, **HP)
        bp, bm, bv = _adam_bound(pr, m0, mr, vr, ge, e_g, f32(lr), t, **HP)
        where = "%s %s gs=%g update %d" % (case, mode, grad_scale, t)
        _assert_within(where + " m", rt.adam_m, mr, bm)
        _assert_within(where + " v", rt.adam_v, vr, bv)
        _assert_within(where + " p", rt.params, pr, bp)
        if rt.shadow is not None:
            assert torch.equal(_bits(rt.shadow), _bits(rt.params.to(rt.shadow.dtype))), where
        if zero_grad:
            assert int(torch.count_nonzero(rt.grads)) == 0, where
        else:
            assert torch.equal(_bits(rt.grads), _bits(g)), where
        if stats:
            ref = _sumsq(g, tid, T)
            _assert_within(where + " tensor_sumsq", rt.tensor_sumsq[:T], ref, 2 * depth[:T] * U32 * ref)
            d_total = float(depth.max()) + T
            total = ref.sum()
            assert abs(float(rt.tensor_sumsq[T]) - float(total)) <= 2 * d_total * U32 * float(total), where
        if st is not None:
            assert st[:5].tolist() == R.loss_scale_update(st0.tolist(), True), where
            assert float(st[6]) == 1.0 / S, where
            norm = math.sqrt(float(total)) * gs / S
            assert abs(float(st[5]) - norm) <= 2 * (d_total * U32 / 2 + 3 * U32) * norm, where


# ---- the loss-scale state machine -------------------------------------------------------------------------------------
def _script():
    """17 updates (scale from 16, growth_steps 3, multiplier 4): None = finite gradients; (value, where) puts one non-finite
    element; "top" = finite gradients under a scale of 2^127 that reaches growth.  NaN, +inf and -inf each meet the first
    element of the arena, the last element of the last tensor and the inside of a small tensor; six of the skips meet a
    scale of 1."""
    nan, inf = float("nan"), float("inf")
    return [None, (nan, "first"), None, None, None, (inf, "last"), (-inf, "small"), (nan, "last"), (inf, "small"),
            (-inf, "first"), (nan, "small"), (inf, "first"), (-inf, "last"), None, None, None, "top"]


@pytest.mark.parametrize("case", ["fp32-toy", "fp16-s"])
def test_loss_scale_state_machine(runtimes, case):
    """Every state word after every update equals the restatement: a skip halves (here: quarters) the scale, not below 1,
    a scale of 2^127 that reaches growth stays and its count restarts, Adam's t counts applied updates only.  A skipped
    update leaves p, m, v and the shadow bitwise unchanged and zeroes the gradients; an applied one matches the fp64 step
    with that t.  fp32-toy runs the state on the fp32 precision (its 5-element conv1 bias holds the small tensor's
    element), fp16-s on the table of speech_transformer_s."""
    rt = _reset(runtimes(case), seed=3)
    if rt.loss_scale_state is None:
        rt.loss_scale_state = torch.zeros(8, dtype=torch.float32, device=rt.device)
    st = rt.loss_scale_state
    st.zero_()
    st[0] = 16.0
    slots = _slots(rt)
    mag = _magnitudes(rt)
    off_small, n_small = rt.table["src.conv1.bias"][0], math.prod(rt.table["src.conv1.bias"][1])
    where_at = {"first": 0, "last": slots[-1][0] + slots[-1][1] - 1, "small": off_small + n_small // 2}
    if case == "fp32-toy":
        assert n_small == 5
    tr = []
    for k, step in enumerate(_script()):
        if step == "top":
            st[0], st[1] = 2.0 ** 127, 2.0
        S = float(st[0])
        lr = R.noam_lr(3990 + k, 256, 4000)
        g = _grads(rt, seed=31 * k + 1, mag=mag)
        # under 2^127 the stored gradients stay at 2^36 times the pattern: their squares still sum to a finite float32
        g = g * (2.0 ** 36 if step == "top" else S)
        finite = not isinstance(step, tuple)
        if not finite:
            g[where_at[step[1]]] = step[0]
        rt.grads.copy_(g)
        before = [x.clone() for x in (rt.params, rt.adam_m if rt.adam_m is not None else rt.params * 0,
                                      rt.adam_v if rt.adam_v is not None else rt.params * 0)]
        shadow0 = rt.shadow.clone() if rt.shadow is not None else None
        st0 = st.clone().tolist()
        rt.adam_step(lr, 999, growth_steps=3, multiplier=4, dynamic_loss_scale=True)
        expect = R.loss_scale_update(st0, finite, growth_steps=3, multiplier=4)
        where = "%s update %d (%r)" % (case, k + 1, step)
        assert st[:5].tolist() == expect, (where, st[:5].tolist(), expect)
        assert float(st[6]) == 1.0 / S, where
        assert int(torch.count_nonzero(rt.grads)) == 0, where
        tr.append(expect[4])
        if not finite:
            for name, a, b in zip("pmv", (rt.params, rt.adam_m, rt.adam_v), before):
                assert torch.equal(_bits(a), _bits(b)), (where, name)
            if shadow0 is not None:
                assert torch.equal(_bits(rt.shadow), _bits(shadow0)), where
            continue
        t = int(expect[4])
        pr, mr, vr, ge = R.optimizer_step(before[0], g, before[1], before[2], slots, f32(lr), t, loss_scale=S, **HP)
        bp, bm, bv = _adam_bound(pr, before[1], mr, vr, ge, 3 * U32, f32(lr), t, **HP)
        _assert_within(where + " m", rt.adam_m, mr, bm)
        _assert_within(where + " v", rt.adam_v, vr, bv)
        _assert_within(where + " p", rt.params, pr, bp)
        if rt.shadow is not None:
            assert torch.equal(_bits(rt.shadow), _bits(rt.params.to(rt.shadow.dtype))), where
    assert st[:5].tolist() == [2.0 ** 127, 0.0, 0.0, 9.0, 8.0]
    assert tr[13] == 5.0                              # the first update after nine skips applies with t = 5


# ---- clipping by value: the sign of the bound, NaN --------------------------------------------------------------------
def _run(rt, seed, updates, **kw):
    _reset(rt, seed)
    for k in range(updates):
        rt.grads.copy_(_grads(rt, seed=100 + k))
        rt.adam_step(R.noam_lr(3999 + k, 256, 4000), k + 1, **kw)
    torch.cuda.synchronize()
    return [x.clone() for x in (rt.params, rt.adam_m, rt.adam_v)]


def test_negative_clip_value_clips_by_its_magnitude(runtimes):
    """GradAccumKerasModel takes abs(clip_value): -0.7 clips exactly as 0.7 does (and is not clipping turned off)."""
    rt = runtimes("fp32-toy")
    pos = _run(rt, 5, 3, clip_value=0.7)
    neg = _run(rt, 5, 3, clip_value=-0.7)
    off = _run(rt, 5, 3)
    for a, b in zip(pos, neg):
        assert torch.equal(_bits(a), _bits(b))
    assert not torch.equal(pos[0], off[0])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_clip_value_keeps_a_nan_gradient(precision):
    """tf.clip_by_value passes a NaN through: the weight, its moments and its 16-bit shadow become NaN, as without
    clipping, instead of taking a full-size step of -clip_value."""
    rt = _toy_rt(precision)
    j = rt.table["enc.0.ffn.w1"][0] + 3
    p0 = rt.params.clone()
    for clip in (0.7, None):
        rt.params.copy_(p0)
        rt.refresh_shadow()
        rt.adam_m = rt.adam_v = None
        g = torch.randn(rt.numel, generator=torch.Generator(device="cuda").manual_seed(9), device="cuda")
        g[j] = float("nan")
        rt.ensure_grads().copy_(g)
        rt.adam_step(1e-3, 1, clip_value=clip)
        torch.cuda.synchronize()
        assert math.isnan(float(rt.params[j])) and math.isnan(float(rt.adam_m[j])) and math.isnan(float(rt.adam_v[j])), clip
        if rt.shadow is not None:
            assert math.isnan(float(rt.shadow[j])), clip
        assert bool(torch.isfinite(rt.params[j + 1:]).all()), clip


# ---- the step without a handle ----------------------------------------------------------------------------------------
def _arena(n, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    p = torch.randn(n, generator=gen, device="cuda") * 0.05
    g = torch.randn(n, generator=gen, device="cuda")
    m = torch.randn(n, generator=gen, device="cuda") * 0.1
    v = torch.rand(n, generator=gen, device="cuda") * 0.5
    return p, g, m, v


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _handleless_args(p, g, m, v, n, lr, t, gs, shadow=None, **clip):
    a = L.OptimArgs()
    a.params, a.grads, a.m, a.v = p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr()
    if shadow is not None:
        a.shadow, a.shadow_dtype = shadow.data_ptr(), L.BF16
    a.numel, a.lr, a.beta1, a.beta2, a.eps = n, lr, HP["beta1"], HP["beta2"], HP["eps"]
    a.step_t, a.grad_scale, a.zero_grad = t, gs, 1
    a.clip_value, a.clip_norm = clip.get("clip_value", 0.0), clip.get("clip_norm", 0.0)
    return a


def test_handleless_step_matches_fp64_and_refuses_unpadded_arenas():
    """b200st_optimizer_step(NULL, ...) (the whole arena one tensor), plain with a bf16 shadow and clipping, updates every
    element of an arena padded to 8, its last one included, as the fp64 step does; an arena of another size is refused
    before any launch and left untouched (its last numel % 4 elements would have kept their old weight, moments and
    gradient)."""
    lib = L.load()
    n = 8 * 1253
    lr, t, gs = 2e-3, 3, 0.25
    # plain Adam with a bf16 shadow
    p, g, m, v = _arena(n, 1)
    p0, g0, m0, v0 = (x.clone() for x in (p, g, m, v))
    shadow = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    L.check(lib.b200st_optimizer_step(None, C.byref(_handleless_args(p, g, m, v, n, lr, t, gs, shadow)), L._stream()))
    pr, mr, vr, ge = R.optimizer_step(p0, g0, m0, v0, [(0, n)], f32(lr), t, grad_scale=gs, **HP)
    bp, bm, bv = _adam_bound(pr, m0, mr, vr, ge, 3 * U32, f32(lr), t, **HP)
    _assert_within("optimizer_step(NULL) bf16 shadow m", m, mr, bm)
    _assert_within("optimizer_step(NULL) bf16 shadow v", v, vr, bv)
    _assert_within("optimizer_step(NULL) bf16 shadow p", p, pr, bp)
    assert float(p[-1]) != float(p0[-1]) and torch.equal(_bits(shadow), _bits(p.to(torch.bfloat16)))
    assert int(torch.count_nonzero(g)) == 0
    # clipping by value and by the norm of the whole arena
    for clip in (dict(clip_value=0.5), dict(clip_norm=20.0)):
        p, g, m, v = _arena(n, 2)
        p0, g0, m0, v0 = (x.clone() for x in (p, g, m, v))
        sumsq = torch.zeros(2, dtype=torch.float32, device="cuda")
        a = _handleless_args(p, g, m, v, n, lr, t, gs, **clip)
        a.tensor_sumsq = sumsq.data_ptr()
        L.check(lib.b200st_optimizer_step(None, C.byref(a), L._stream()))
        pr, mr, vr, ge = R.optimizer_step(p0, g0, m0, v0, [(0, n)], f32(lr), t, grad_scale=gs, **clip, **HP)
        e_g = 3 * U32 + ((_sumsq_depth(n) * U32 / 2 + 5 * U32) if "clip_norm" in clip else 0.0)
        assert "clip_norm" not in clip or float(g0.double().norm()) * gs > 1.1 * clip["clip_norm"]      # the clip acts
        bp, bm, bv = _adam_bound(pr, m0, mr, vr, ge, e_g, f32(lr), t, **HP)
        _assert_within("optimizer_step(NULL) %s m" % clip, m, mr, bm)
        _assert_within("optimizer_step(NULL) %s v" % clip, v, vr, bv)
        _assert_within("optimizer_step(NULL) %s p" % clip, p, pr, bp)
        assert float(p[-1]) != float(p0[-1]) and int(torch.count_nonzero(g)) == 0
    # unpadded arenas, with and without a shadow: refused with the reason, nothing launched, nothing written
    for bad in (n + 1, n + 4, 1001):
        p, g, m, v = _arena(n + 8, 3)
        shadow = p.to(torch.bfloat16)
        before = [x.clone() for x in (p, g, m, v, shadow)]
        torch.cuda.synchronize()
        launches = L.launch_count()
        for sh in (shadow, None):
            rc = lib.b200st_optimizer_step(None, C.byref(_handleless_args(p, g, m, v, bad, lr, t, gs, sh)), L._stream())
            assert rc != 0 and "multiple of 8" in lib.b200st_last_error().decode()
        torch.cuda.synchronize()
        assert L.launch_count() == launches, bad
        for x, y in zip((p, g, m, v, shadow), before):
            assert torch.equal(_bits(x), _bits(y)), bad


# ---- more than 512 parameter tensors -----------------------------------------------------------------------------------
def test_more_than_512_tensors_plain_step_and_refusals():
    """A text Transformer with 567 parameter tensors: the plain step matches fp64; clip_norm and the dynamic loss scale,
    whose statistics pass holds at most 512 tensors, are refused with that reason before any launch."""
    cfg = dict(model="text", d=8, heads=2, ffn=8, enc_layers=20, dec_layers=16, vocab=16, src_vocab=16)
    rt = U.text_runtime(cfg, "fp32")
    assert int(rt.lib.b200st_param_count(rt.handle)) == 567
    _reset(rt, 11)
    slots = _slots(rt)
    for k in range(3):
        lr = R.noam_lr(3999 + k, 256, 4000)
        g = _grads(rt, seed=k)
        rt.grads.copy_(g)
        p0 = rt.params.clone()
        m0 = rt.adam_m.clone() if rt.adam_m is not None else torch.zeros_like(p0)
        v0 = rt.adam_v.clone() if rt.adam_v is not None else torch.zeros_like(p0)
        rt.adam_step(lr, k + 1, grad_scale=0.5)
        pr, mr, vr, ge = R.optimizer_step(p0, g, m0, v0, slots, f32(lr), k + 1, grad_scale=0.5, **HP)
        bp, bm, bv = _adam_bound(pr, m0, mr, vr, ge, 3 * U32, f32(lr), k + 1, **HP)
        _assert_within("567 tensors m", rt.adam_m, mr, bm)
        _assert_within("567 tensors v", rt.adam_v, vr, bv)
        _assert_within("567 tensors p", rt.params, pr, bp)
    state = [x.clone() for x in (rt.params, rt.adam_m, rt.adam_v, rt.grads)]
    for kw in (dict(clip_norm=1.0), dict(dynamic_loss_scale=True)):
        torch.cuda.synchronize()
        launches = L.launch_count()
        with pytest.raises(L.B200STError, match="up to 512 parameter tensors"):
            rt.adam_step(1e-3, 4, **kw)
        torch.cuda.synchronize()
        assert L.launch_count() == launches, kw
        for x, y in zip((rt.params, rt.adam_m, rt.adam_v, rt.grads), state):
            assert torch.equal(_bits(x), _bits(y)), kw


# ---- resume ------------------------------------------------------------------------------------------------------------
RESUME_CFG = dict(model="speech", d=64, heads=4, enc_layers=1, dec_layers=1, ffn=64, channels=64, feat=80, in_channels=1,
                  vocab=96)


def _resume_rt(precision):
    rt = U.speech_runtime(RESUME_CFG, precision)
    rt.load_parameters(R.init_params(RESUME_CFG, seed=1, random_bias=True))
    return rt


def _resume_update(rt, k, skip):
    """Update k (from 1) of the run: seeded gradients under the current scale, non-finite at update `skip`."""
    S = float(rt.loss_scale_state[0]) if rt.fp16 else 1.0
    g = _grads(rt, seed=k) * S
    if k == skip:
        g[7] = float("inf")
    rt.ensure_grads().copy_(g)
    rt.adam_step(R.noam_lr(k - 1, 64, 4000), k, grad_scale=0.5)


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
def test_resume_continues_the_interrupted_run(tmp_path, precision):
    """8 updates in one run, and the same 8 interrupted after 5 by save_npz, a fresh Runtime and load_npz: after update 8
    the two agree bit for bit in p, m, v, the shadow and the loss-scale state (scale, finite steps in a row, last step
    skipped, applied steps; ctl[3] counts the skips of the current run and ctl[5] comes from atomics).  In fp16 update 3
    is skipped, so Adam's t is the device's count of applied updates, which the checkpoint carries."""
    skip = 3 if precision == "fp16" else 0
    whole = _resume_rt(precision)
    steps = {}
    for k in range(1, 9):
        p = whole.params.clone()
        _resume_update(whole, k, skip)
        steps[k] = whole.params - p
    part = _resume_rt(precision)
    for k in range(1, 6):
        _resume_update(part, k, skip)
    path = str(tmp_path / "ckpt-5.npz")
    CK.save_npz(part, path)
    resumed = _resume_rt(precision)
    state = resumed.loss_scale_state
    CK.load_npz(resumed, path)
    assert resumed.loss_scale_state is state                  # in place: captured CUDA graphs hold its pointer
    p = resumed.params.clone()
    _resume_update(resumed, 6, skip)
    d6 = resumed.params - p
    ratio = float(d6.abs().median() / steps[6].abs().median())
    for k in (7, 8):
        _resume_update(resumed, k, skip)
    torch.cuda.synchronize()
    for name in ("params", "adam_m", "adam_v", "shadow"):
        assert torch.equal(_bits(getattr(resumed, name)), _bits(getattr(whole, name))), (
            "%s differs after update 8 (the resumed run's update 6 was %.2fx the uninterrupted one's)" % (name, ratio))
    if precision == "fp16":
        for i in (0, 1, 2, 4, 6):
            assert float(resumed.loss_scale_state[i]) == float(whole.loss_scale_state[i]), i
        assert float(whole.loss_scale_state[4]) == 7.0 and float(whole.loss_scale_state[3]) == 1.0
