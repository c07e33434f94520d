"""Decoding with 16-bit weights (use_shadow=True, the benchmark's path) against an fp64 decoder on the same rounded weights.

In shadow mode the decode kernels read the embedding / tied logits table and the decoder's projection kernels (SHADOW_READ)
from the 16-bit arena; biases, LayerNorm parameters and the cross-attention K/V projection (b200st_decode_init) stay fp32,
and every activation is fp32.  The reference is the oracle's decoder in fp64 with exactly those tensors replaced by their
round-to-nearest 16-bit values (what b200st_refresh_shadow writes), so the only difference left is fp32 against fp64
arithmetic and the tolerances can be tight.  The encoder memory is fixed fp32 data handed to both sides, so the 16-bit
encoder does not enter the decode checks (it has its own test at the end)."""
import functools

import pytest
import torch

from neurst_b200 import decode as D
from oracle import restatement as R
from tests import beam_oracle as BO
from tests import parity_utils as U
from tests.test_beam_search_gpu import _check

pytestmark = pytest.mark.gpu

SMALL = dict(model="speech", d=64, heads=4, enc_layers=2, dec_layers=2, ffn=128, channels=64, feat=80, in_channels=1, vocab=96)
S = dict(R.CONFIGS["speech_transformer_s"])
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
# parameter-name suffixes (after "dec.<i>.") of the tensors the decode kernels read from the 16-bit shadow, and the table
SHADOW_READ = ("trg.emb", "self.qkv.kernel", "self.out.kernel", "cross.q.kernel", "cross.out.kernel", "ffn.w1", "ffn.w2")


def _shadow_kind(name):
    if name == "trg.emb":
        return name
    parts = name.split(".", 2)
    return parts[2] if parts[0] == "dec" and len(parts) == 3 and parts[2] in SHADOW_READ else None


def shadow_rounded(P, dtype, keep=None):
    """fp64 copy of P with every tensor the shadow-mode decoder reads in 16 bits rounded to nearest in `dtype`, except the
    kind `keep` (left at full precision: the reference of a decoder that read that tensor wrongly)."""
    return {k: (v.to(dtype).double() if _shadow_kind(k) not in (None, keep) else v.double()) for k, v in P.items()}


def ragged_memory(cfg, B, Tm, seed):
    """Fixed fp32 encoder memory [B, Tm, d] with ragged lengths (row 0 full) and its additive bias (0 / -1e9)."""
    g = torch.Generator().manual_seed(seed)
    memory = torch.randn(B, Tm, cfg["d"], generator=g)
    lengths = torch.randint(max(1, Tm // 2), Tm + 1, (B,), generator=g)
    lengths[0] = Tm
    bias = R.input_padding_to_bias(R.input_length_to_padding(lengths, Tm, torch.float32))
    return memory, bias


def teacher_forced_logits(P, cfg, memory, bias, ids, dtype=torch.float64):
    """Logits [B, L, V] of the decoder fed ids [B, L] (position t sees ids[:, :t+1]): one causal pass of the oracle's
    decoder, which equals its cached step at every position."""
    Q = {k: v.to(dtype) for k, v in P.items()}
    y = R.decoder(Q, R.target_embed(Q, ids), memory.to(dtype), bias.to(dtype), cfg["dec_layers"], cfg["heads"])
    return R.logits_layer(Q, y)


def decoder_search(P, cfg, memory, bias, bos, eos, unk, beam_size, alpha, **kw):
    """tests/beam_oracle.beam_search over the oracle's cached decoder on a given memory (fp64)."""
    B, H, d = memory.shape[0], cfg["heads"], cfg["d"]
    layers = [dict(keys=torch.zeros(B, 0, H, d // H, dtype=torch.float64), values=torch.zeros(B, 0, H, d // H, dtype=torch.float64))
              for _ in range(cfg["dec_layers"])]
    cache = dict(memory=memory.double(), memory_bias=bias.double(), layers=layers)

    def symbols_to_logits_fn(ids, cache, time):
        x = R.target_embed(P, ids, time=time).unsqueeze(1)
        y = R.decoder(P, x, cache["memory"], cache["memory_bias"], cfg["dec_layers"], H, caches=cache["layers"])
        return R.logits_layer(P, y[:, 0])

    with torch.no_grad():
        return BO.beam_search(symbols_to_logits_fn, torch.full((B,), int(bos), dtype=torch.long), cache, eos, unk, beam_size,
                              alpha, encoder_inputs_maxlen=memory.shape[1], **kw)


def _step_inputs(cfg, B, Tm, n_pos, seed):
    P = R.init_params(cfg, seed=seed, random_bias=True)
    memory, bias = ragged_memory(cfg, B, Tm, seed + 100)
    ids = torch.randint(0, cfg["vocab"], (B, n_pos), generator=torch.Generator().manual_seed(seed + 200))
    return P, memory, bias, ids


def _runtime(cfg, precision, P):
    rt = U.speech_runtime(cfg, precision)
    rt.load_parameters(P)          # fp32 master weights: the library rounds them into the shadow (b200st_refresh_shadow)
    return rt


def _cache(rt, memory, bias, max_len, beam=1):
    return D.create_decoding_cache(rt, memory.cuda(), bias.cuda(), max_len, use_shadow=True, beam=beam)


# ---- teacher-forced step logits (b200st_decode_step) ---------------------------------------------------------------------
# max-abs tolerance on logits of magnitude ~10.  fp32 arithmetic noise on CPU (fp32 oracle vs fp64, same rounded weights) is
# 2e-6 (d 64) to 6e-6 (d 256); the smallest effect of leaving one SHADOW_READ kind unrounded (cross.q.kernel at seed 0)
# is 1.3e-4 / 9.2e-5 with fp16 weights and 1.4e-3 / 6.9e-4 with bf16 weights (d 64 / d 256).  Measured on an H100
# (700 W): 1.2e-6 (d 64) and 2.8e-6 (d 256) for both precisions; a shadow rounded toward zero instead is off by 4e-3 (fp16)
# and 3e-2 (bf16).
N_POS = 24
DIMS = {"small": SMALL, "s": S}
STEP_TOL = {("small", "fp16"): 2.5e-5, ("s", "fp16"): 1.8e-5, ("small", "bf16"): 2.5e-4, ("s", "bf16"): 1.3e-4}


@functools.lru_cache(maxsize=None)
def _step_reference(dims, B, Tm, precision):
    cfg, dt = DIMS[dims], DTYPES[precision]
    P, memory, bias, ids = _step_inputs(cfg, B, Tm, N_POS, seed=0)
    ref = teacher_forced_logits(shadow_rounded(P, dt), cfg, memory, bias, ids)
    effect = {k: float((teacher_forced_logits(shadow_rounded(P, dt, keep=k), cfg, memory, bias, ids) - ref).abs().max())
              for k in SHADOW_READ}
    return P, memory, bias, ids, ref, effect


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("dims,B,Tm", [("small", 2, 61), ("small", 8, 61), ("s", 2, 500)])
def test_step_logits_match_rounded_fp64_decoder(dims, B, Tm, precision):
    P, memory, bias, ids, ref, effect = _step_reference(dims, B, Tm, precision)
    tol = STEP_TOL[dims, precision]
    weakest = min(effect, key=effect.get)
    # the tolerance must resolve any single shadow tensor read at full precision (or rounded another way)
    assert tol <= effect[weakest] / 5, "tolerance %.1e does not resolve %s (effect %.1e)" % (tol, weakest, effect[weakest])
    rt = _runtime(DIMS[dims], precision, P)
    cache = _cache(rt, memory, bias, N_POS)
    out = torch.stack([D.decoder_step_logits(rt, ids[:, t], cache, t) for t in range(N_POS)], 1)
    err = float((out.cpu().double() - ref).abs().max())
    print("\n[step %s B=%d Tm=%d %s] logits max-abs error %.2e, tolerance %.1e, smallest single-tensor effect %.2e (%s)" %
          (dims, B, Tm, precision, err, tol, effect[weakest], weakest))
    assert err < tol, err


# ---- greedy search: token ids identical in the persistent kernel, the captured step graph and eager launches ---------------
GREEDY_CASES = {   # name -> dims, utterances, memory length, chaotic gain, seed, max / extra / min decode length
    "small_b2": ("small", 2, 61, 4.0, 1, 24, 8, 0),
    "small_b8": ("small", 8, 61, 4.0, 1, 24, 8, 0),
    # the benchmark's case: one utterance (2000 frames -> Tm 500), 200 steps forced by minimum_decode_length = 200
    "cfg5": ("s", 1, 500, 2.5, 7, 200, 200, 200),
}


@functools.lru_cache(maxsize=None)
def _chaotic(dims, B, Tm, gain, seed):
    P = U.chaotic_decode_params(R.init_params(DIMS[dims], seed=seed, random_bias=True), gain, seed)
    memory, bias = ragged_memory(DIMS[dims], B, Tm, seed + 100)
    return P, memory, bias


@functools.lru_cache(maxsize=None)
def _greedy_reference(name, precision):
    """The fp64 search on the rounded weights, and the fp32 arithmetic noise of its decoder: max-abs logits difference of
    the fp32 and the fp64 oracle teacher-forced along the hypothesis."""
    dims, B, Tm, gain, seed, max_len, extra, min_len = GREEDY_CASES[name]
    cfg, V = DIMS[dims], DIMS[dims]["vocab"]
    P, memory, bias = _chaotic(dims, B, Tm, gain, seed)
    Pr = shadow_rounded(P, DTYPES[precision])
    ref = decoder_search(Pr, cfg, memory, bias, V - 2, V - 1, V - 3, 1, 0.0, maximum_decode_length=max_len,
                         extra_decode_length=extra, minimum_decode_length=min_len)   # alpha 0: gap = top-1 / top-2 log-prob margin
    inputs = torch.cat([torch.full((B, 1), V - 2), ref["hypotheses"][:, :ref["steps"] - 1]], 1)
    l64 = teacher_forced_logits(Pr, cfg, memory, bias, inputs)
    noise = float((teacher_forced_logits(Pr, cfg, memory, bias, inputs, torch.float32).double() - l64).abs().max())
    return ref, noise


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("name", ["small_b2", "small_b8"])
@pytest.mark.parametrize("use_graph,persistent", [(True, True), (True, False), (False, False)])
def test_greedy_token_ids_exact(name, precision, use_graph, persistent):
    """Gap / noise (CPU, fp32 vs fp64 logits along the hypothesis) at gain 4, seed 1: B 2 fp16 3.6e-3 / 2.5e-5, bf16
    4.0e-3 / 1.5e-5; B 8 (rows ending at lengths 5 to 24) fp16 3.6e-3 / 4.6e-5, bf16 9.5e-3 / 3.8e-5."""
    _greedy_check(name, precision, use_graph, persistent, lambda lp, ref: float((lp - ref).abs().max()) < 1e-3)


def test_greedy_token_ids_exact_cfg5():
    """The benchmark's decode: speech_transformer_s, fp16 shadow, persistent kernel, 200 steps.  Gain 2.5, seed 7: 46
    distinct tokens, gap 1.4e-2, noise 6.4e-5 (at gain 3 the gap was below 10x the noise for each of seeds 0-2)."""
    _greedy_check("cfg5", "fp16", True, True, lambda lp, ref: float(((lp - ref).abs() / ref.abs().clamp(min=1.0)).max()) < 2e-3)


def _greedy_check(name, precision, use_graph, persistent, logprob_ok):
    dims, B, Tm, gain, seed, max_len, extra, min_len = GREEDY_CASES[name]
    ref, noise = _greedy_reference(name, precision)
    hyp = ref["hypotheses"]
    n_distinct = len(set(hyp[:, :ref["steps"]].reshape(-1).tolist()))
    assert ref["gap"] >= 10 * noise, "near-tie in the oracle's search (gap %.2e, noise %.2e): pick another case" % (ref["gap"], noise)
    assert n_distinct >= 8, "degenerate hypothesis: the test would not exercise the context dependence"
    P, memory, bias = _chaotic(dims, B, Tm, gain, seed)
    V = DIMS[dims]["vocab"]
    rt = _runtime(DIMS[dims], precision, P)
    ids, logprob, length = D.greedy_search(rt, None, V - 2, V - 1, V - 3, maximum_decode_length=max_len, extra_decode_length=extra,
                                           minimum_decode_length=min_len, use_shadow=True, use_graph=use_graph,
                                           persistent=persistent, cache=_cache(rt, memory, bias, max_len))
    torch.cuda.synchronize()
    print("\n[greedy %s %s mode %d] %d steps, %d distinct tokens, gap %.2e, noise %.2e, oracle logprob %s cuda %s" %
          (name, precision, int(rt.lib.b200st_greedy_used_graph()), ref["steps"], n_distinct, ref["gap"], noise,
           [round(float(x), 4) for x in ref["logprob"]], [round(float(x), 4) for x in logprob]))
    assert int(rt.lib.b200st_greedy_used_graph()) == (2 if persistent else int(use_graph))
    assert torch.equal(ids.cpu(), hyp), [(i, a, b) for i, (a, b) in enumerate(zip(ids.cpu().view(-1).tolist(), hyp.view(-1).tolist()))
                                         if a != b][:5]
    assert torch.equal(length.cpu().long(), ref["length"])
    assert logprob_ok(logprob.cpu(), ref["logprob"]), (logprob.cpu().tolist(), ref["logprob"].tolist())


# ---- beam search (b200st_beam_search) with the shadow ------------------------------------------------------------------------
BEAM_SEED = {"fp16": 2, "bf16": 1}      # chaotic gain 4; the smallest gap of the four (precision, alpha) cases is 3.4e-4
CFG5_BEAM = dict(gain=2.5, seed=3, steps=64)


@functools.lru_cache(maxsize=None)
def _beam_reference(precision, alpha):
    P, memory, bias = _chaotic("small", 2, 61, 4.0, BEAM_SEED[precision])
    return decoder_search(shadow_rounded(P, DTYPES[precision]), SMALL, memory, bias, 94, 95, 93, 4, alpha,
                          maximum_decode_length=24, extra_decode_length=8)


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("alpha", [0.6, -1.0])
@pytest.mark.parametrize("use_graph", [True, False])
def test_beam_token_ids_exact(precision, alpha, use_graph):
    """Two utterances x beam 4 = the 8 rows of a decoding step."""
    ref = _beam_reference(precision, alpha)
    P, memory, bias = _chaotic("small", 2, 61, 4.0, BEAM_SEED[precision])
    rt = _runtime(SMALL, precision, P)
    ids, scores, logprob, length = D.beam_search(rt, None, 94, 95, 93, beam_size=4, length_penalty=alpha, maximum_decode_length=24,
                                                 extra_decode_length=8, use_shadow=True, use_graph=use_graph,
                                                 cache=_cache(rt, memory, bias, 24, beam=4))
    torch.cuda.synchronize()
    _check(ref, ids, scores, length)
    assert torch.allclose(logprob.cpu(), ref["logprob"], rtol=1e-4, atol=1e-5)


def test_beam_token_ids_exact_cfg5():
    """speech_transformer_s, one utterance (Tm 500), beam 4, 1/len scores, fp16 shadow, 64 steps.  Over 200 steps the
    4th / 5th candidate boundary came within 1.5e-6 in score units for the three seeds tried; at 64 steps seed 3 (gain
    2.5) has a gap of 1.8e-4 and 21 distinct tokens."""
    P, memory, bias = _chaotic("s", 1, 500, CFG5_BEAM["gain"], CFG5_BEAM["seed"])
    V = S["vocab"]
    ref = decoder_search(shadow_rounded(P, torch.float16), S, memory, bias, V - 2, V - 1, V - 3, 4, -1.0,
                         maximum_decode_length=CFG5_BEAM["steps"], extra_decode_length=50)
    rt = _runtime(S, "fp16", P)
    ids, scores, _, length = D.beam_search(rt, None, V - 2, V - 1, V - 3, beam_size=4, length_penalty=-1.0,
                                           maximum_decode_length=CFG5_BEAM["steps"], extra_decode_length=50, use_shadow=True,
                                           cache=_cache(rt, memory, bias, CFG5_BEAM["steps"], beam=4))
    torch.cuda.synchronize()
    n_distinct = len(set(ref["hypotheses"][0].tolist()))
    print("\n[cfg-5 beam 4 fp16] %d steps, length %d, %d distinct tokens, gap %.2e, oracle score %.5f cuda %.5f" %
          (ref["steps"], int(ref["length"][0]), n_distinct, ref["gap"], float(ref["scores"][0]), float(scores[0])))
    _check(ref, ids, scores, length)
    assert n_distinct >= 8, "degenerate hypothesis: the test would not exercise the context dependence"


# ---- the inference encoder (b200st_encode) in 16 bits ------------------------------------------------------------------------
# the BASELINE max-abs logits tolerances of the 16-bit precisions; the max-abs enc_out error measured on an
# H100 (700 W): 2.7e-3 (fp16) and 2.1e-2 (bf16), padded positions included
ENC_TOL = {"fp16": 5e-3, "bf16": 6e-2}


@functools.lru_cache(maxsize=None)
def _encoder_reference():
    P = R.init_params(S, seed=31, random_bias=True)
    g = torch.Generator().manual_seed(31)
    src = torch.randn(2, 2000, 80, 1, generator=g)
    lens = torch.tensor([2000, 1111])
    src[1, 1111:] = 0.0
    P64 = {k: v.double() for k, v in P.items()}
    with torch.no_grad():
        emb = R.add_position(R.conv_subsample(P64, src.double()))
        padding = R.input_length_to_padding(R.length_after_conv(lens), emb.shape[1], torch.float64)
        enc = R.encoder(P64, emb, padding, S["enc_layers"], S["heads"])
    return P, src, lens, enc, padding


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
def test_inference_encoder_matches_fp64(precision):
    """speech_transformer_s encoder on [2, 2000, 80] with lengths 2000 and 1111 (T' 500 and 278)."""
    P, src, lens, ref, padding = _encoder_reference()
    rt = _runtime(S, precision, P)
    enc, bias = D.encode(rt, dict(src=src, src_length=lens))
    torch.cuda.synchronize()
    diff = (enc.cpu().double() - ref).abs()
    valid = padding == 0
    err, err_pad = float(diff[valid].max()), float(diff[~valid].max())
    print("\n[encoder %s] enc_out max-abs error %.2e on valid positions, %.2e on padded ones, tolerance %.0e" %
          (precision, err, err_pad, ENC_TOL[precision]))
    assert torch.equal(bias.cpu(), R.input_padding_to_bias(padding).float())
    assert err < ENC_TOL[precision] and err_pad < ENC_TOL[precision], (err, err_pad)
