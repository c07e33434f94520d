"""Decoding steps of more than 8 rows (the wide step: 16-bit shadow weights on the tensor cores, up to 256 rows) against the
fp64 decoder on the same rounded weights, with the tolerances and search guards of tests/test_decode_shadow_gpu.py: the
wide step keeps the shadow contract (16-bit weights, fp32 activations, caches and accumulation), so the same oracle and the
same tolerances apply.  Also: bit-reproducibility, independence of a row from the rest of its batch, the limits, and the
recipes' `batch_size` in `predict`."""
import functools

import pytest
import torch

from neurst_b200 import decode as D
from neurst_b200 import lib as L
from oracle import restatement as R
from tests import parity_utils as U
from tests.test_beam_search_gpu import _check
from tests.test_decode_shadow_gpu import (DIMS, DTYPES, SHADOW_READ, SMALL, STEP_TOL, _cache, _chaotic, _runtime, _step_inputs,
                                          decoder_search, ragged_memory, shadow_rounded, teacher_forced_logits)

pytestmark = pytest.mark.gpu

N_POS = 24
EFFECT_ROWS = 64        # the single-tensor effects are a property of the weights: measured on the first 64 rows
# speech_transformer_m (d 512, 8 heads): there the output projections (K = d = 512) are split along K and the tied logits
# (K = 512, N = 8192) are not.  CPU, the test's 64 rows, Tm 500, seed 0: fp32 arithmetic noise 6.6e-6 (fp16 weights) /
# 6.8e-6 (bf16); smallest single-tensor effect (cross.q.kernel) 1.08e-4 / 9.8e-4.  Measured on an H100 (700 W): 1.7e-5
# (fp16) and 1.4e-5 (bf16), the bit-reproducible step's fixed value for these inputs.
DIMS_WIDE = dict(DIMS, m=dict(R.CONFIGS["speech_transformer_m"]))
STEP_TOL_WIDE = {**STEP_TOL, ("m", "fp16"): 1.8e-5, ("m", "bf16"): 1.3e-4}


@functools.lru_cache(maxsize=None)
def _step_reference(dims, B, Tm, precision):
    cfg, dt = DIMS_WIDE[dims], DTYPES[precision]
    P, memory, bias, ids = _step_inputs(cfg, B, Tm, N_POS, seed=0)
    ref = teacher_forced_logits(shadow_rounded(P, dt), cfg, memory, bias, ids)
    m, b, i = memory[:EFFECT_ROWS], bias[:EFFECT_ROWS], ids[:EFFECT_ROWS]
    effect = {k: float((teacher_forced_logits(shadow_rounded(P, dt, keep=k), cfg, m, b, i) - ref[:EFFECT_ROWS]).abs().max())
              for k in SHADOW_READ}
    return P, memory, bias, ids, ref, effect


def _step_logits(rt, memory, bias, ids):
    cache = _cache(rt, memory, bias, N_POS)
    return torch.stack([D.decoder_step_logits(rt, ids[:, t], cache, t) for t in range(N_POS)], 1)


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("dims,B,Tm", [("small", 64, 61), ("small", 256, 61), ("s", 64, 500), ("s", 256, 500), ("m", 64, 500)])
def test_wide_step_logits_match_rounded_fp64_decoder(dims, B, Tm, precision):
    P, memory, bias, ids, ref, effect = _step_reference(dims, B, Tm, precision)
    tol = STEP_TOL_WIDE[dims, precision]
    weakest = min(effect, key=effect.get)
    assert tol <= effect[weakest] / 5, "tolerance %.1e does not resolve %s (effect %.1e)" % (tol, weakest, effect[weakest])
    rt = _runtime(DIMS_WIDE[dims], precision, P)
    out = _step_logits(rt, memory, bias, ids)
    err = float((out.cpu().double() - ref).abs().max())
    print("\n[wide step %s B=%d Tm=%d %s] logits max-abs error %.2e, tolerance %.1e, smallest single-tensor effect %.2e (%s)" %
          (dims, B, Tm, precision, err, tol, effect[weakest], weakest))
    assert err < tol, err


# ---- greedy search on 64 utterances ------------------------------------------------------------------------------------------
# small dims, chaotic gain 4, Tm 61.  Over 64 utterances the fp64 search meets near-ties more often than over 8: at 24 steps
# none of seeds 1-8 kept gap >= 10 x noise for both precisions; at 12 steps seed 2 does (CPU: fp16 gap 2.2e-3 / noise
# 8.1e-5, bf16 1.4e-3 / 5.9e-5, 44 distinct tokens).
GREEDY_SEED, GREEDY_LEN = 2, 12


@functools.lru_cache(maxsize=None)
def _greedy_reference(B, precision):
    P, memory, bias = _chaotic("small", B, 61, 4.0, GREEDY_SEED)
    Pr = shadow_rounded(P, DTYPES[precision])
    ref = decoder_search(Pr, SMALL, memory, bias, 94, 95, 93, 1, 0.0, maximum_decode_length=GREEDY_LEN, extra_decode_length=8)
    inputs = torch.cat([torch.full((B, 1), 94), ref["hypotheses"][:, :ref["steps"] - 1]], 1)
    l64 = teacher_forced_logits(Pr, SMALL, memory, bias, inputs)
    noise = float((teacher_forced_logits(Pr, SMALL, memory, bias, inputs, torch.float32).double() - l64).abs().max())
    return ref, noise


def _greedy(precision, memory, bias, P, use_graph=True, persistent=True):
    rt = _runtime(SMALL, precision, P)
    out = D.greedy_search(rt, None, 94, 95, 93, maximum_decode_length=GREEDY_LEN, extra_decode_length=8, use_shadow=True,
                          use_graph=use_graph, persistent=persistent, cache=_cache(rt, memory, bias, GREEDY_LEN))
    torch.cuda.synchronize()
    return rt, out


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("use_graph", [True, False])
def test_wide_greedy_token_ids_exact(precision, use_graph):
    B = 64
    ref, noise = _greedy_reference(B, precision)
    hyp = ref["hypotheses"]
    n_distinct = len(set(hyp[:, :ref["steps"]].reshape(-1).tolist()))
    assert ref["gap"] >= 10 * noise, "near-tie in the oracle's search (gap %.2e, noise %.2e): pick another case" % (ref["gap"], noise)
    assert n_distinct >= 8, "degenerate hypothesis: the test would not exercise the context dependence"
    P, memory, bias = _chaotic("small", B, 61, 4.0, GREEDY_SEED)
    # use_graph asks for the persistent kernel, which does not exist above 8 rows: the captured graph runs instead
    rt, (ids, logprob, length) = _greedy(precision, memory, bias, P, use_graph=use_graph, persistent=True)
    mode = int(rt.lib.b200st_greedy_used_graph())
    print("\n[wide greedy B=%d %s mode %d] %d steps, %d distinct tokens, gap %.2e, noise %.2e" %
          (B, precision, mode, ref["steps"], n_distinct, ref["gap"], noise))
    assert mode == int(use_graph)
    assert torch.equal(ids.cpu(), hyp), [(i, a, b) for i, (a, b) in enumerate(zip(ids.cpu().view(-1).tolist(), hyp.view(-1).tolist()))
                                         if a != b][:5]
    assert torch.equal(length.cpu().long(), ref["length"])
    assert float((logprob.cpu() - ref["logprob"]).abs().max()) < 1e-3


# ---- beam search: 16 x 4 and 64 x 4 rows -------------------------------------------------------------------------------------
# utterances -> (seed, maximum_decode_length): the smallest oracle gap over both alphas (CPU) is 1.7e-4 for 16 x 4 at 24
# steps and 1.8e-4 for 64 x 4 at 8 steps (at 12 and 24 steps no seed of 1-11 stayed above the 1e-4 guard for 64 utterances)
BEAM_CASE = {16: (10, 24), 64: (2, 8)}


@functools.lru_cache(maxsize=None)
def _beam_reference(B, alpha):
    seed, max_len = BEAM_CASE[B]
    P, memory, bias = _chaotic("small", B, 61, 4.0, seed)
    return decoder_search(shadow_rounded(P, torch.float16), SMALL, memory, bias, 94, 95, 93, 4, alpha, maximum_decode_length=max_len,
                          extra_decode_length=8)


def _beam(B, alpha, use_graph=True, memory=None, bias=None):
    seed, max_len = BEAM_CASE[B]
    P, mem, b = _chaotic("small", B, 61, 4.0, seed)
    rt = _runtime(SMALL, "fp16", P)
    out = D.beam_search(rt, None, 94, 95, 93, beam_size=4, length_penalty=alpha, maximum_decode_length=max_len, extra_decode_length=8,
                        use_shadow=True, use_graph=use_graph,
                        cache=_cache(rt, mem if memory is None else memory, b if bias is None else bias, max_len, beam=4))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("B", [16, 64])
@pytest.mark.parametrize("alpha", [0.6, -1.0])
@pytest.mark.parametrize("use_graph", [True, False])
def test_wide_beam_token_ids_exact(B, alpha, use_graph):
    ref = _beam_reference(B, alpha)
    ids, scores, logprob, length = _beam(B, alpha, use_graph)
    _check(ref, ids, scores, length)
    assert torch.allclose(logprob.cpu(), ref["logprob"], rtol=1e-4, atol=1e-5)


def test_wide_beam_token_ids_exact_speech_transformer_s():
    """speech_transformer_s, 16 utterances (Tm <= 500, ragged) x beam 4, 1/len scores, fp16 shadow.  With 16 utterances x
    4 x 8192 candidates the oracle met near-ties within 64 steps (seed 3: gap 1.9e-6); at 16 steps seed 3 (gain 2.5) has a
    gap of 1.03e-4, above the 1e-4 guard."""
    S = DIMS["s"]
    V, steps = S["vocab"], 16
    P = U.chaotic_decode_params(R.init_params(S, seed=3, random_bias=True), 2.5, 3)
    memory, bias = ragged_memory(S, 16, 500, 103)
    ref = decoder_search(shadow_rounded(P, torch.float16), S, memory, bias, V - 2, V - 1, V - 3, 4, -1.0, maximum_decode_length=steps,
                         extra_decode_length=50)
    rt = _runtime(S, "fp16", P)
    ids, scores, _, length = D.beam_search(rt, None, V - 2, V - 1, V - 3, beam_size=4, length_penalty=-1.0, maximum_decode_length=steps,
                                           extra_decode_length=50, use_shadow=True, cache=_cache(rt, memory, bias, steps, beam=4))
    torch.cuda.synchronize()
    print("\n[wide beam s 16x4 fp16] %d steps, gap %.2e" % (ref["steps"], ref["gap"]))
    _check(ref, ids, scores, length)


def test_wide_beam_deep_positions_teacher_forced_logprob():
    """64 utterances x beam 4 over 24 steps, every beam returned.  Over 64 utterances the fp64 search always meets a near-tie
    somewhere within 16 steps (no seed of 1-19 at gains 6, 8 and 12 kept the 1e-4 gap), so token ids cannot be compared with
    it; instead each hypothesis is run through the fp64 decoder on the rounded weights and its log-probabilities, summed up to
    its length, must give the accumulated log-probability the search reports.  A wrong ancestry slot at any position (the
    self-attention cache read far back through the reordered beams) changes that context and the sum."""
    B, beam, max_len, seed = 64, 4, 24, 1
    P, memory, bias = _chaotic("small", B, 61, 4.0, seed)
    rt = _runtime(SMALL, "fp16", P)
    ids, scores, logprob, length = D.beam_search(rt, None, 94, 95, 93, beam_size=beam, top_k=beam, length_penalty=0.6,
                                                 maximum_decode_length=max_len, extra_decode_length=8, use_shadow=True,
                                                 cache=_cache(rt, memory, bias, max_len, beam=beam))
    torch.cuda.synchronize()
    ids, logprob, length = ids.cpu(), logprob.cpu().double(), length.cpu().long()
    n = ids.shape[0]
    inputs = torch.cat([torch.full((n, 1), 94), ids[:, :-1]], 1)
    z = teacher_forced_logits(shadow_rounded(P, torch.float16), SMALL, memory.repeat_interleave(beam, 0),
                              bias.repeat_interleave(beam, 0), inputs)
    tok = torch.log_softmax(z, -1).gather(2, ids.unsqueeze(2))[..., 0]
    mask = torch.arange(max_len).unsqueeze(0) < length.unsqueeze(1)
    ref = (tok * mask).sum(1)
    err = float((ref - logprob).abs().max())
    print("\n[wide beam 64x4 deep] lengths %d..%d, %d distinct tokens, max |logprob - teacher-forced fp64| %.2e" %
          (int(length.min()), int(length.max()), len(set(ids.view(-1).tolist())), err))
    assert int(length.max()) >= 16, "hypotheses too short to reach deep positions"
    assert err < 1e-3, err
    assert bool((scores.cpu().view(B, beam)[:, :-1] >= scores.cpu().view(B, beam)[:, 1:]).all())


# ---- determinism and row independence ----------------------------------------------------------------------------------------
def test_wide_step_is_bit_reproducible():
    P, memory, bias, ids = _step_inputs(SMALL, 64, 61, N_POS, seed=0)
    rt = _runtime(SMALL, "fp16", P)
    a, b = _step_logits(rt, memory, bias, ids), _step_logits(rt, memory, bias, ids)
    assert torch.equal(a, b)
    r1, r2 = _beam(16, 0.6), _beam(16, 0.6)
    assert all(torch.equal(x, y) for x, y in zip(r1, r2))
    Pg, mg, bg = _chaotic("small", 64, 61, 4.0, GREEDY_SEED)
    g1, g2 = _greedy("fp16", mg, bg, Pg)[1], _greedy("fp16", mg, bg, Pg)[1]
    assert all(torch.equal(x, y) for x, y in zip(g1, g2))


def test_wide_rows_do_not_depend_on_their_batch():
    """16 utterances decoded as rows 0..15 of a 16-utterance batch and as rows 48..63 of a 64-utterance batch."""
    P, memory, bias = _chaotic("small", 64, 61, 4.0, GREEDY_SEED)
    first = _beam(16, 0.6, memory=memory[:16], bias=bias[:16])
    moved = _beam(16, 0.6, memory=torch.cat([memory[16:], memory[:16]]), bias=torch.cat([bias[16:], bias[:16]]))
    ids, scores, _, length = first
    ids2, scores2, _, length2 = (x[48:] for x in moved)
    bit_equal = torch.equal(scores, scores2)
    print("\n[row independence] beam scores bit-equal: %s, max relative difference %.2e" %
          (bit_equal, float(((scores - scores2).abs() / scores.abs()).max())))
    assert torch.equal(ids, ids2) and torch.equal(length, length2)
    assert torch.allclose(scores, scores2, rtol=1e-6, atol=0.0)


# ---- limits ------------------------------------------------------------------------------------------------------------------
def test_wide_limits():
    P, memory, bias = _chaotic("small", 64, 61, 4.0, GREEDY_SEED)
    rt = _runtime(SMALL, "fp16", P)
    big = torch.cat([memory] * 4)
    cache = D.create_decoding_cache(rt, big.cuda(), torch.cat([bias] * 4).cuda(), 4, use_shadow=True)
    cache.state.B = 257                                           # past B200ST_DECODE_MAX_ROWS: refused before any launch
    with pytest.raises(L.B200STError, match="1..256"):
        D.decoder_step_logits(rt, torch.zeros(257, dtype=torch.long), cache, 0)
    with pytest.raises(L.B200STError, match="rows"):
        D.create_decoding_cache(rt, torch.cat([big, big[:1]]).cuda(), torch.cat([bias] * 4 + [bias[:1]]).cuda(), 4, use_shadow=True)
    with pytest.raises(L.B200STError, match="beam_size"):
        D.beam_search(rt, None, 94, 95, 93, beam_size=9, maximum_decode_length=8, extra_decode_length=0, use_shadow=True,
                      cache=_cache(rt, memory[:2], bias[:2], 8, beam=9))
    rt32 = _runtime(SMALL, "fp32", P)
    with pytest.raises(L.B200STError, match="rows"):                       # 3 x 4 rows with the fp32 weights
        D.create_decoding_cache(rt32, memory[:3].cuda(), bias[:3].cuda(), 24, beam=4)
    with pytest.raises(L.B200STError, match="rows"):
        D.create_decoding_cache(rt32, memory[:12].cuda(), bias[:12].cuda(), 24)
    torch.cuda.synchronize()


# ---- predict with the recipes' batch_size ------------------------------------------------------------------------------------
def test_predict_batch_size(tmp_path, monkeypatch):
    import os

    from neurst_b200 import cli
    from neurst_b200.models import SpeechTransformer
    from tests import test_cli as T
    T._write_dataset(tmp_path, vocab=93)
    y = T._write_yaml(tmp_path, data=str(tmp_path / "train.tfrecords"), n_tokens=93)
    model_dir = str(tmp_path / "model")
    tiny = ["--model.params.encoder.num_layers", "2", "--model.params.decoder.num_layers", "2",
            "--model.params.encoder.hidden_size", "128", "--model.params.decoder.hidden_size", "128", "--model.params.modality.dim", "128",
            "--model.params.encoder.num_attention_heads", "2", "--model.params.decoder.num_attention_heads", "2",
            "--model.params.encoder.filter_size", "256", "--model.params.decoder.filter_size", "256",
            "--model.params.modality.source.channels", "64"]
    common = ["--model_dir", model_dir, "--task.params.batch_size", "3000", "--task.params.max_src_len", "400",
              "--task.params.max_trg_len", "24", "--task.params.min_src_bucket_boundary", "128",
              "--task.params.experimental_frame_transcript_ratio", "20", "--save_checkpoint_steps", "3", "--summary_steps", "2"] + tiny
    assert cli.main(["--config_paths", y] + common + ["--train_steps", "4"])["global_step"] == 4
    one = tmp_path / "one"
    one.mkdir()
    os.link(str(tmp_path / "train.tfrecords-00000-of-00003"), str(one / "train.tfrecords-00000-of-00001"))
    calls = []
    orig = SpeechTransformer.beam_search

    def counted(self, inputs, **kw):
        calls.append((int(inputs["src"].shape[0]), bool(kw.get("use_shadow"))))
        return orig(self, inputs, **kw)

    monkeypatch.setattr(SpeechTransformer, "beam_search", counted)
    texts = {}
    for bs in (None, 16, 4):
        paths = y
        if bs is not None:
            extra = tmp_path / ("bs%d.yml" % bs)
            extra.write_text("batch_size: %d\n" % bs)
            paths = y + "," + str(extra)
        out = str(tmp_path / ("hyp_%s.txt" % bs))
        calls.clear()
        res = cli.main(["--config_paths", paths] + common + [
            "--entry.class", "predict", "--output_file", out, "--dataset.params.data_path", str(one / "train.tfrecords"),
            "--search_method", "beam_search", "--search_method.params.beam_size", "4", "--search_method.params.length_penalty", "-1",
            "--search_method.params.maximum_decode_length", "12"])
        assert res["n_hypotheses"] == 70
        texts[bs] = open(out, encoding="utf-8").read()
        if bs is None:
            assert len(calls) == 35 and not any(s for _, s in calls), calls          # 8 // beam 4 = 2 utterances per call, as before
        else:
            assert len(calls) == -(-70 // bs) and all(s for _, s in calls) and calls[0][0] == bs, calls
    assert texts[16] == texts[4]
    torch.cuda.synchronize()
