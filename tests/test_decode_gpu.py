"""Inference path (SURVEY.md 8 f1, BASELINE cfg-5): b200st_encode / decode_init / decode_step / greedy_search through the
C ABI vs the oracle's greedy loop (sequence_beam_search with beam_size 1) — token ids must be IDENTICAL."""
import pytest
import torch

from oracle import restatement as R
from tests import parity_utils as U
from neurst_b200 import decode as D
from neurst_b200.models import SpeechTransformer, speech_transformer_hparams

pytestmark = pytest.mark.gpu

SMALL = dict(model="speech", d=64, heads=4, enc_layers=2, dec_layers=2, ffn=128, channels=64, feat=80, in_channels=1, vocab=96)
BOS, EOS, UNK = 94, 95, 93


def _small_case(seed, precision="fp32"):
    P = U.chaotic_decode_params(R.init_params(SMALL, seed=seed, random_bias=True), 4.0, seed)
    g = torch.Generator().manual_seed(seed)
    src = torch.randn(2, 61, 80, 1, generator=g)
    lens = torch.tensor([61, 40])
    src[1, 40:] = 0.0
    rt = U.speech_runtime(SMALL, precision)
    rt.load_parameters(P)
    return P, src, lens, rt


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
@pytest.mark.parametrize("use_graph,persistent", [(True, True), (True, False), (False, False)])
def test_greedy_token_ids_exact_small(seed, use_graph, persistent):
    P, src, lens, rt = _small_case(seed)
    hyp, lp, ln = R.greedy_search(P, SMALL, src, lens, BOS, EOS, UNK, maximum_decode_length=24, extra_decode_length=8)
    ids, logprob, length = D.greedy_search(rt, dict(src=src, src_length=lens), BOS, EOS, UNK, maximum_decode_length=24,
                                           extra_decode_length=8, use_graph=use_graph, persistent=persistent)
    torch.cuda.synchronize()
    assert int(rt.lib.b200st_greedy_used_graph()) == (2 if persistent else int(use_graph))
    assert torch.equal(ids.cpu(), hyp), (ids.cpu().tolist(), hyp.tolist())
    assert torch.equal(length.cpu().long(), ln)
    assert float((logprob.cpu() - lp).abs().max()) < 1e-3


def test_min_length_and_enable_unk():
    P, src, lens, rt = _small_case(1)
    for kw in (dict(minimum_decode_length=6), dict()):
        hyp, _, ln = R.greedy_search(P, SMALL, src, lens, BOS, EOS, None, maximum_decode_length=16, extra_decode_length=0, **kw)
        ids, _, length = D.greedy_search(rt, dict(src=src, src_length=lens), BOS, EOS, None, maximum_decode_length=16,
                                         extra_decode_length=0, enable_unk=True, **kw)
        assert torch.equal(ids.cpu(), hyp) and torch.equal(length.cpu().long(), ln)


def test_cached_steps_match_teacher_forced_forward():
    """symbols_to_logits_fn(symbols, cache, time) of the inference path reproduces, position by position, the logits of the
    fused full forward on the same prefix (encoder_decoder_model.py:243-253 vs :263-279)."""
    P, src, lens, rt = _small_case(2)
    hp = dict(speech_transformer_hparams("speech_transformer_s")["model.params"])
    hp.update({"modality.source.channels": 64, "modality.dim": 64})
    for side in ("encoder", "decoder"):
        hp.update({side + ".num_layers": 2, side + ".hidden_size": 64, side + ".num_attention_heads": 4, side + ".filter_size": 128,
                   side + ".attention_dropout_rate": 0.0, side + ".ffn_dropout_rate": 0.0,
                   side + ".layer_postprocess_dropout_rate": 0.0})
    model = SpeechTransformer.new(hp, {"audio_feature_dim": 80, "audio_feature_channels": 1},
                                  {"vocab_size": 96, "eos_id": EOS, "bos_id": BOS, "unk_id": UNK}, precision="fp32")
    model.load_parameters(P)
    g = torch.Generator().manual_seed(5)
    trg_input = torch.cat([torch.full((2, 1), BOS), torch.randint(0, 93, (2, 6), generator=g)], 1)
    inputs = dict(src=src, src_length=lens, trg_input=trg_input)
    full = model.forward(inputs, is_training=False)                                   # [B, L, V]
    fn_t, init_t = model.get_symbols_to_logits_fn(inputs, is_training=False, is_inference=False)
    assert float((fn_t(init_t["decoder_input"], init_t["decoder_internal_cache"]) - full).abs().max()) == 0.0
    fn, init = model.get_symbols_to_logits_fn(dict(src=src, src_length=lens, trg_input=trg_input[:, 0]), is_training=False,
                                              is_inference=True, decode_padded_length=16)
    assert init["encoder_inputs_maxlen"] == R.length_after_conv(61) and init["eos_id"] == EOS
    cache = init["decoder_internal_cache"]
    for t in range(trg_input.shape[1]):
        logits = fn(trg_input[:, t], cache, t)
        assert float((logits - full[:, t]).abs().max()) < 2e-4, t
    ref_like = cache.as_dict(trg_input.shape[1])
    assert ref_like["layer_0"]["self_attention"]["keys"].shape == (2, 7, 4, 16)


def test_cfg5_greedy_token_ids_exact():
    """BASELINE cfg-5: speech_transformer_s, one utterance [1,2000,80], up to 200 decoding steps, KV caches on the device."""
    cfg = dict(R.CONFIGS["speech_transformer_s"])
    P = U.chaotic_decode_params(R.init_params(cfg, seed=21, random_bias=True), 8.0, 21)
    g = torch.Generator().manual_seed(21)
    src = torch.randn(1, 2000, 80, 1, generator=g)
    lens = torch.tensor([2000])
    V = cfg["vocab"]
    bos, eos, unk = V - 2, V - 1, V - 3
    hyp, lp, ln = R.greedy_search(P, cfg, src, lens, bos, eos, unk, maximum_decode_length=200, extra_decode_length=50)
    rt = U.speech_runtime(cfg, "fp32")
    rt.load_parameters(P)
    ids, logprob, length = D.greedy_search(rt, dict(src=src, src_length=lens), bos, eos, unk, maximum_decode_length=200,
                                           extra_decode_length=50)
    torch.cuda.synchronize()
    n_distinct = len(set(hyp[0].tolist()))
    print("\n[cfg-5] %d steps, %d distinct tokens, oracle logprob %.4f cuda %.4f" % (int(ln[0]), n_distinct, float(lp[0]), float(logprob[0])))
    assert torch.equal(ids.cpu(), hyp), [(i, a, b) for i, (a, b) in enumerate(zip(ids[0].tolist(), hyp[0].tolist())) if a != b][:5]
    assert n_distinct >= 8, "degenerate hypothesis: the test would not exercise the context dependence"
    assert int(length[0]) == int(ln[0]) and abs(float(logprob[0]) - float(lp[0])) < 2e-3 * max(1.0, abs(float(lp[0])))
