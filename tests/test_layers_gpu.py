"""Reference known-answer tests (TF-generated vectors in tests/neurst/**) replayed against the CUDA layer API
(neurst_b200.layers / neurst_b200.models, fp32 precision) — same structure and tolerances as the reference tests."""
import math

import numpy
import pytest
import torch

from neurst_b200.layers import MultiHeadAttention, MultiHeadSelfAttention, TransformerDecoder, TransformerEncoder
from neurst_b200.models import LabelSmoothedCrossEntropy, SpeechTransformer
from oracle import restatement as R
from tests import golden_utils as G

pytestmark = pytest.mark.gpu


def _sq(out, expect):
    return float(((out.detach().cpu().double() - torch.tensor(numpy.asarray(expect))) ** 2).sum())


def test_multihead_attention():
    # tests/neurst/layers/attentions/multi_head_attention_test.py:7-60
    k = G.load("kat_mha_cross")
    layer = MultiHeadAttention(input_depth=1, num_heads=2, num_units=4, output_depth=3, attention_dropout_rate=0.)
    layer.load_parameters({"att.q.kernel": k["shape:(1, 4)"], "att.q.bias": k["shape:(4,)"],
                           "att.kv.kernel": k["shape:(1, 8)"], "att.kv.bias": k["shape:(8,)"],
                           "att.out.kernel": k["shape:(4, 3)"], "att.out.bias": k["shape:(3,)"]})
    output = layer(G.t(k["var:query"]), G.t(k["var:memory"]), is_training=False)
    assert _sq(output, k["expect:0"]) < 1e-9


def test_multiheadself_attention():
    # multi_head_attention_test.py:63-111 (additive 2-D bias)
    k = G.load("kat_mha_self")
    layer = MultiHeadSelfAttention(input_depth=2, num_heads=2, num_units=4, output_depth=3, attention_dropout_rate=0.)
    layer.load_parameters({"att.qkv.kernel": k["shape:(2, 12)"], "att.qkv.bias": k["shape:(12,)"],
                           "att.out.kernel": k["shape:(4, 3)"], "att.out.bias": k["shape:(3,)"]})
    output = layer(G.t(k["var:query"]), bias=G.t(k["var:bias"]), is_training=False)
    assert _sq(output, k["expect:0"]) < 1e-9


def test_multiheadself_attention_under_dec():
    # multi_head_attention_test.py:114-186 (decode step with the concat KV cache, called twice)
    k = G.load("kat_mha_self_cache")
    layer = MultiHeadSelfAttention(input_depth=2, num_heads=2, num_units=4, output_depth=3, attention_dropout_rate=0.)
    layer.load_parameters({"att.qkv.kernel": k["shape:(2, 12)"], "att.qkv.bias": k["shape:(12,)"],
                           "att.out.kernel": k["shape:(4, 3)"], "att.out.bias": k["shape:(3,)"]})
    cache = {"keys": G.t(k["dict:keys"]).reshape(1, 2, 2, 2).cuda(), "values": G.t(k["dict:values"]).reshape(1, 2, 2, 2).cuda()}
    query = G.t(k["var:query"])
    layer(query, cache=cache, is_training=False)
    output = layer(query, cache=cache, is_training=False)
    assert _sq(output, k["expect:0"]) < 1e-9
    assert _sq(cache["keys"].reshape(1, 4, 4), k["expect:1"]) < 1e-9
    assert _sq(cache["values"].reshape(1, 4, 4), k["expect:2"]) < 1e-9


def test_attention_argument_errors():
    with pytest.raises(ValueError):
        MultiHeadAttention(input_depth=4, num_heads=3, num_units=4)


def test_transformer_encoder():
    # tests/neurst/layers/encoders/transformer_encoder_test.py:21-122 (assert_equal_numpy: L2 < 1e-6)
    k = G.load("kat_encoder")
    encoder = TransformerEncoder(num_layers=1, num_attention_heads=2, hidden_size=4, filter_size=16, attention_dropout_rate=0.1,
                                 ffn_dropout_rate=0.1, layer_postprocess_dropout_rate=0.1)
    cfg = dict(model="none", d=4, heads=2, enc_layers=1, dec_layers=0, ffn=16, vocab=1)
    encoder.load_parameters(G.kat_params(k, cfg, "enc"))
    out = encoder(G.t(k["var:inputs"]), G.t(k["var:input_padding"]), is_training=False)
    assert math.sqrt(_sq(out, k["expect:0"])) < 1e-6


def test_transformer_decoder():
    # tests/neurst/layers/decoders/transformer_decoder_test.py:20-181: train mode, cached inference step, cache contents
    from tests.test_oracle import _decoder_step_input
    k = G.load("kat_decoder")
    decoder = TransformerDecoder(num_layers=1, num_attention_heads=2, hidden_size=4, filter_size=16, attention_dropout_rate=0.1,
                                 ffn_dropout_rate=0.1, layer_postprocess_dropout_rate=0.1)
    cfg = dict(model="none", d=4, heads=2, enc_layers=0, dec_layers=1, ffn=16, vocab=1)
    decoder.load_parameters(G.kat_params(k, cfg, "dec"))
    encoder_outputs, encoder_inputs_padding = G.t(k["var:encoder_outputs"]), G.t(k["var:encoder_inputs_padding"])
    cache = decoder.create_decoding_internal_cache(encoder_outputs, encoder_inputs_padding)
    assert _sq(decoder(G.t(k["var:decoder_inputs"]), cache, is_training=False), k["expect:0"]) < 1e-9
    # for inference
    cache = decoder.create_decoding_internal_cache(encoder_outputs, encoder_inputs_padding, is_inference=True)
    step = decoder(G.t(_decoder_step_input()), cache, is_training=False)
    assert _sq(step, k["expect:1"]) < 1e-9
    sa = cache["decoding_states"]["layer_0"]["self_attention"]
    assert _sq(sa["keys"].reshape(2, 1, 4), k["expect:2"]) < 1e-9
    assert _sq(sa["values"].reshape(2, 1, 4), k["expect:3"]) < 1e-9


def test_transformer_decoder_without_cross_attention():
    """with_encoder_decoder_attention=False: every layer is self-attention -> FFN, against the fp64 decoder without memory."""
    torch.manual_seed(0)
    cfg = dict(model="none", d=16, heads=4, enc_layers=0, dec_layers=2, ffn=24, vocab=1)
    P = R.init_params(cfg, seed=9, random_bias=True)
    decoder = TransformerDecoder(num_layers=2, num_attention_heads=4, hidden_size=16, filter_size=24,
                                 with_encoder_decoder_attention=False)
    decoder.load_parameters(P)
    x = torch.randn(3, 7, 16)
    out = decoder(x, decoder.create_decoding_internal_cache(None, None), is_training=False).cpu().double()
    expect = R.decoder({k: v.double() for k, v in P.items()}, x.double(), None, None, 2, 4)
    assert float((out - expect).abs().max()) < 1e-5


def test_incremental_decode_matches_full_decode():
    """cached steps reproduce the full (training-mode) decoder outputs position by position."""
    torch.manual_seed(0)
    cfg = dict(model="none", d=16, heads=4, enc_layers=0, dec_layers=2, ffn=24, vocab=1)
    P = R.init_params(cfg, seed=5, random_bias=True)
    decoder = TransformerDecoder(num_layers=2, num_attention_heads=4, hidden_size=16, filter_size=24)
    decoder.load_parameters(P)
    mem, pad = torch.randn(2, 5, 16), torch.tensor([[0., 0, 0, 0, 0], [0, 0, 0, 1, 1]])
    x = torch.randn(2, 4, 16)
    full = decoder(x, decoder.create_decoding_internal_cache(mem, pad), is_training=False).cpu()
    cache = decoder.create_decoding_internal_cache(mem, pad, is_inference=True)
    for t in range(4):
        step = decoder(x[:, t], cache, is_training=False).cpu()
        assert float((step - full[:, t]).abs().max()) < 1e-5


def test_speech_transformer_model_api_and_criterion():
    """SpeechTransformer.new(args, src_meta, trg_meta) with the reference's flat args; logits vs the reference-PT fixture;
    LabelSmoothedCrossEntropy through the reference call contract vs the oracle."""
    z, P, cfg = G.refpt_case("refpt_speech_toy")
    args = SpeechTransformer.build_model_args_by_name("speech_transformer_toy")["model.params"]
    model = SpeechTransformer.new(args, {"audio_feature_dim": 80, "audio_feature_channels": 1},
                                  {"vocab_size": cfg["vocab"], "eos_id": 11, "bos_id": 10, "unk_id": 9}, precision="fp32")
    model.load_parameters(P)
    inputs = {"src": G.t(z["src"]), "src_length": torch.tensor(z["src_length"]), "trg_input": torch.tensor(z["trg_input"])}
    logits = model(inputs, is_training=False)
    assert float((logits.cpu() - G.t(z["logits"])).abs().max()) < 1e-4
    trg = torch.randint(0, cfg["vocab"], tuple(z["trg_input"].shape))
    trg_length = torch.tensor([5, 3, 1])
    crit = LabelSmoothedCrossEntropy({"label_smoothing": 0.1})
    nll, n_samples, n_tokens = crit({"trg": trg, "trg_length": trg_length}, logits)
    onll, ons, ont = R.label_smoothed_ce(logits.cpu().double(), trg, trg_length, 0.1)
    assert float((nll.cpu().double() - onll).abs().max()) < 1e-4
    assert n_tokens.cpu().tolist() == ont.tolist() and n_samples.cpu().tolist() == ons.tolist()
    assert abs(float(crit.reduce_loss({"trg": trg, "trg_length": trg_length}, logits)) - float(onll.sum() / ont.sum())) < 1e-4
