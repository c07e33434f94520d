"""Host-side mirror of the reference model / criterion API on top of libb200st.

  SpeechTransformer          neurst/models/speech_transformer.py:27-280  (PT twin neurst_pt/models/speech_transformer.py)
  Transformer                neurst/models/transformer.py:27-260         (cfg-1 plumbing model)
  WaitkTransformer           neurst/models/waitk_transformer.py:23-144   (simultaneous translation, offline wait-k)
  EncoderDecoderEnsembleModel  neurst/models/encoder_decoder_ensemble_model.py  (generation only)
  LabelSmoothedCrossEntropy  neurst/criterions/label_smoothed_cross_entropy.py:26-157

`Model.new(args, src_meta, trg_meta)` takes the reference's flat `model.params` dict (the yaml / hparams_set keys);
`forward(inputs, is_training)` takes the reference's input dict (neurst/tasks/speech2text.py:135-161) and returns
logits [B, L, V].  Training uses the fused `forward_backward(inputs)` entry (loss + all gradients in one C call).
"""
import re

import torch

from neurst_b200 import lib as L
from neurst_b200.runtime import Runtime, make_config


def speech_transformer_hparams(name):
    """neurst/models/speech_transformer.py:190-282 (`build_model_args_by_name`)."""
    table = {
        "speech_transformer_toy": dict(dmodel=8, heads=2, enc=2, dec=2, ffn=10, channels=5),
        "speech_transformer_s": dict(dmodel=256, heads=4, enc=12, dec=6, ffn=2048, channels=256),
        "speech_transformer_m": dict(dmodel=512, heads=8, enc=12, dec=6, ffn=2048, channels=256),
        "speech_transformer_l": dict(dmodel=1024, heads=16, enc=12, dec=6, ffn=4096, channels=512),
    }
    if name not in table:
        return None
    t = table[name]
    dmodel, rate = t["dmodel"], 0.1
    params = {
        "modality.source.kernel_size": 3, "modality.source.strides": 2, "modality.source.channels": t["channels"],
        "modality.source.layer_norm": True, "modality.dim": dmodel, "modality.share_embedding_and_softmax_weights": True,
        "modality.timing": "sinusoids",
    }
    for side, nl in (("encoder", t["enc"]), ("decoder", t["dec"])):
        params.update({side + ".num_layers": nl, side + ".hidden_size": dmodel, side + ".num_attention_heads": t["heads"],
                       side + ".filter_size": t["ffn"], side + ".attention_dropout_rate": rate,
                       side + ".attention_type": "dot_product", side + ".ffn_activation": "relu",
                       side + ".ffn_dropout_rate": rate, side + ".layer_postprocess_dropout_rate": rate})
    return {
        "model.class": "SpeechTransformer", "model.params": params,
        "optimizer.class": "Adam", "optimizer.params": {"epsilon": 1.e-9, "beta_1": 0.9, "beta_2": 0.98},
        "lr_schedule.class": "noam",
        "lr_schedule.params": {"initial_factor": 5.0 if dmodel > 256 else 3.5, "end_factor": 2.0 if dmodel > 256 else 1.5,
                               "dmodel": dmodel, "warmup_steps": 25000, "start_decay_at": 50000, "decay_steps": 50000},
    }


def transformer_hparams(name):
    """neurst/models/transformer.py:136-240 (`Transformer.build_model_args_by_name`): the text presets and the
    `transformer_<d>_<n>e_<m>d[_<h>h][_dp0.x]` pattern, with their Adam and noam defaults; None for other names."""
    table = {"transformer_toy": (8, 2, 2, 2, 10, 0.1), "transformer_base": (512, 8, 6, 6, 2048, 0.1),
             "transformer_s": (256, 4, 6, 6, 2048, 0.1), "transformer_big": (1024, 16, 6, 6, 4096, 0.3),
             "transformer_big_dp01": (1024, 16, 6, 6, 4096, 0.1)}
    if name in table:
        dmodel, heads, enc, dec, ffn, rate = table[name]
    elif re.match(r"^transformer_\d+_\d+e_\d+d(_\d+h)?(_dp0\.\d+)?$", str(name)):
        eles = name.split("_")
        dmodel, enc, dec, heads, idx = int(eles[1]), int(eles[2][:-1]), int(eles[3][:-1]), 8, 4
        if len(eles) > idx and eles[idx][-1] == "h":
            heads = int(eles[idx][:-1])
            idx += 1
        if dmodel % heads != 0:
            raise ValueError("Invalid arguments in hparams_set: dimension({}) must be divisible by head({})".format(dmodel, heads))
        rate = float(eles[idx][2:]) if len(eles) > idx and eles[idx][0:2] == "dp" else 0.1
        ffn = dmodel * 4
    else:
        return None
    params = {"modality.share_source_target_embedding": False, "modality.share_embedding_and_softmax_weights": True,
              "modality.dim": dmodel, "modality.timing": "sinusoids"}
    for side, nl in (("encoder", enc), ("decoder", dec)):
        params.update({side + ".num_layers": nl, side + ".hidden_size": dmodel, side + ".num_attention_heads": heads,
                       side + ".filter_size": ffn, side + ".attention_dropout_rate": rate,
                       side + ".attention_type": "dot_product", side + ".ffn_activation": "relu",
                       side + ".ffn_dropout_rate": rate, side + ".post_normalize": False,
                       side + ".layer_postprocess_dropout_rate": rate})
    return {
        "model.class": "Transformer", "model.params": params,
        "optimizer.class": "Adam", "optimizer.params": {"epsilon": 1.e-9, "beta_1": 0.9, "beta_2": 0.98},
        "lr_schedule.class": "noam", "lr_schedule.params": {"initial_factor": 1.0, "dmodel": dmodel, "warmup_steps": 4000},
    }


def waitk_transformer_hparams(name):
    """neurst/models/waitk_transformer.py:75-84: `waitk_transformer_<name>` and `waitktransformer_<name>` are the Transformer
    preset `<name>` with model.class WaitkTransformer and a monotonic encoder; None for other names."""
    name = str(name)
    args = None
    if name.startswith("waitk_transformer_"):
        args = transformer_hparams(name[6:])
    elif name.startswith("waitktransformer_"):
        args = transformer_hparams(name[5:])
    if args is not None:
        args["model.class"] = "WaitkTransformer"
        args["model.params"]["encoder.attention_monotonic"] = True
    return args


def parse_wait_k(value):
    """WaitkTranslation's `wait_k` (waitk_translation.py:23-31): an int, a list of ints, or a YAML string of either."""
    import yaml
    k = yaml.safe_load(value) if isinstance(value, str) else value
    if isinstance(k, bool) or not (isinstance(k, int) or (isinstance(k, (list, tuple)) and k)):
        raise ValueError("wait_k must be an int or a non-empty list of ints, got %r" % (value,))
    ks = list(k) if isinstance(k, (list, tuple)) else [k]
    for x in ks:
        if isinstance(x, bool) or not isinstance(x, int) or x < 1:
            raise ValueError("wait_k must be >= 1 (a lag of k source tokens), got %r" % (value,))
    return ks if isinstance(k, (list, tuple)) else k


def _model_flags(speech):
    """(name, python type, default, help) of every `model.params` key — the flag list of the reference's
    `class_or_method_args()` (neurst_pt/models/speech_transformer.py:35-106, neurst/models/transformer.py:45-120):
    same names and defaults, so `registry.build_x` fills a user's partial params dict exactly as for the reference class."""
    fl = [("modality.share_embedding_and_softmax_weights", bool, False,
           "Whether to share the target embedding table and softmax weights."),
          ("modality.dim", int, None, "The default embedding dimension for both source and target side."),
          ("modality.source.dim", int, None, "The source-side embedding dimension, or `modality.dim` if not provided."),
          ("modality.target.dim", int, None, "The target-side embedding dimension, or `modality.dim` if not provided."),
          ("modality.timing", str, None, "The positional encoding of both source and target side."),
          ("modality.source.timing", str, None, "The source-side positional encoding, or `modality.timing`."),
          ("modality.target.timing", str, None, "The target-side positional encoding, or `modality.timing`.")]
    if speech:
        fl += [("modality.source.kernel_size", int, 3, "The kernel size for the first two conv layer"),
               ("modality.source.strides", int, 2, "The stride size for the first two conv layer"),
               ("modality.source.channels", int, 256, "The channels for the first two conv layer"),
               ("modality.source.layer_norm", bool, False, "Whether to apply layer norm in convolution layers.")]
    else:
        fl += [("modality.share_source_target_embedding", bool, False,
                "Whether to share source and target embedding table."),
               ("encoder.attention_monotonic", bool, False,
                "Whether to apply a triangle mask to make the encoder self-attention monotonic (causal).")]
    for side in ("encoder", "decoder"):
        fl += [(side + ".num_layers", int, None, "The number of stacking layers of the %s." % side),
               (side + ".hidden_size", int, None, "The number of hidden units of the %s." % side),
               (side + ".num_attention_heads", int, None, "The number of attention heads of the %s." % side),
               (side + ".filter_size", int, None, "The filter size of the %s ffn." % side),
               (side + ".ffn_activation", str, "relu", "The activation function of the %s ffn layer." % side),
               (side + ".attention_dropout_rate", float, 0., "The dropout rate of the %s attention layers." % side),
               (side + ".attention_type", str, "dot_product", "The type of the attention function of the %s." % side),
               (side + ".ffn_dropout_rate", float, 0., "The dropout rate of the %s ffn layer." % side),
               (side + ".layer_postprocess_dropout_rate", float, 0., "The dropout rate of each layer's post process."),
               (side + ".layer_postprocess_epsilon", float, 1e-6, "The epsilon for layer normalization in the %s." % side)]
    return fl


def _check_supported(args, speech):
    def same(a, b):
        return args.get(a) == args.get(b)
    for k in ("num_layers",):
        pass
    if not (same("encoder.hidden_size", "decoder.hidden_size") and same("encoder.num_attention_heads",
                                                                       "decoder.num_attention_heads")
            and same("encoder.filter_size", "decoder.filter_size")):
        raise NotImplementedError("libb200st needs identical encoder/decoder hidden, heads and filter sizes")
    for k in ("modality.dim", "modality.source.dim", "modality.target.dim"):
        if args.get(k) is not None and args.get(k) != args.get("encoder.hidden_size"):
            raise NotImplementedError("%s must equal the hidden size" % k)
    if args.get("modality.dim") is None and args.get("modality.target.dim") is None:
        raise NotImplementedError("modality.dim must be given (and equal the hidden size)")
    for side in ("source", "target"):
        if (args.get("modality.%s.timing" % side) or args.get("modality.timing")) != "sinusoids":
            raise NotImplementedError("only sinusoid position signals are supported")
    if not args.get("modality.share_embedding_and_softmax_weights", False):
        raise NotImplementedError("the output layer must share the target embedding (all reference presets do)")
    for side in ("encoder", "decoder"):
        if args.get(side + ".ffn_activation", "relu") != "relu" or args.get(side + ".attention_type", "dot_product") != "dot_product":
            raise NotImplementedError("only relu / dot_product are supported")
    for k, dflt in (("attention_dropout_rate", 0.), ("ffn_dropout_rate", 0.), ("layer_postprocess_dropout_rate", 0.),
                    ("layer_postprocess_epsilon", 1e-6)):
        if args.get("encoder." + k, dflt) != args.get("decoder." + k, dflt):
            raise NotImplementedError("libb200st uses one %s for both stacks (encoder.%s != decoder.%s)" % (k, k, k))
    if speech and (args.get("modality.source.kernel_size", 3) != 3 or args.get("modality.source.strides", 2) != 2):
        raise NotImplementedError("the conv front-end is 3x3 stride 2 (all reference presets)")


class _EncoderDecoder:
    def __init__(self, args, src_meta, trg_meta, rt):
        self._args = args
        self._src_meta = src_meta
        self._trg_meta = trg_meta
        self._rt = rt
        self._step_seed = 0

    args = property(lambda self: self._args)
    runtime = property(lambda self: self._rt)
    wait_k = None           # the WaitkTransformer's lag (an int or a list); None: no lag

    def lag(self, is_training):
        """The cross-attention lag of one call (0: none); see WaitkTransformer.lag."""
        return 0

    def named_parameters(self):
        return self._rt.named_parameters()

    def load_parameters(self, P):
        self._rt.load_parameters(P)

    def init_parameters(self, seed=0):
        """glorot-uniform kernels, zero biases, LN gamma=1/beta=0, embedding N(0, d^-0.5) (text_modalities.py:73-74)."""
        g = torch.Generator().manual_seed(seed)
        P = {}
        for name, (_, shp) in self._rt.table.items():
            if name.endswith("emb"):
                t = torch.randn(shp, generator=g) * (shp[1] ** -0.5)
            elif name.endswith(".gamma"):
                t = torch.ones(shp)
            elif len(shp) == 1:
                t = torch.zeros(shp)
            else:
                rf = shp[0] * shp[1] if len(shp) == 4 else 1
                lim = (6.0 / (shp[-2] * rf + shp[-1] * rf)) ** 0.5
                t = (torch.rand(shp, generator=g) * 2 - 1) * lim
            P[name] = t
        self._rt.load_parameters(P)
        return self

    def _batch(self, inputs, is_training, **extra):
        b = dict(inputs)
        if "trg_padding" in b and "trg_length" not in b:
            b["trg_length"] = (1.0 - torch.as_tensor(b["trg_padding"]).float()).sum(-1).long()
        self._step_seed += 1
        b.update(training=bool(is_training), seed=b.get("seed", self._step_seed))
        if "wait_k" not in b:
            b["wait_k"] = self.lag(is_training)
        b.update(extra)
        return b

    def forward(self, inputs, is_training=True):
        """Returns the logits tensor [B, L, V] (encoder_decoder_model.py:263-279)."""
        b = self._batch(inputs, is_training, want_logits=True)
        b.pop("trg", None)
        return self._rt.run(b, backward=False)["logits"]

    __call__ = forward

    def get_symbols_to_logits_fn(self, inputs, is_training, is_inference, decode_padded_length=None):
        """EncoderDecoderModel.get_symbols_to_logits_fn (neurst/models/encoder_decoder_model.py:211-261) ->
        (symbols_to_logits_fn(symbols, cache, time=None), generation_initializer).

        Training / teacher forcing (`is_inference=False`): the cache holds the inputs, `fn(trg_input [B,L], cache)` is the
        fused full forward (logits [B,L,V]).  Inference: the encoder runs once (b200st_encode), the cache is a
        `decode.DecodingCache` (pre-projected memory + preallocated self-attention K/V of `decode_padded_length` or
        `maximum_decode_length` positions), `fn(symbols [B], cache, time)` is one b200st_decode_step (logits [B,V])."""
        from neurst_b200 import decode as D
        trg_meta = self._trg_meta
        if not is_inference:
            held = dict(inputs)

            def symbols_to_logits_fn(symbols, cache, time=None):
                b = dict(cache["inputs"])
                b["trg_input"] = symbols
                return self.forward(b, is_training=is_training)

            init = {"decoder_input": inputs["trg_input"], "decoder_internal_cache": {"inputs": held, "decoding_states": None},
                    "encoder_inputs_maxlen": None, "eos_id": trg_meta["eos_id"], "unk_id": trg_meta.get("unk_id")}
            return symbols_to_logits_fn, init
        if is_training:
            raise NotImplementedError("dropout inside the incremental decoding loop is not supported")
        rt = self._rt
        enc, bias = D.encode(rt, inputs)
        max_len = int(decode_padded_length or self._args.get("maximum_decode_length", 256))
        cache = D.create_decoding_cache(rt, enc, bias, max_len, use_shadow=bool(self._args.get("decode_with_shadow", False)),
                                        wait_k=self.lag(False))

        def symbols_to_logits_fn(symbols, cache, time=None):
            return D.decoder_step_logits(rt, symbols, cache, 0 if time is None else int(time))

        init = {"decoder_input": inputs["trg_input"], "decoder_internal_cache": cache, "encoder_inputs_maxlen": enc.shape[1],
                "eos_id": trg_meta["eos_id"], "unk_id": trg_meta.get("unk_id")}
        return symbols_to_logits_fn, init

    def _bos(self, inputs):
        """The searches' first decoder input: trg_input when given, else BOS for every utterance."""
        bos = inputs.get("trg_input")
        if bos is None:
            bos = torch.full((inputs["src"].shape[0],), int(self._trg_meta["bos_id"]), dtype=torch.long)
        return bos

    def greedy_search(self, inputs, maximum_decode_length=256, extra_decode_length=50, minimum_decode_length=0, enable_unk=False,
                      use_shadow=False):
        """SequenceGenerator with search_method BeamSearch(beam_size=1) (neurst/exps/sequence_generator.py:62-86,
        neurst/layers/search/beam_search.py:254-439) on the device: -> (token ids [B, maximum_decode_length], log-probs [B]).
        At most decode.MAX_ROWS (8) utterances per call with the fp32 weights, decode.MAX_ROWS_SHADOW (256) with use_shadow."""
        from neurst_b200 import decode as D
        tm = self._trg_meta
        ids, logprob, _ = D.greedy_search(self._rt, inputs, self._bos(inputs), tm["eos_id"], tm.get("unk_id"),
                                          maximum_decode_length, extra_decode_length, minimum_decode_length, enable_unk,
                                          use_shadow, wait_k=self.lag(False))
        return ids, logprob

    def beam_search(self, inputs, beam_size=4, length_penalty=0.6, top_k=1, maximum_decode_length=256, extra_decode_length=50,
                    minimum_decode_length=0, enable_unk=False, use_shadow=False):
        """SequenceGenerator with search_method BeamSearch (neurst/layers/search/beam_search.py:439-530) on the device:
        -> (hypotheses [B*top_k, maximum_decode_length], scores [B*top_k]), BeamSearch.call's return.  At most
        decode.MAX_ROWS // beam_size utterances per call with the fp32 weights, decode.MAX_ROWS_SHADOW // beam_size with
        use_shadow (the 16-bit weights; beam_size <= 8)."""
        from neurst_b200 import decode as D
        tm = self._trg_meta
        ids, scores, _, _ = D.beam_search(self._rt, inputs, self._bos(inputs), tm["eos_id"], tm.get("unk_id"), beam_size,
                                          length_penalty, top_k, maximum_decode_length, extra_decode_length,
                                          minimum_decode_length, enable_unk, use_shadow, wait_k=self.lag(False))
        return ids, scores

    def sampling_search(self, inputs, sample_num=1, top_k=0, top_p=1.0, maximum_decode_length=256, extra_decode_length=50,
                        minimum_decode_length=0, seed=1234, row_offset=0, use_shadow=False):
        """SequenceGenerator with search_method TopSampling (neurst/layers/search/sampling.py:265-345) on the device:
        -> (samples [B*sample_num, maximum_decode_length], their log-probabilities [B*sample_num]), row b * sample_num + s
        being sample s of utterance b.  The draws are keyed by (seed, row_offset + row, step) (decode.sampling_search).
        At most decode.MAX_ROWS // sample_num utterances per call with the fp32 weights, decode.MAX_ROWS_SHADOW // sample_num
        with use_shadow; sample_num <= 8."""
        from neurst_b200 import decode as D
        tm = self._trg_meta
        ids, logprob, _ = D.sampling_search(self._rt, inputs, self._bos(inputs), tm["eos_id"], tm.get("unk_id"), sample_num,
                                            top_k, top_p, maximum_decode_length, extra_decode_length, minimum_decode_length,
                                            seed, row_offset, use_shadow, wait_k=self.lag(False))
        return ids, logprob

    def evaluate(self, inputs, is_training=False):
        """logits + criterion outputs (nll_sum [B], n_tokens [B], loss) in one call."""
        return self._rt.run(self._batch(inputs, is_training, want_logits=True), backward=False)

    def forward_backward(self, inputs, is_training=True, loss_scale=1.0):
        """loss = sum(nll)/sum(tokens) and d loss / d params accumulated into the gradient arena."""
        return self._rt.run(self._batch(inputs, is_training, want_logits=False, loss_scale=loss_scale), backward=True)


class SpeechTransformer(_EncoderDecoder):
    """ Defines the Speech Transformer model. """

    @staticmethod
    def class_or_method_args():
        """Flag table of neurst_pt/models/speech_transformer.py:35-106 as (name, type, default, help) tuples; the registry
        plug-in (neurst_b200/plugin.py) turns them into the reference's `Flag` objects."""
        return _model_flags(True)

    @classmethod
    def build_model_args_by_name(cls, name):
        return speech_transformer_hparams(name)

    @classmethod
    def new(cls, args, src_meta, trg_meta, name=None, precision="bf16", label_smoothing=0.0, device="cuda"):
        _check_supported(args, True)
        cfg = make_config(
            L.MODEL_SPEECH, args["encoder.hidden_size"], args["encoder.num_attention_heads"], args["encoder.filter_size"],
            args["encoder.num_layers"], args["decoder.num_layers"], trg_meta["vocab_size"],
            feat=src_meta["audio_feature_dim"], in_channels=src_meta["audio_feature_channels"],
            channels=args.get("modality.source.channels", 256), conv_layer_norm=args.get("modality.source.layer_norm", False),
            precision=precision, ln_eps=args.get("encoder.layer_postprocess_epsilon", 1e-6),
            attention_dropout=args.get("encoder.attention_dropout_rate", 0.), ffn_dropout=args.get("encoder.ffn_dropout_rate", 0.),
            postprocess_dropout=args.get("encoder.layer_postprocess_dropout_rate", 0.), label_smoothing=label_smoothing)
        return cls(args, src_meta, trg_meta, Runtime(cfg, device))


class Transformer(_EncoderDecoder):
    """ Text Transformer (reference cfg-1 plumbing model). """

    @staticmethod
    def class_or_method_args():
        return _model_flags(False)

    @classmethod
    def build_model_args_by_name(cls, name):
        return transformer_hparams(name)

    @classmethod
    def new(cls, args, src_meta, trg_meta, name=None, precision="fp32", label_smoothing=0.0, device="cuda"):
        _check_supported(args, False)
        if args.get("encoder.post_normalize") or args.get("decoder.post_normalize"):
            raise NotImplementedError("post_normalize=True is not supported by libb200st (all presets are pre-norm)")
        share = bool(args.get("modality.share_source_target_embedding", False))
        if share and src_meta["vocab_size"] != trg_meta["vocab_size"]:
            raise ValueError("Source vocab_size should be equal to target vocab_size when modality.share_source_target_embedding"
                             "=True (%d vs %d)" % (src_meta["vocab_size"], trg_meta["vocab_size"]))
        cfg = make_config(
            L.MODEL_TEXT, args["encoder.hidden_size"], args["encoder.num_attention_heads"], args["encoder.filter_size"],
            args["encoder.num_layers"], args["decoder.num_layers"], trg_meta["vocab_size"], src_vocab=src_meta["vocab_size"],
            precision=precision, ln_eps=args.get("encoder.layer_postprocess_epsilon", 1e-6),
            attention_dropout=args.get("encoder.attention_dropout_rate", 0.), ffn_dropout=args.get("encoder.ffn_dropout_rate", 0.),
            postprocess_dropout=args.get("encoder.layer_postprocess_dropout_rate", 0.), label_smoothing=label_smoothing,
            share_src_trg_embedding=share, encoder_monotonic=bool(args.get("encoder.attention_monotonic", False)))
        return cls(args, src_meta, trg_meta, Runtime(cfg, device))


class WaitkTransformer(Transformer):
    """ neurst/models/waitk_transformer.py: a Transformer (same variables) whose decoder cross-attention lags the source by
    `wait_k` tokens: target position i sees the source keys j < i + k (transformer_decoder.py:194-208).  Its presets also make
    the encoder monotonic, so that encoding the whole source once equals the streaming agent's incremental encoding. """

    @classmethod
    def build_model_args_by_name(cls, name):
        return waitk_transformer_hparams(name)

    @classmethod
    def new(cls, args, src_meta, trg_meta, name=None, precision="fp32", label_smoothing=0.0, device="cuda", wait_k=None,
            random_seed=0):
        """wait_k: the task's lag (an int, a list, or a YAML string of either).  random_seed seeds the multi-path draw."""
        if wait_k is None:
            raise ValueError("WaitkTransformer needs wait_k (the decode lagging)")
        model = super(WaitkTransformer, cls).new(args, src_meta, trg_meta, name=name, precision=precision,
                                                 label_smoothing=label_smoothing, device=device)
        model.wait_k = parse_wait_k(wait_k)
        model._lag_gen = torch.Generator().manual_seed(int(random_seed))
        return model

    def lag(self, is_training):
        """waitk_transformer.py:102-110: training with a list draws one k uniformly per call (multi-path); otherwise the first
        k of the list.  The draw comes from a generator seeded by the run's random_seed, so that every replica draws the same
        k at the same step (the reference draws with an unseeded tf.random.uniform on each replica)."""
        ks = self.wait_k
        if not isinstance(ks, list):
            return int(ks)
        if is_training and len(ks) > 1:
            return int(ks[int(torch.randint(len(ks), (1,), generator=self._lag_gen))])
        return int(ks[0])


class EncoderDecoderEnsembleModel:
    """ neurst/models/encoder_decoder_ensemble_model.py: several encoder-decoder models decoding as one, for generation only.
    Its searches mix the members' next-token distributions on the device at every step (decode.ensemble_beam_search). """

    def __init__(self, encoder_decoder_models):
        self._encoder_decoder_models = list(encoder_decoder_models)

    @classmethod
    def new(cls, encoder_decoder_models):
        return cls(encoder_decoder_models)

    @property
    def model_num(self):
        return len(self._encoder_decoder_models)

    @property
    def models(self):
        return list(self._encoder_decoder_models)

    def get_symbols_to_logits_fn(self, inputs, is_training=False, is_inference=True, decode_padded_length=None):
        """-> (symbols_to_logits_fn(symbols, cache_per_model, time=None) returning the list of the members' logits [B, V],
        generation_initializer whose decoder_internal_cache is the list of the members' caches), as the reference's."""
        fns, init = [], None
        for model in self._encoder_decoder_models:
            fn, model_init = model.get_symbols_to_logits_fn(inputs, False, True, decode_padded_length=decode_padded_length)
            fns.append(fn)
            if init is None:
                init = dict(model_init, decoder_internal_cache=[model_init["decoder_internal_cache"]])
            else:
                init["decoder_internal_cache"].append(model_init["decoder_internal_cache"])

        def symbols_to_logits_fn(symbols, cache_per_model, time=None):
            return [fn(symbols, cache, time=time) for fn, cache in zip(fns, cache_per_model)]

        return symbols_to_logits_fn, init

    def _bos(self, inputs):
        return self._encoder_decoder_models[0]._bos(inputs)

    def beam_search(self, inputs, beam_size=4, length_penalty=0.6, top_k=1, maximum_decode_length=256, extra_decode_length=50,
                    minimum_decode_length=0, enable_unk=False, ensemble_weights="average", use_shadow=False):
        """BeamSearch with `ensemble_weights` over the members -> (hypotheses [B*top_k, maximum_decode_length],
        scores [B*top_k]), with the row limits of the single model's beam_search."""
        from neurst_b200 import decode as D
        tm = self._encoder_decoder_models[0]._trg_meta
        ids, scores, _, _ = D.ensemble_beam_search([m.runtime for m in self._encoder_decoder_models], inputs, self._bos(inputs),
                                                   tm["eos_id"], tm.get("unk_id"), ensemble_weights, beam_size, length_penalty, top_k,
                                                   maximum_decode_length, extra_decode_length, minimum_decode_length, enable_unk,
                                                   use_shadow)
        return ids, scores

    def greedy_search(self, inputs, maximum_decode_length=256, extra_decode_length=50, minimum_decode_length=0, enable_unk=False,
                      ensemble_weights="average", use_shadow=False):
        """The ensemble's beam_search with beam_size 1 (the reference's greedy search) -> (token ids [B, maximum_decode_length],
        log-probs [B])."""
        from neurst_b200 import decode as D
        tm = self._encoder_decoder_models[0]._trg_meta
        ids, _, logprob, _ = D.ensemble_beam_search([m.runtime for m in self._encoder_decoder_models], inputs, self._bos(inputs),
                                                    tm["eos_id"], tm.get("unk_id"), ensemble_weights, 1, 0.6, 1, maximum_decode_length,
                                                    extra_decode_length, minimum_decode_length, enable_unk, use_shadow)
        return ids, logprob

    def call(self, inputs, is_training=True):
        raise NotImplementedError("No need to implement call function for EncoderDecoderEnsembleModel.")


class LabelSmoothedCrossEntropy:
    """ Criterion with the reference's call contract: (model_inp, logits) -> (nll_sum [B], n_samples [1], n_tokens [B]). """

    def __init__(self, args):
        self._label_smoothing = args["label_smoothing"]

    def __call__(self, model_inp, model_out):
        import ctypes as C
        logits = model_out["logits"] if isinstance(model_out, dict) else model_out
        if not torch.is_tensor(logits):
            raise ValueError("Not supported type of model_out: {}".format(type(model_out)))
        logits = logits.float().contiguous().cuda()
        B, Lq, V = logits.shape
        trg = torch.as_tensor(model_inp["trg"]).long().contiguous().cuda()
        length = model_inp.get("trg_length", model_inp.get("length"))
        if length is None:
            padding = model_inp.get("trg_padding", model_inp.get("padding"))
            length = (1.0 - torch.as_tensor(padding).float()).sum(-1)
        length = torch.as_tensor(length).long().contiguous().cuda()
        nll = torch.zeros(B, device="cuda")
        ntok = torch.zeros(B, device="cuda")
        loss = torch.zeros(1, device="cuda")
        L.check(L.load().b200st_lsce(logits.data_ptr(), trg.data_ptr(), length.data_ptr(), B, Lq, V, self._label_smoothing,
                                     nll.data_ptr(), ntok.data_ptr(), loss.data_ptr(), None, 0, 1.0, L._stream()))
        return nll, torch.tensor([float(B)], device="cuda"), ntok

    def reduce_loss(self, model_inp, model_out):
        nll_sum, _, n_tokens = self(model_inp, model_out)
        return nll_sum.sum() / n_tokens.sum()
