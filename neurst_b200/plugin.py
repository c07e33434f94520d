"""Registry plug-in: makes the reference's own `build_model` / `build_encoder` / ... return the libb200st-backed classes.

The reference's plug-in mechanism is the class registry (neurst/utils/registry.py:24-137) filled by
`--include <package>` (neurst/utils/flags_core.py:207-247).  `register()` adds, to the `pt` registries (and to the `tf`
ones when TensorFlow — hence the reference's TF packages — imports):

  model     B200SpeechTransformer (aliases b200speechtransformer, b200_speech_transformer, B200ST), B200Transformer
  encoder   B200TransformerEncoder        decoder  B200TransformerDecoder
  base_layer  B200MultiHeadAttention, B200MultiHeadSelfAttention

Registering a *different* class under an existing name raises in the reference (registry.py:120-122), so the drop-in uses
new names; `override=True` additionally points the stock names ("SpeechTransformer", "TransformerEncoder", ...) at the
H100 classes by assigning REGISTRIES[backend][registry][name] directly, which is what a deployment that wants existing
yaml files to run unchanged does.

Each registered class subclasses the registry's base class (`issubclass` is enforced, registry.py:111-112), exposes the
reference's `class_or_method_args()` as reference `Flag` objects — so `build_x` takes the
`builder(params_with_defaults, *extra)` branch (registry.py:90-102) — and delegates to neurst_b200.models / .layers,
i.e. to the C ABI.  No tensor math lives here.
"""
import importlib

_REGISTERED = {}
_CLASSES = {}      # (backend, registry, class name) -> the registered class (created once per process)


def reference_available():
    try:
        importlib.import_module("neurst.utils.registry")
        importlib.import_module("neurst_pt.models")
        return True
    except Exception:
        return False


def _ref_flags(table):
    from neurst.utils.flags_core import Flag
    return [Flag(name, dtype=ty, default=dflt, help=hlp) for name, ty, dflt, hlp in table]


def _make_model_class(base, cls_name, impl_cls, speech):
    from neurst_b200 import models as M

    class _B200Model(base):
        """ libb200st-backed drop-in for the reference model class of the same role. """
        IMPL = impl_cls

        def __init__(self, args, impl):
            base.__init__(self, args)
            self._impl = impl

        @staticmethod
        def class_or_method_args():
            return _ref_flags(M._model_flags(speech))

        @classmethod
        def new(cls, args, src_meta, trg_meta, name=None, **kw):
            return cls(args, impl_cls.new(args, src_meta, trg_meta, name=name, **kw))

        @classmethod
        def build_model_args_by_name(cls, name):
            return impl_cls.build_model_args_by_name(name)

        impl = property(lambda self: self._impl)
        runtime = property(lambda self: self._impl.runtime)

        def forward(self, inputs, is_training=True):
            return self._impl.forward(inputs, is_training=is_training)

        def __call__(self, inputs, is_training=True):       # nn.Module.__call__ would insist on tensors / hooks
            return self.forward(inputs, is_training=is_training)

        def get_symbols_to_logits_fn(self, inputs, is_training, is_inference, decode_padded_length=None):
            return self._impl.get_symbols_to_logits_fn(inputs, is_training, is_inference, decode_padded_length)

        def forward_backward(self, inputs, is_training=True, loss_scale=1.0):
            return self._impl.forward_backward(inputs, is_training=is_training, loss_scale=loss_scale)

        def named_parameters(self, *a, **k):
            return self._impl.named_parameters()

        def load_parameters(self, P):
            return self._impl.load_parameters(P)

    _B200Model.__name__ = _B200Model.__qualname__ = cls_name
    return _B200Model


def _make_layer_class(base, cls_name, impl_cls):
    class _B200Layer(base):
        """ libb200st-backed drop-in for the reference layer of the same name (constructor signature unchanged). """
        IMPL = impl_cls

        def __init__(self, *args, **kwargs):
            base.__init__(self)
            self._impl = impl_cls(*args, **kwargs)

        impl = property(lambda self: self._impl)

        def forward(self, *args, **kwargs):
            return self._impl.forward(*args, **kwargs)

        def __call__(self, *args, **kwargs):
            return self._impl.forward(*args, **kwargs)

        def __getattr__(self, name):
            if name.startswith("__") or name == "_impl":
                raise AttributeError(name)
            try:
                return base.__getattr__(self, name)
            except AttributeError:
                return getattr(self.__dict__["_impl"], name)

    _B200Layer.__name__ = _B200Layer.__qualname__ = cls_name
    return _B200Layer


def register(override=False):
    """Writes the H100 classes into the reference registries.  Returns {backend: {registry: [names]}}.
    Needs `neurst.utils.registry` + `neurst_pt` importable (the reference on sys.path); raises ImportError otherwise."""
    if _REGISTERED and not override:
        return _REGISTERED
    from neurst.utils import registry as REG
    from neurst_b200 import layers as Ly
    from neurst_b200 import models as M
    import torch.nn as nn

    out = {}

    def put(backend, reg_name, register_fn, make_cls, aliases, stock):
        key = (backend, reg_name, make_cls[2])
        if key not in _CLASSES:
            _CLASSES[key] = make_cls[0](*make_cls[1:])
            register_fn(aliases)(_CLASSES[key])
        cls = _CLASSES[key]
        names = sorted(REG.REGISTRIED_CLS2ALIAS[backend][reg_name][cls.__name__])
        if override:
            for n in stock:
                REG.REGISTRIES[backend][reg_name][n] = cls
            names += list(stock)
        out.setdefault(backend, {}).setdefault(reg_name, []).extend(names)

    # ---- pt backend: always (neurst_pt imports without TensorFlow) ----
    from neurst_pt.models import register_model as pt_register_model
    from neurst_pt.models.model import BaseModel as PtBaseModel
    from neurst_pt.layers import register_base_layer as pt_register_layer
    from neurst_pt.layers.encoders import register_encoder as pt_register_encoder
    from neurst_pt.layers.decoders import register_decoder as pt_register_decoder
    from neurst_pt.layers.encoders.encoder import Encoder as PtEncoder
    from neurst_pt.layers.decoders.decoder import Decoder as PtDecoder

    put("pt", "model", pt_register_model, (_make_model_class, PtBaseModel, "B200SpeechTransformer", M.SpeechTransformer, True),
        ["B200ST", "b200_speech_transformer"], ["SpeechTransformer", "speechtransformer", "speech_transformer"])
    put("pt", "model", pt_register_model, (_make_model_class, PtBaseModel, "B200Transformer", M.Transformer, False),
        ["b200_transformer"], ["Transformer", "transformer"])
    put("pt", "encoder", pt_register_encoder, (_make_layer_class, PtEncoder, "B200TransformerEncoder", Ly.TransformerEncoder),
        ["b200_transformer_encoder"], ["TransformerEncoder", "transformerencoder", "transformer_encoder"])
    put("pt", "decoder", pt_register_decoder, (_make_layer_class, PtDecoder, "B200TransformerDecoder", Ly.TransformerDecoder),
        ["b200_transformer_decoder"], ["TransformerDecoder", "transformerdecoder", "transformer_decoder"])
    put("pt", "base_layer", pt_register_layer, (_make_layer_class, nn.Module, "B200MultiHeadAttention", Ly.MultiHeadAttention),
        ["b200_multi_head_attention"], ["MultiHeadAttention", "multiheadattention", "multi_head_attention"])
    put("pt", "base_layer", pt_register_layer, (_make_layer_class, nn.Module, "B200MultiHeadSelfAttention", Ly.MultiHeadSelfAttention),
        ["b200_multi_head_self_attention"],
        ["MultiHeadSelfAttention", "multiheadselfattention", "multi_head_self_attention"])

    # ---- tf backend: only where TensorFlow (and therefore neurst.models) imports ----
    try:
        import tensorflow as tf
        if not hasattr(tf, "keras"):
            raise ImportError("not a real TensorFlow")
        from neurst.models import register_model as tf_register_model
        from neurst.models.model import BaseModel as TfBaseModel
        put("tf", "model", tf_register_model, (_make_model_class, TfBaseModel, "B200SpeechTransformer", M.SpeechTransformer, True),
            ["B200ST", "b200_speech_transformer"], ["SpeechTransformer", "speechtransformer", "speech_transformer"])
    except Exception:
        pass
    _REGISTERED.clear()
    _REGISTERED.update(out)
    return out
