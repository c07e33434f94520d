"""Checkpoint interchange with the reference's name-based format (SURVEY.md 8 f3).

The reference saves `tf.train.Checkpoint(**{variable_name: variable})` (NameBasedCheckpointManager,
neurst/utils/checkpoints.py:148-183) and restores by name under the checkpoint's scope name (:340-360).  The variable
names are fixed by the layer constructors (transformer_layers.py:70-87,179-209; audio_modalities.py:71-81;
text_modalities.py:64-81; speech_transformer.py:116-139), listed in SURVEY.md Appendix B.  This module maps the flat
libb200st arena to those names and to the `neurst_pt` module attributes:

  tf_variable_names(table)            our name -> reference TF variable name (kernels already share the TF layout)
  save_npz / load_npz                 NumPy archive keyed by the TF variable names: the interchange file.  On a TensorFlow box
                                      `{n: tf.train.load_variable(ckpt, n + "/.ATTRIBUTES/VARIABLE_VALUE") ...}` -> np.savez
                                      converts a published checkpoint; np.load -> tf.Variable.assign the other way.
  from_reference_pt / to_reference_pt  copy weights from / into an instantiated `neurst_pt` SpeechTransformer (layout map of
                                      tests/neurst_pt/models/speech_transformer_test.py:57-152: conv OIHW <-> HWIO, Linear.T)

A reader of TensorFlow's bundle files (.index SSTable + .data shards) is NOT included: there is no TensorFlow here and
no checkpoint fixture in the reference tree to validate one against (parity unpinned — see DESIGN.md).
"""
import re

import numpy as np
import torch

MODEL_SCOPE = "SpeechTransformer"
TEXT_MODEL_SCOPE = "Transformer"


def is_text_table(table):
    """A text Transformer's table: no audio front-end (the source is the embedding table srcemb.emb or, tied, trg.emb)."""
    return "src.conv1.kernel" not in table and "trg.emb" in table


def model_scope(table):
    """The reference model's name scope: `SpeechTransformer` or, for the text model, `Transformer`."""
    return TEXT_MODEL_SCOPE if is_text_table(table) else MODEL_SCOPE


def tf_variable_names(table, scope=None):
    """{our parameter name: reference variable name} for every tensor of a SpeechTransformer or text Transformer parameter
    table.  The text model's modalities are `input_symbol_modality` (source table, `emb/weights`) and
    `target_symbol_modality` (`shared/{weights,bias}`), or one `shared_symbol_modality` when the source and target tables
    are tied (encoder_decoder_model.py:148-178); each sits in its `_posenc_wrapper` (sinusoid timing)."""
    scope = model_scope(table) if scope is None else scope
    out = {}
    src = scope + "/input_audio_modality_posenc_wrapper/input_audio_modality"
    trg = scope + "/target_symbol_modality_posenc_wrapper/target_symbol_modality"
    if is_text_table(table) and "srcemb.emb" not in table:
        trg = scope + "/shared_symbol_modality_posenc_wrapper/shared_symbol_modality"
    fixed = {
        "srcemb.emb": scope + "/input_symbol_modality_posenc_wrapper/input_symbol_modality/emb/weights",
        "src.conv1.kernel": src + "/conv1/kernel", "src.conv1.bias": src + "/conv1/bias",
        "src.conv2.kernel": src + "/conv2/kernel", "src.conv2.bias": src + "/conv2/bias",
        "src.ln1.gamma": src + "/ln1/gamma", "src.ln1.beta": src + "/ln1/beta",
        "src.ln2.gamma": src + "/ln2/gamma", "src.ln2.beta": src + "/ln2/beta",
        "src.dense.kernel": src + "/output_dense/kernel", "src.dense.bias": src + "/output_dense/bias",
        "trg.emb": trg + "/shared/weights", "trg.bias": trg + "/shared/bias",
        "enc.out_ln.gamma": scope + "/TransformerEncoder/output_ln/gamma", "enc.out_ln.beta": scope + "/TransformerEncoder/output_ln/beta",
        "dec.out_ln.gamma": scope + "/TransformerDecoder/output_ln/gamma", "dec.out_ln.beta": scope + "/TransformerDecoder/output_ln/beta",
    }
    sub = {"att": ("self_attention_prepost_wrapper", "self_attention"), "self": ("self_attention_prepost_wrapper", "self_attention"),
           "cross": ("encdec_attention_prepost_wrapper", "encdec_attention"), "ffn": ("ffn_prepost_wrapper", "ffn")}
    leaf = {"ln.gamma": "ln/gamma", "ln.beta": "ln/beta",
            "qkv.kernel": "qkv_transform/kernel", "qkv.bias": "qkv_transform/bias", "q.kernel": "q_transform/kernel",
            "q.bias": "q_transform/bias", "kv.kernel": "kv_transform/kernel", "kv.bias": "kv_transform/bias",
            "out.kernel": "output_transform/kernel", "out.bias": "output_transform/bias",
            "w1": "dense1/kernel", "b1": "dense1/bias", "w2": "dense2/kernel", "b2": "dense2/bias"}
    for name in table:
        if name in fixed:
            out[name] = fixed[name]
            continue
        m = re.match(r"(enc|dec)\.(\d+)\.(att|self|cross|ffn)\.(.+)$", name)
        if not m:
            raise KeyError("no reference variable name for parameter %r" % name)
        stack = "TransformerEncoder" if m.group(1) == "enc" else "TransformerDecoder"
        wrap, inner = sub[m.group(3)]
        tail = leaf[m.group(4)]
        tail = tail if tail.startswith("ln/") else inner + "/" + tail
        out[name] = "%s/%s/layer_%s/%s/%s" % (scope, stack, m.group(2), wrap, tail)
    return out


def archive_scope(keys, table):
    """The top-level scope of an archive's variable names when they share one, else the model's own scope."""
    scopes = {k.split("/")[0] for k in keys if "/" in k}
    return scopes.pop() if len(scopes) == 1 else model_scope(table)


def save_npz(rt, path, scope=None, extra=None):
    """Writes every parameter under its reference variable name (+ optional Adam slots as `<name>/.OPTIMIZER_SLOT/{m,v}`)."""
    names = tf_variable_names(rt.table, scope)
    arrays = {names[k]: rt.view(k).detach().cpu().numpy() for k in rt.table}
    if extra:
        arrays.update(extra)
    if getattr(rt, "adam_m", None) is not None:
        for k in rt.table:
            arrays[names[k] + "/.OPTIMIZER_SLOT/m"] = rt.view(k, rt.adam_m).detach().cpu().numpy()
            arrays[names[k] + "/.OPTIMIZER_SLOT/v"] = rt.view(k, rt.adam_v).detach().cpu().numpy()
    np.savez(path, **arrays)
    return sorted(arrays)


def load_npz(rt, path, scope=None, strict=True, pattern=None, slots=True):
    """Restores by name.  `scope=None` uses the archive's own top-level scope (checkpoint_scope_name, checkpoints.py:322-338).
    `pattern`: restore only the variables whose name in THIS model (its own scope) matches the regular expression
    (re.search), each read from the archive under the archive's scope (restore_checkpoint_if_possible,
    checkpoints.py:340-360); the Adam slots are then left alone, as they are with `slots=False` (pretraining restores the
    model's weights only)."""
    z = np.load(path)
    keys = [k for k in z.files if "/.OPTIMIZER_SLOT/" not in k]
    if scope is None:
        scope = archive_scope(keys, rt.table)
    names = tf_variable_names(rt.table, scope)
    if pattern is not None:
        own = tf_variable_names(rt.table)
        names = {k: v for k, v in names.items() if re.search(pattern, own[k]) is not None}
    missing = [v for v in names.values() if v not in z.files]
    if missing and strict:
        raise KeyError("checkpoint misses %d variables, e.g. %s" % (len(missing), missing[:3]))
    P = {k: torch.from_numpy(np.asarray(z[v])) for k, v in names.items() if v in z.files}
    for k, t in P.items():
        if tuple(t.shape) != tuple(rt.table[k][1]):
            raise ValueError("shape mismatch for %s: checkpoint %s vs model %s" % (names[k], tuple(t.shape), rt.table[k][1]))
        rt.view(k).copy_(t.to(torch.float32))
    rt._shadow_stale = True
    if slots and pattern is None and all((names[k] + "/.OPTIMIZER_SLOT/m") in z.files for k in rt.table):
        if rt.adam_m is None:
            rt.adam_m, rt.adam_v = torch.zeros_like(rt.params), torch.zeros_like(rt.params)
        for k in rt.table:
            rt.view(k, rt.adam_m).copy_(torch.from_numpy(z[names[k] + "/.OPTIMIZER_SLOT/m"]))
            rt.view(k, rt.adam_v).copy_(torch.from_numpy(z[names[k] + "/.OPTIMIZER_SLOT/v"]))
    return sorted(P)


# ---- neurst_pt module <-> our names (layout map of tests/neurst_pt/models/speech_transformer_test.py:57-152) -------------
def _pt_slots(model):
    """Yields (our name, torch parameter, to_ours(t), to_theirs(t))."""
    ident = (lambda t: t, lambda t: t)
    tr = (lambda t: t.t(), lambda t: t.t())
    conv = (lambda t: t.permute(2, 3, 1, 0), lambda t: t.permute(3, 2, 0, 1))     # OIHW <-> HWIO
    sm = model._src_modality._embedding_layer if hasattr(model._src_modality, "_embedding_layer") else model._src_modality
    yield ("src.conv1.kernel", sm._conv_layer1.weight) + conv
    yield ("src.conv1.bias", sm._conv_layer1.bias) + ident
    yield ("src.conv2.kernel", sm._conv_layer2.weight) + conv
    yield ("src.conv2.bias", sm._conv_layer2.bias) + ident
    if hasattr(sm, "_norm_layer1"):
        yield ("src.ln1.gamma", sm._norm_layer1.weight) + ident
        yield ("src.ln1.beta", sm._norm_layer1.bias) + ident
        yield ("src.ln2.gamma", sm._norm_layer2.weight) + ident
        yield ("src.ln2.beta", sm._norm_layer2.bias) + ident
    yield ("src.dense.kernel", sm._dense_layer.weight) + tr
    yield ("src.dense.bias", sm._dense_layer.bias) + ident

    def att(pre, wrap, cross):
        yield (pre + ".ln.gamma", wrap._norm_layer.weight) + ident
        yield (pre + ".ln.beta", wrap._norm_layer.bias) + ident
        a = wrap._layer
        if cross:
            yield (pre + ".q.kernel", a._q_transform_layer._kernel) + ident
            yield (pre + ".q.bias", a._q_transform_layer._bias) + ident
            yield (pre + ".kv.kernel", a._kv_transform_layer._kernel) + ident
            yield (pre + ".kv.bias", a._kv_transform_layer._bias) + ident
        else:
            yield (pre + ".qkv.kernel", a._qkv_transform_layer._kernel) + ident
            yield (pre + ".qkv.bias", a._qkv_transform_layer._bias) + ident
        yield (pre + ".out.kernel", a._output_transform_layer._kernel) + ident
        yield (pre + ".out.bias", a._output_transform_layer._bias) + ident

    def ffn(pre, wrap):
        yield (pre + ".ln.gamma", wrap._norm_layer.weight) + ident
        yield (pre + ".ln.beta", wrap._norm_layer.bias) + ident
        f = wrap._layer
        yield (pre + ".w1", f._dense1.weight) + tr
        yield (pre + ".b1", f._dense1.bias) + ident
        yield (pre + ".w2", f._dense2.weight) + tr
        yield (pre + ".b2", f._dense2.bias) + ident

    for i, layer in enumerate(model._encoder._stacking_layers):
        yield from att("enc.%d.att" % i, layer[0], False)
        yield from ffn("enc.%d.ffn" % i, layer[1])
    yield ("enc.out_ln.gamma", model._encoder._output_norm_layer.weight) + ident
    yield ("enc.out_ln.beta", model._encoder._output_norm_layer.bias) + ident
    for i, layer in enumerate(model._decoder._stacking_layers):
        yield from att("dec.%d.self" % i, layer[0], False)
        yield from att("dec.%d.cross" % i, layer[1], True)
        yield from ffn("dec.%d.ffn" % i, layer[2])
    yield ("dec.out_ln.gamma", model._decoder._output_norm_layer.weight) + ident
    yield ("dec.out_ln.beta", model._decoder._output_norm_layer.bias) + ident
    tm = model._trg_modality._embedding_layer if hasattr(model._trg_modality, "_embedding_layer") else model._trg_modality
    yield ("trg.emb", tm._shared_weights) + ident
    yield ("trg.bias", tm._bias) + ident


def from_reference_pt(model):
    """{our name: tensor in the TF layout} from an instantiated reference `neurst_pt` SpeechTransformer."""
    return {name: to_ours(p.detach()).contiguous().clone() for name, p, to_ours, _ in _pt_slots(model)}


def to_reference_pt(P, model):
    """Copies {our name: tensor} into the reference module's parameters (in place)."""
    with torch.no_grad():
        for name, p, _, to_theirs in _pt_slots(model):
            p.copy_(to_theirs(torch.as_tensor(P[name]).to(p.dtype)).reshape(p.shape))
    return model
