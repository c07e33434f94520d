"""ORACLE (test infrastructure only): generates tests/golden/*.npz.  Run in the build container only
(`python oracle/make_golden.py`); it reads the reference tree ($NEURST_REFERENCE), which the test machines need not have.

Two kinds of fixtures:
  kat_*.npz   — the TF-generated known-answer vectors hard-coded in the reference's own tests
                (tests/neurst/**), extracted here by parsing those test files' literals with `ast`
                (weights, inputs, expected outputs; nothing is executed).
  refpt_*.npz — inputs, weights (converted to the TF layouts of SURVEY Appx B) and outputs of the
                UNMODIFIED reference PyTorch mirror (neurst_pt) run on CPU through oracle/ref_shim.py.
"""
import ast
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.environ.get("NEURST_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden")


# ----------------------------------------------------------------------------------------------
# KAT extraction
# ----------------------------------------------------------------------------------------------
def _num_literal(node):
    """Returns a numpy array if `node` (or its first positional arg, for tf.convert_to_tensor / numpy.array
    calls) is a nested numeric list literal, else None."""
    if isinstance(node, ast.Call) and node.args:
        return _num_literal(node.args[0])
    if isinstance(node, (ast.List, ast.Tuple)):
        try:
            return np.array(ast.literal_eval(node), dtype=np.float64)
        except Exception:
            return None
    return None


def _first_literal(nodes):
    for n in nodes:
        for sub in ast.walk(n):
            if isinstance(sub, ast.Call):
                arr = _num_literal(sub)
                if arr is not None and arr.size > 0:
                    return arr
    return None


def _str_consts(node):
    return [s.value for s in ast.walk(node) if isinstance(s, ast.Constant) and isinstance(s.value, str)]


def extract_kat(path, func):
    """dict with keys  w:<substring tested against w.name>  |  shape:<tuple>  |  var:<assigned name>  |
    dict:<key> (literal dict entries)  |  expect:<i> (literals inside assert statements, in order)."""
    tree = ast.parse(open(path).read())
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == func][0]
    out = {}
    n_expect = 0

    def visit_if(node):
        test = node.test
        key = None
        strs = _str_consts(test)
        if strs:
            key = "w:" + "".join(strs)
        elif isinstance(test, ast.Compare) and isinstance(test.comparators[0], ast.Tuple):
            key = "shape:" + str(tuple(ast.literal_eval(test.comparators[0])))
        arr = _first_literal(node.body)
        if key is not None and arr is not None:
            out[key] = arr
        for o in node.orelse:
            if isinstance(o, ast.If):
                visit_if(o)

    for node in ast.walk(fn):
        if isinstance(node, ast.Assign) and len(node.targets) == 1 and isinstance(node.targets[0], ast.Name):
            arr = _num_literal(node.value) if isinstance(node.value, (ast.Call, ast.List)) else None
            if arr is not None and arr.size > 0:
                out.setdefault("var:" + node.targets[0].id, arr)
            if isinstance(node.value, ast.Dict):
                for k, v in zip(node.value.keys, node.value.values):
                    a = _num_literal(v)
                    if a is not None and isinstance(k, ast.Constant):
                        out["dict:" + str(k.value)] = a
    for node in fn.body:
        for sub in ast.walk(node):
            if isinstance(sub, ast.If):
                visit_if(sub)
            if (isinstance(sub, ast.Call) and isinstance(sub.func, ast.Attribute) and sub.func.attr == "set_weights"
                    and "call:set_weights" not in out):
                arr = _first_literal(sub.args)
                if arr is not None:
                    out["call:set_weights"] = arr
    for node in ast.walk(fn):
        if isinstance(node, ast.Assert) or (isinstance(node, ast.Expr) and isinstance(node.value, ast.Call)
                                            and "assert" in ast.dump(node.value.func)):
            for sub in ast.walk(node):
                if isinstance(sub, ast.Call):
                    a = _num_literal(sub)
                    if a is not None and a.size > 1 and isinstance(sub.func, ast.Attribute) and sub.func.attr == "array":
                        out["expect:%d" % n_expect] = a
                        n_expect += 1
    return out


KATS = [
    ("kat_mha_cross", "tests/neurst/layers/attentions/multi_head_attention_test.py", "test_multihead_attention"),
    ("kat_mha_self", "tests/neurst/layers/attentions/multi_head_attention_test.py", "test_multiheadself_attention"),
    ("kat_mha_self_cache", "tests/neurst/layers/attentions/multi_head_attention_test.py",
     "test_multiheadself_attention_under_dec"),
    ("kat_encoder", "tests/neurst/layers/encoders/transformer_encoder_test.py", "test_transformer_encoder"),
    ("kat_decoder", "tests/neurst/layers/decoders/transformer_decoder_test.py", "test_transformer_decoder"),
    ("kat_transformer", "tests/neurst/models/transformer_test.py", "test_seq2seq"),
    ("kat_position", "tests/neurst/layers/common_layers_test.py", "test_position_embedding"),
]


def make_kats():
    for name, rel, func in KATS:
        path = os.path.join(REF, rel)
        try:
            d = extract_kat(path, func)
        except IndexError:
            print("skip %s: %s not found" % (name, func))
            continue
        np.savez(os.path.join(OUT, name + ".npz"), **d)
        print(name, {k: v.shape for k, v in d.items()})


# ----------------------------------------------------------------------------------------------
# reference-PT generated fixtures
# ----------------------------------------------------------------------------------------------
def pt_speech_transformer_params(model):
    """Reference PT module -> flat dict in TF layouts (inverse of the map in
    tests/neurst_pt/models/speech_transformer_test.py:57-152 / SURVEY Appx B)."""
    import torch
    P = {}

    def g(t):
        return t.detach().clone().double().numpy()

    sm = model._src_modality._embedding_layer if hasattr(model._src_modality, "_embedding_layer") else model._src_modality
    if hasattr(sm, "_conv_layer1"):
        P["src.conv1.kernel"] = g(sm._conv_layer1.weight.permute(2, 3, 1, 0)); P["src.conv1.bias"] = g(sm._conv_layer1.bias)
        P["src.conv2.kernel"] = g(sm._conv_layer2.weight.permute(2, 3, 1, 0)); P["src.conv2.bias"] = g(sm._conv_layer2.bias)
        P["src.ln1.gamma"] = g(sm._norm_layer1.weight); P["src.ln1.beta"] = g(sm._norm_layer1.bias)
        P["src.ln2.gamma"] = g(sm._norm_layer2.weight); P["src.ln2.beta"] = g(sm._norm_layer2.bias)
        P["src.dense.kernel"] = g(sm._dense_layer.weight.t()); P["src.dense.bias"] = g(sm._dense_layer.bias)

    def att(pre, wrap, cross):
        P[pre + ".ln.gamma"] = g(wrap._norm_layer.weight); P[pre + ".ln.beta"] = g(wrap._norm_layer.bias)
        a = wrap._layer
        if cross:
            P[pre + ".q.kernel"] = g(a._q_transform_layer._kernel); P[pre + ".q.bias"] = g(a._q_transform_layer._bias)
            P[pre + ".kv.kernel"] = g(a._kv_transform_layer._kernel); P[pre + ".kv.bias"] = g(a._kv_transform_layer._bias)
        else:
            P[pre + ".qkv.kernel"] = g(a._qkv_transform_layer._kernel); P[pre + ".qkv.bias"] = g(a._qkv_transform_layer._bias)
        P[pre + ".out.kernel"] = g(a._output_transform_layer._kernel); P[pre + ".out.bias"] = g(a._output_transform_layer._bias)

    def ffn(pre, wrap):
        P[pre + ".ln.gamma"] = g(wrap._norm_layer.weight); P[pre + ".ln.beta"] = g(wrap._norm_layer.bias)
        f = wrap._layer
        P[pre + ".w1"] = g(f._dense1.weight.t()); P[pre + ".b1"] = g(f._dense1.bias)
        P[pre + ".w2"] = g(f._dense2.weight.t()); P[pre + ".b2"] = g(f._dense2.bias)

    for i, layer in enumerate(model._encoder._stacking_layers):
        att("enc.%d.att" % i, layer[0], False); ffn("enc.%d.ffn" % i, layer[1])
    P["enc.out_ln.gamma"] = g(model._encoder._output_norm_layer.weight)
    P["enc.out_ln.beta"] = g(model._encoder._output_norm_layer.bias)
    for i, layer in enumerate(model._decoder._stacking_layers):
        att("dec.%d.self" % i, layer[0], False); att("dec.%d.cross" % i, layer[1], True); ffn("dec.%d.ffn" % i, layer[2])
    P["dec.out_ln.gamma"] = g(model._decoder._output_norm_layer.weight)
    P["dec.out_ln.beta"] = g(model._decoder._output_norm_layer.bias)
    tm = model._trg_modality._embedding_layer
    P["trg.emb"] = g(tm._shared_weights); P["trg.bias"] = g(tm._bias)
    return P


def _all_reference_params(model):
    """The reference keeps layer stacks in python lists (invisible to .parameters()); walk them explicitly."""
    import torch
    ps = list(model.parameters())
    for stack in (model._encoder._stacking_layers, model._decoder._stacking_layers):
        for layer in stack:
            for sub in layer:
                if sub is not None:
                    ps.extend(sub.parameters())
    return ps


def make_refpt():
    import torch
    from oracle import ref_shim
    ref_shim.install()
    from neurst_pt.models.speech_transformer import SpeechTransformer

    def build(d, heads, enc_layers, dec_layers, ffn_size, channels, vocab, seed):
        torch.manual_seed(seed)
        np.random.seed(seed)
        params = {
            "modality.source.kernel_size": 3, "modality.source.strides": 2, "modality.source.channels": channels,
            "modality.source.layer_norm": True, "modality.dim": d, "modality.source.dim": None,
            "modality.target.dim": None, "modality.share_embedding_and_softmax_weights": True,
            "modality.timing": "sinusoids", "modality.source.timing": None, "modality.target.timing": None,
        }
        for side, nl in (("encoder", enc_layers), ("decoder", dec_layers)):
            params.update({side + ".num_layers": nl, side + ".hidden_size": d, side + ".num_attention_heads": heads,
                           side + ".filter_size": ffn_size, side + ".attention_dropout_rate": 0.1,
                           side + ".attention_type": "dot_product", side + ".ffn_activation": "relu",
                           side + ".ffn_dropout_rate": 0.1, side + ".layer_postprocess_dropout_rate": 0.1,
                           side + ".layer_postprocess_epsilon": 1e-6})
        src_meta = {"audio_feature_dim": 80, "audio_feature_channels": 1}
        trg_meta = {"vocab_size": vocab, "eos_id": vocab - 1, "bos_id": vocab - 2, "unk_id": vocab - 3}
        with torch.no_grad():
            model = SpeechTransformer.new(params, src_meta, trg_meta)
            # make every bias / LN parameter non-trivial so the fixtures exercise them
            g = torch.Generator().manual_seed(seed + 1)
            for p in _all_reference_params(model):
                if p.dim() == 1:
                    p.add_(0.1 * torch.randn(p.shape, generator=g))
        return model

    cases = [
        ("refpt_speech_toy", dict(d=8, heads=2, enc_layers=2, dec_layers=2, ffn_size=10, channels=5, vocab=12, seed=11),
         dict(B=3, T=37, L=5, lengths=[37, 30, 18])),
        ("refpt_speech_small", dict(d=64, heads=4, enc_layers=2, dec_layers=2, ffn_size=128, channels=64, vocab=96, seed=12),
         dict(B=2, T=50, L=7, lengths=[50, 41])),
    ]
    for name, mk, io in cases:
        model = build(**mk)
        g = torch.Generator().manual_seed(100 + mk["seed"])
        B, T, L = io["B"], io["T"], io["L"]
        src = torch.randn(B, T, 80, 1, generator=g)
        lengths = torch.tensor(io["lengths"], dtype=torch.long)
        for b in range(B):
            src[b, io["lengths"][b]:] = 0.0
        trg_input = torch.randint(0, mk["vocab"], (B, L), generator=g)
        with torch.no_grad():
            logits = model({"src": src.clone(), "src_length": lengths, "trg_input": trg_input}, is_training=False)
            sm = model._src_modality
            emb = sm(src.clone())
            conv = sm._embedding_layer(src.clone())
        P = pt_speech_transformer_params(model)
        big = {"P:" + k: v.astype(np.float32) for k, v in P.items() if v.size >= 32768}      # second file: no file above 1 MB
        if sum(v.nbytes for v in big.values()) > 400000:
            np.savez(os.path.join(OUT, name + "_part2.npz"), **big)
            P = {k: v for k, v in P.items() if "P:" + k not in big}
        np.savez(os.path.join(OUT, name + ".npz"), src=src.numpy(), src_length=lengths.numpy(),
                 trg_input=trg_input.numpy(), logits=logits.numpy(), emb=emb.numpy(), conv=conv.numpy(),
                 cfg=np.array([mk["d"], mk["heads"], mk["enc_layers"], mk["dec_layers"], mk["ffn_size"], mk["channels"],
                               mk["vocab"]]),
                 **{"P:" + k: v.astype(np.float32) for k, v in P.items()})
        print(name, "logits", tuple(logits.shape))


def make_interchange():
    """interchange_reference.json: what tests/test_interchange_cpu.py compares with when the reference tree is absent —
    the unmodified reference forward on the oracle's seeded weights (through the checkpoint weight map) and the reference's
    create_audio_bucket_boundaries for the tested (maxlen, minlen) pairs."""
    import ast
    import json
    import torch
    from oracle import build_ref, restatement as R
    from neurst_b200 import checkpoints as CK
    cfg = dict(model="speech", d=16, heads=2, enc_layers=2, dec_layers=2, ffn=24, channels=8, feat=80, in_channels=1, vocab=20)
    os.environ["NEURST_REFERENCE_SRC"] = REF
    model = build_ref.reference_speech_transformer(cfg, 20)
    P = R.init_params(cfg, seed=5, random_bias=True)
    CK.to_reference_pt(P, model)
    g = torch.Generator().manual_seed(0)
    src = torch.randn(2, 41, 80, 1, generator=g)
    lens = torch.tensor([41, 30]); ti = torch.randint(0, 17, (2, 5), generator=g)
    with torch.no_grad():
        ref = model({"src": src, "src_length": lens, "trg_input": ti}, is_training=False)
    tree = ast.parse(open(os.path.join(REF, "neurst/tasks/speech2text.py")).read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "create_audio_bucket_boundaries")
    ns = {"math": __import__("math")}
    exec(compile(ast.Module([fn], []), "ref", "exec"), ns)
    pairs = [(3000, 128), (2000, 100), (800, None), (3000, 300)]
    out = {"source": "unmodified reference neurst_pt SpeechTransformer forward / neurst.tasks.speech2text.create_audio_bucket_boundaries",
           "logits_shape": list(ref.shape), "logits": [float(x) for x in ref.reshape(-1).tolist()],
           "bucket_boundaries": [{"maxlen": a, "minlen": b, "boundaries": list(ns["create_audio_bucket_boundaries"](a, b))} for a, b in pairs]}
    with open(os.path.join(OUT, "interchange_reference.json"), "w") as f:
        json.dump(out, f)
    print("interchange_reference.json", tuple(ref.shape))


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    make_kats()
    make_refpt()
    make_interchange()
