"""Machine translation on the text Transformer, host side: plans of the seq2seq task, the text hparams sets, the
processed-text data path, token buckets, checkpoint names and pattern-based pretraining."""
import os

import numpy as np
import pytest
import torch

from neurst_b200 import checkpoints as CK
from neurst_b200 import cli
from neurst_b200.data import (Seq2Seq, TokenBucketer, adjust_batch_size, associated_bucket_boundaries,
                              create_batch_bucket_boundaries)
from neurst_b200.models import Transformer, speech_transformer_hparams, transformer_hparams
from neurst_b200.text import ParallelTextDataset

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _vocab(path, tokens):
    with open(path, "w", encoding="utf-8") as f:
        f.write("".join(t + "\t1\n" for t in tokens))
    return str(path)


def _mt_cfg(tmp_path, src_tokens=("a", "b", "c@@", "d"), trg_tokens=("x", "y", "z"), **extra):
    src = tmp_path / "train.src"
    trg = tmp_path / "train.trg"
    src.write_text("a  b\nc@@ d a\n")
    trg.write_text("x y\n  z   x\n")
    cfg = {"entry.class": "trainer", "task.class": "seq2seq",
           "task.params": {"batch_by_tokens": True, "batch_size": 25000, "max_src_len": 120, "max_trg_len": 150,
                           "src_data_pipeline.params": {"vocab_path": _vocab(tmp_path / "vocab.src", src_tokens)},
                           "trg_data_pipeline.params": {"vocab_path": _vocab(tmp_path / "vocab.trg", trg_tokens),
                                                        "language": "de"}},
           "dataset.class": "ParallelTextDataset",
           "dataset.params": {"src_file": str(src), "trg_file": str(trg), "data_is_processed": True},
           "hparams_set": "transformer_s"}
    cfg.update(extra)
    return cfg


# ------------------------------------------------------------------------------------------------ plans
@pytest.mark.parametrize("name", ["seq_to_seq", "Seq2Seq", "seq2seq", "SeqToSeq"])
def test_seq2seq_task_names_resolve_to_the_text_plan(tmp_path, name):
    plan = cli.resolve(_mt_cfg(tmp_path, **{"task.class": name}))
    assert plan["model_class"] == "Transformer"
    assert plan["model_params"]["encoder.hidden_size"] == 256 and plan["model_params"]["encoder.num_layers"] == 6
    assert plan["lr_schedule"] == {"initial_factor": 1.0, "dmodel": 256, "warmup_steps": 4000}
    assert plan["task"] == {"max_src_len": 120, "max_trg_len": 150, "truncate_src": False, "truncate_trg": False,
                            "batch_size": 25000, "batch_size_per_gpu": None, "batch_by_tokens": True}
    assert plan["dataset"]["data_is_processed"] is True and plan["dataset"]["src_file"].endswith("train.src")
    assert plan["src_meta"]["vocab_size"] == 7 and plan["trg_meta"]["vocab_size"] == 6


def test_text_plan_defaults_and_model_class(tmp_path):
    cfg = _mt_cfg(tmp_path)
    del cfg["hparams_set"]
    plan = cli.resolve(dict(cfg, **{"model.class": "Transformer"}))
    assert plan["model_params"] == transformer_hparams("transformer_s")["model.params"]
    assert plan["precision"] == "fp16" and plan["label_smoothing"] == 0.1


def test_text_plan_refusals(tmp_path):
    with pytest.raises(SystemExit, match="raw text"):
        cli.resolve(_mt_cfg(tmp_path, **{"dataset.params": {"src_file": "s", "trg_file": "t"}}))
    with pytest.raises(SystemExit, match="ParallelTextDataset only"):
        cli.resolve(_mt_cfg(tmp_path, **{"dataset.class": "AudioTFRecordDataset"}))
    with pytest.raises(SystemExit, match="Transformer only"):
        cli.resolve(_mt_cfg(tmp_path, **{"model.class": "SpeechTransformer"}))
    with pytest.raises(SystemExit, match="SpeechTransformer preset"):
        cli.resolve(_mt_cfg(tmp_path, hparams_set="speech_transformer_s"))
    for extra in ({}, {"model.class": "SpeechTransformer"}):
        with pytest.raises(SystemExit, match="Transformer preset"):
            cli.resolve(dict({"task.class": "SpeechToText", "hparams_set": "transformer_s",
                              "task.params": {"batch_size": 1000, "vocab_size": 8}}, **extra))
    with pytest.raises(SystemExit, match="AudioTFRecordDataset only"):
        cli.resolve({"task.class": "SpeechToText", "dataset.class": "ParallelTextDataset",
                     "task.params": {"batch_size": 1000, "vocab_size": 8}})
    cfg = _mt_cfg(tmp_path)
    cfg["task.params"] = dict(cfg["task.params"], **{"src_data_pipeline.params": {"vocab_path": str(tmp_path / "none")}})
    with pytest.raises(SystemExit, match="src_data_pipeline.params.vocab_path"):
        cli.resolve(cfg)
    cfg = _mt_cfg(tmp_path)
    cfg["task.params"] = {k: v for k, v in cfg["task.params"].items() if k != "batch_size"}
    with pytest.raises(SystemExit, match="batch_size"):
        cli.resolve(cfg)
    with pytest.raises(SystemExit, match="unknown hparams_set"):
        cli.resolve(_mt_cfg(tmp_path, hparams_set="transformer_xl"))


def test_shared_source_target_embedding_needs_identical_vocabularies(tmp_path):
    share = {"model.params": {"modality.share_source_target_embedding": True}}
    with pytest.raises(SystemExit, match="identical"):
        cli.resolve(_mt_cfg(tmp_path, **share))
    plan = cli.resolve(_mt_cfg(tmp_path, src_tokens=("x", "y", "z"), **share))
    assert plan["model_params"]["modality.share_source_target_embedding"] is True


def test_text_validator_plan(tmp_path):
    cfg = _mt_cfg(tmp_path, **{"validator.class": "SeqGenerationValidator", "validator.params": {
        "eval_dataset": "ParallelTextDataset",
        "eval_dataset.params": {"src_file": "dev.src", "trg_file": "dev.trg", "data_is_processed": True},
        "eval_batch_size": 64, "eval_search_method": "beam_search", "eval_metric": "tok_bleu"}})
    vp = cli.resolve(cfg)["validator"]
    assert vp["dataset"] == {"src_file": "dev.src", "trg_file": "dev.trg", "data_is_processed": True}
    assert vp["metric"] == "tok_bleu" and vp["language"] == "de"
    cfg["validator.params"]["eval_dataset.params"] = {"src_file": "dev.src", "trg_file": "dev.trg"}
    with pytest.raises(SystemExit, match="raw text"):
        cli.resolve(cfg)


def test_speech_plan_is_unchanged_by_the_text_path():
    plan = cli.resolve({"task.params": {"batch_size": 1000, "vocab_size": 8}})
    assert plan["model_class"] == "SpeechTransformer" and "src_meta" not in plan
    assert "pretrain_variable_pattern" not in plan
    assert plan["model_params"] == speech_transformer_hparams("speech_transformer_s")["model.params"]


def test_pretrain_patterns_from_the_command_line():
    paths, over = cli.parse_command_line(["--pretrain_model", "asr/best_avg", "mt/best_avg", "--pretrain_variable_pattern",
                                          "(TransformerEncoder)|(input_audio)", "(TransformerDecoder)|(target_symbol)"])
    cfg = cli.load_config(paths, over)
    cfg["task.params"] = {"batch_size": 1000, "vocab_size": 8}
    plan = cli.resolve(cfg)
    assert plan["pretrain_model"] == ["asr/best_avg", "mt/best_avg"]
    assert plan["pretrain_variable_pattern"] == ["(TransformerEncoder)|(input_audio)", "(TransformerDecoder)|(target_symbol)"]
    with pytest.raises(SystemExit, match="must match"):
        cli.resolve(dict(cfg, **{"entry.params": {"pretrain_model": ["a", "b"], "pretrain_variable_pattern": "x"}}))
    with pytest.raises(SystemExit, match="unexpected argument"):
        cli.parse_command_line(["--config_paths", "a.yml", "b.yml"])


def test_model_configs_record_the_text_class(tmp_path):
    plan = dict(cli.resolve(_mt_cfg(tmp_path)), model_dir=str(tmp_path / "m"))
    cli.write_model_configs(plan)
    assert cli.member_model_params(plan, plan["model_dir"]) == plan["model_params"]
    speech = dict(cli.resolve({"task.params": {"batch_size": 1000, "vocab_size": 8}}), model_dir=str(tmp_path / "s"))
    cli.write_model_configs(speech)
    with pytest.raises(SystemExit, match="Transformer only"):
        cli.member_model_params(plan, speech["model_dir"])
    with pytest.raises(SystemExit, match="SpeechTransformer only"):
        cli.member_model_params(speech, plan["model_dir"])


# ------------------------------------------------------------------------------------------------ hparams
def _expected(d, heads, enc, dec, ffn, rate):
    p = {"modality.share_source_target_embedding": False, "modality.share_embedding_and_softmax_weights": True,
         "modality.dim": d, "modality.timing": "sinusoids"}
    for side, n in (("encoder", enc), ("decoder", dec)):
        p.update({side + ".num_layers": n, side + ".hidden_size": d, side + ".num_attention_heads": heads,
                  side + ".filter_size": ffn, side + ".attention_dropout_rate": rate, side + ".attention_type": "dot_product",
                  side + ".ffn_activation": "relu", side + ".ffn_dropout_rate": rate, side + ".post_normalize": False,
                  side + ".layer_postprocess_dropout_rate": rate})
    return {"model.class": "Transformer", "model.params": p, "optimizer.class": "Adam",
            "optimizer.params": {"epsilon": 1.e-9, "beta_1": 0.9, "beta_2": 0.98}, "lr_schedule.class": "noam",
            "lr_schedule.params": {"initial_factor": 1.0, "dmodel": d, "warmup_steps": 4000}}


@pytest.mark.parametrize("name,expect", [
    ("transformer_toy", (8, 2, 2, 2, 10, 0.1)), ("transformer_base", (512, 8, 6, 6, 2048, 0.1)),
    ("transformer_s", (256, 4, 6, 6, 2048, 0.1)), ("transformer_big", (1024, 16, 6, 6, 4096, 0.3)),
    ("transformer_big_dp01", (1024, 16, 6, 6, 4096, 0.1)), ("transformer_512_6e_3d", (512, 8, 6, 3, 2048, 0.1)),
    ("transformer_256_12e_6d_4h", (256, 4, 12, 6, 1024, 0.1)), ("transformer_384_3e_3d_dp0.3", (384, 8, 3, 3, 1536, 0.3)),
    ("transformer_128_2e_1d_2h_dp0.05", (128, 2, 2, 1, 512, 0.05))])
def test_text_hparams_sets_equal_the_reference_table(name, expect):
    assert transformer_hparams(name) == _expected(*expect)
    assert Transformer.build_model_args_by_name(name) == _expected(*expect)


def test_unknown_and_invalid_text_hparams():
    assert transformer_hparams("transformer_m") is None and transformer_hparams("speech_transformer_s") is None
    assert speech_transformer_hparams("transformer_s") is None
    with pytest.raises(ValueError, match="divisible"):
        transformer_hparams("transformer_100_2e_2d_8h")


# ------------------------------------------------------------------------------------------------ text data
def test_vocab_metas_of_both_sides(tmp_path):
    plan = cli.resolve(_mt_cfg(tmp_path))
    sm, tm = plan["src_meta"], plan["trg_meta"]
    assert sm["tokens"] == ["a", "b", "c@@", "d"]
    assert (sm["vocab_size"], sm["unk_id"], sm["bos_id"], sm["eos_id"], sm["pad_id"]) == (7, 4, 5, 6, 6)
    assert tm["tokens"] == ["x", "y", "z"]
    assert (tm["vocab_size"], tm["unk_id"], tm["bos_id"], tm["eos_id"], tm["pad_id"]) == (6, 3, 4, 5, 5)


def test_reader_collapses_whitespace_and_shards_as_the_reference(tmp_path):
    src, trg = tmp_path / "s", tmp_path / "t"
    src.write_text("".join(" w%d \t v%d\n" % (i, i) for i in range(1, 8)))
    trg.write_text("".join("u%d  \n" % i for i in range(1, 8)))
    ds = ParallelTextDataset({"src_file": str(src), "trg_file": str(trg), "data_is_processed": True})
    rows = list(ds.build_iterator()())
    assert rows[0] == {"feature": "w1 v1", "label": "u1"} and len(rows) == 7 and ds.num_samples == 7
    # 7 lines, 3 shards: 2 per shard; 1-based line n goes to shard k when k*2 <= n < (k+1)*2, the last shard to the end
    parts = [[r["label"] for r in ds.build_iterator(shard_id=k, total_shards=3)()] for k in range(3)]
    assert parts == [["u1"], ["u2", "u3"], ["u4", "u5", "u6", "u7"]]


def test_processed_text_encoding_with_eos_unk_and_truncation(tmp_path):
    plan = cli.resolve(_mt_cfg(tmp_path, **{"task.params": dict(_mt_cfg(tmp_path)["task.params"], truncate_src=True,
                                                                max_src_len=3)}))
    task = Seq2Seq(plan["src_meta"], plan["trg_meta"], **plan["task"])
    data = {"feature": "a b q c@@ d", "label": "z w"}
    train = task.preprocess_fn({"feature": "processed", "label": "processed"}, training=True)(data)
    assert train["feature"].tolist() == [0, 1, 6]                 # truncated: first max_len - 1 tokens + EOS
    assert train["transcript"].tolist() == [2, 3, 5]               # "w" is UNK, EOS appended
    ev = task.preprocess_fn({"feature": "processed", "label": "processed"}, training=False)(data)
    assert ev["feature"].tolist() == [0, 1, 4, 2, 3, 6]            # no truncation outside training; "q" is UNK
    infer = task.preprocess_fn({"feature": "processed"}, training=False, with_label=False)(data)
    assert set(infer) == {"feature"}
    with pytest.raises(RuntimeError, match="BPE"):
        task.preprocess_fn({"feature": "raw", "label": "raw"}, training=True)


def test_eval_batches_keep_order_and_pad_to_the_longest(tmp_path):
    plan = cli.resolve(_mt_cfg(tmp_path))
    task = Seq2Seq(plan["src_meta"], plan["trg_meta"], **plan["task"])
    group = [{"feature": torch.tensor([0, 6]), "transcript": torch.tensor([0, 1, 5])},
             {"feature": torch.tensor([1, 2, 3, 6]), "transcript": torch.tensor([5])}]
    b = task.group_to_input(group, infer=False)
    assert b["src"].tolist() == [[0, 6, 6, 6], [1, 2, 3, 6]]
    assert b["src_padding"].tolist() == [[0, 0, 1, 1], [0, 0, 0, 0]]
    assert b["trg"].tolist() == [[0, 1, 5], [5, 5, 5]] and b["trg_length"].tolist() == [3, 1]
    assert b["trg_input"].tolist() == [[4, 0, 1], [4, 5, 5]]
    i = task.group_to_input(group, infer=True)
    assert set(i) == {"src", "src_padding", "trg_input"} and i["trg_input"].tolist() == [4, 4]


# ------------------------------------------------------------------------------------------------ token buckets
def test_bucket_boundaries_hand_worked():
    assert create_batch_bucket_boundaries(10) == [8, 9, 11]
    assert create_batch_bucket_boundaries(20) == [8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 21]
    assert create_batch_bucket_boundaries(5) == [6]
    a, b = associated_bucket_boundaries([8, 9, 11], create_batch_bucket_boundaries(20))
    assert (a, b) == ([8, 9, 11], [12, 16, 21])
    assert adjust_batch_size(100, bucket_boundaries={"feature": a, "label": b}, num_replicas_in_sync=2) == [8, 6, 4]
    assert adjust_batch_size(101, num_replicas_in_sync=2) == 100
    assert adjust_batch_size(None, 30, bucket_boundaries={"feature": a, "label": b}, num_replicas_in_sync=2) == [4, 2, 2]


def test_token_bucketer_batches_and_shapes():
    b = TokenBucketer(10, 20, batch_size=100, batch_by_tokens=True, world=2)
    assert b.src_bounds == [8, 9, 11] and b.trg_bounds == [12, 16, 21] and b.batch_sizes == [8, 6, 4]
    assert b.shapes() == [(8, 4, 12), (9, 3, 16), (11, 2, 21)]
    assert b.bucket_of(8, 12) == 0 and b.bucket_of(8, 13) == 1 and b.bucket_of(10, 3) == 2 and b.bucket_of(12, 3) is None

    def ex(n, m, tag):
        return {"feature": torch.full((n,), tag), "transcript": torch.full((m,), tag)}
    stream = [ex(10, 2, i) for i in range(3)] + [ex(3, 3, 10 + i) for i in range(8)] + [ex(10, 2, 3)]
    out = list(b.batches(stream))
    assert [k for k, _ in out] == [0, 2]                        # a bucket leaves when its global batch is full
    assert [int(e["feature"][0]) for e in out[0][1][0]] == [10, 12, 14, 16]
    assert [int(e["feature"][0]) for e in out[0][1][1]] == [11, 13, 15, 17]
    assert [len(g) for g in out[1][1]] == [2, 2]
    with pytest.raises(ValueError, match="fewer than one pair"):
        TokenBucketer(10, 20, batch_size=20, batch_by_tokens=True, world=2)
    assert TokenBucketer(10, 20, batch_size=6, world=2).batch_sizes == [6, 6, 6]


def test_train_batches_drop_long_pairs_and_pad_to_the_bucket(tmp_path):
    plan = cli.resolve(_mt_cfg(tmp_path))
    tp = dict(plan["task"], max_src_len=10, max_trg_len=20, batch_size=24, batch_by_tokens=True)
    task = Seq2Seq(plan["src_meta"], plan["trg_meta"], world=1, **tp)
    exs = [{"feature": torch.tensor([0, 1, 6]), "transcript": torch.tensor([0, 5])} for _ in range(3)]
    exs.insert(1, {"feature": torch.arange(11), "transcript": torch.tensor([0, 5])})          # too long: dropped
    exs.insert(2, {"feature": torch.tensor([6]), "transcript": torch.tensor([0, 5])})         # empty source: dropped
    (batch,), = list(task.train_batches(exs[:5]))[:1] or [(None,)]
    assert batch["src"].shape == (2, 8) and batch["trg"].shape == (2, 12)   # 24 tokens // max(8, 12) = 2 pairs
    assert batch["src"][0].tolist() == [0, 1, 6, 6, 6, 6, 6, 6] and batch["src_padding"][0].tolist() == [0, 0, 0] + [1] * 5


# ------------------------------------------------------------------------------------------------ checkpoints
def _text_table(share):
    from oracle import restatement as R
    cfg = dict(model="text", d=8, heads=2, enc_layers=2, dec_layers=2, ffn=10, vocab=8, src_vocab=8, share_src_trg=share)
    return R.param_shapes(cfg)


def test_text_variable_names_match_the_reference_kat():
    z = np.load(os.path.join(GOLDEN, "kat_transformer.npz"))
    kat = [k[2:] for k in z.files if k.startswith("w:")]
    names = CK.tf_variable_names(_text_table(False))
    assert all(v.startswith("Transformer/") for v in names.values())
    for k in kat:                                                   # every reference variable has our tensor
        assert any(v.endswith("/" + k) for v in names.values()), k
    assert names["srcemb.emb"] == "Transformer/input_symbol_modality_posenc_wrapper/input_symbol_modality/emb/weights"
    assert names["trg.emb"] == "Transformer/target_symbol_modality_posenc_wrapper/target_symbol_modality/shared/weights"
    assert names["trg.bias"].endswith("target_symbol_modality/shared/bias")
    tied = CK.tf_variable_names(_text_table(True))
    assert "srcemb.emb" not in tied
    assert tied["trg.emb"] == "Transformer/shared_symbol_modality_posenc_wrapper/shared_symbol_modality/shared/weights"
    assert tied["trg.bias"].endswith("shared_symbol_modality/shared/bias")
    assert len(set(names.values())) == len(names)


class _FakeRT:
    def __init__(self, shapes, fill):
        self.table, off = {}, 0
        for k, shp in shapes.items():
            self.table[k] = (off, tuple(shp))
            off += int(np.prod(shp))
        self.params = torch.full((off,), float(fill))
        self.adam_m = self.adam_v = None

    def view(self, name, arena=None):
        off, shp = self.table[name]
        return (self.params if arena is None else arena)[off:off + int(np.prod(shp))].view(*shp)


def test_pretrain_patterns_select_tensors_per_archive(tmp_path):
    from oracle import restatement as R
    st_shapes = R.param_shapes(R.CONFIGS["speech_transformer_toy"])
    mt_shapes = {k: v for k, v in _text_table(False).items()}
    mt_shapes["trg.emb"], mt_shapes["trg.bias"] = st_shapes["trg.emb"], st_shapes["trg.bias"]
    for k in list(mt_shapes):          # the MT stack shaped as the ST one (same d, ffn, layer counts)
        if k in st_shapes:
            mt_shapes[k] = st_shapes[k]
    mt_shapes = {k: v for k, v in mt_shapes.items() if k in st_shapes or k == "srcemb.emb"}
    asr, mt, st = _FakeRT(st_shapes, 1.0), _FakeRT(mt_shapes, 2.0), _FakeRT(st_shapes, 0.0)
    CK.save_npz(asr, str(tmp_path / "asr.npz"))
    CK.save_npz(mt, str(tmp_path / "mt.npz"))
    got_asr = CK.load_npz(st, str(tmp_path / "asr.npz"), strict=False, pattern="(TransformerEncoder)|(input_audio)")
    got_mt = CK.load_npz(st, str(tmp_path / "mt.npz"), strict=False, pattern="(TransformerDecoder)|(target_symbol)")
    assert got_asr == sorted(k for k in st_shapes if k.startswith(("enc.", "src.")))
    assert got_mt == sorted(k for k in st_shapes if k.startswith(("dec.", "trg.")))
    for k in st_shapes:
        assert float(st.view(k).flatten()[0]) == (1.0 if k.startswith(("enc.", "src.")) else 2.0), k
    # no pattern: every name found (the previous behaviour)
    st2 = _FakeRT(st_shapes, 0.0)
    assert CK.load_npz(st2, str(tmp_path / "asr.npz"), strict=False) == sorted(st_shapes)
