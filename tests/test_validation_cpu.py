"""Validation during training, host side: the validator plan resolved from a training yaml plus a validation yaml, the
WER / BLEU / criterion metrics on hand-computed cases, the recorder with its keep-best and averaging savers over a fake
parameter table, and restoring from a directory whose `checkpoint` index names a kept-best archive."""
import json
import math
import os

import numpy as np
import pytest

from neurst_b200 import cli
from neurst_b200 import metrics as M
from neurst_b200 import validation as V
from tests.test_cli import _write_yaml

VALIDATION_YAML = """
validator.class: SeqGenerationValidator
validator.params:
  eval_dataset: AudioTFRecordDataset
  eval_dataset.params:
    data_path: DEV
    feature_key: audio
    transcript_key: translation
  eval_batch_size: 64
  eval_start_at: 6000
  eval_steps: 2000
  eval_criterion: label_smoothed_cross_entropy
  eval_search_method: beam_search
  eval_search_method.params:
    beam_size: 4
    length_penalty: -1
    maximum_decode_length: 150
  eval_metric: wer
  eval_top_checkpoints_to_keep: 10
  eval_auto_average_checkpoints: True
"""


def _cfg(tmp_path, *overrides, validation=VALIDATION_YAML):
    y = _write_yaml(tmp_path)
    paths = [y]
    if validation is not None:
        v = tmp_path / "validation.yml"
        v.write_text(validation)
        paths.append(str(v))
    return cli.load_config(paths, list(overrides))


def test_validator_plan_defaults_and_flags(tmp_path):
    plan = cli.resolve(_cfg(tmp_path, ("eval_steps", 500), ("eval_estop_patience", 3), ("eval_dataset.params.data_path", "DEV2")))
    vp = plan["validator"]
    assert vp["class"] == "SeqGenerationValidator"
    assert (vp["eval_steps"], vp["eval_start_at"], vp["eval_on_begin"], vp["batch_size"]) == (500, 6000, False, 64)
    assert vp["dataset"] == {"data_path": "DEV2", "feature_key": "audio", "transcript_key": "translation"}
    assert vp["criterion"] and vp["label_smoothing"] == 0.0          # the eval criterion's own default, not training's 0.1
    assert vp["search_method"] == "beam_search"
    assert vp["search"]["beam_size"] == 4 and vp["search"]["length_penalty"] == -1.0 and vp["search"]["maximum_decode_length"] == 150
    assert vp["metric"] == "wer" and vp["language"] == "de"
    assert (vp["estop_patience"], vp["top_checkpoints_to_keep"], vp["auto_average_checkpoints"]) == (3, 10, True)
    assert vp["best_checkpoint_path"] is None and vp["best_avg_checkpoint_path"] is None
    # the flat flags land in validator.params, nothing leaks into entry.params
    cfg = _cfg(tmp_path, ("eval_steps", 500))
    assert cfg["validator.params"]["eval_steps"] == 500 and "eval_steps" not in cfg["entry.params"]
    # the reference's defaults: a bare CriterionValidator under the alias key
    plan = cli.resolve(_cfg(tmp_path, validation="validator: CriterionValidator\nvalidator.params:\n  eval_dataset: AudioTFRecordDataset\n"
                                                 "  eval_dataset.params: {data_path: DEV}\n  eval_criterion: label_smoothed_cross_entropy\n"))
    vp = plan["validator"]
    assert vp["class"] == "CriterionValidator" and (vp["eval_steps"], vp["eval_start_at"], vp["batch_size"]) == (1000, 0, 32)
    assert vp["dataset"]["transcript_key"] == "transcript" and vp["metric"] is None


def test_plan_without_validator_is_unchanged(tmp_path):
    with_flag = cli.resolve(_cfg(tmp_path, ("eval_steps", 500), validation=None))
    plain = cli.resolve(_cfg(tmp_path, validation=None))
    assert "validator" not in plain and with_flag == plain


@pytest.mark.parametrize("extra, message", [
    ("validator.class: BleuValidator\n", "BleuValidator"),
    ("validator.params:\n  eval_metric: chrf\n", "chrf"),
    ("validator.params:\n  eval_metric: rouge\n", "rouge"),
    ("validator.params:\n  eval_search_method: sampling\n", "sampling"),
    ("validator.params:\n  eval_dataset: ParallelTextDataset\n", "ParallelTextDataset"),
    ("validator.params:\n  eval_criterion: cross_entropy\n", "cross_entropy"),
    ("validator.params:\n  eval_metric.params: {language: fr}\n", "eval_metric.params language"),
    # 100 utterances x beam 4 rows exceed the 256 a 16-bit decoding step holds: refused before training starts
    ("validator.params:\n  eval_batch_size: 100\n", "batch_size 100 x beam_size 4 exceeds the 256 rows"),
])
def test_validator_refusals(tmp_path, extra, message):
    import yaml
    cfg = cli.deep_merge(_cfg(tmp_path), yaml.safe_load(extra))
    with pytest.raises(SystemExit, match=message):
        cli.resolve(cfg)


def test_bleu_refuses_languages_it_does_not_tokenize(tmp_path):
    cfg = _cfg(tmp_path, ("eval_metric", "bleu"),
               ("task.params.transcript_data_pipeline.params", {"language": "zh", "vocab_path": str(tmp_path / "vocab.de")}))
    with pytest.raises(SystemExit, match="zh"):
        cli.resolve(cfg)


# ------------------------------------------------------------------------------------------------ metrics
def test_wer_counts_and_tie_order():
    w = M.Wer("en")
    # one substitution (b -> x) and one insertion (e) over 4 reference words
    r = w(["a x c d e"], ["a b c d"])
    assert r == {"WER": 50.0, "WER-substitutions": 25.0, "WER-insertions": 25.0, "WER-deletions": 0.0}
    # "a b" -> "b c": two substitutions or a deletion plus an insertion; `min` keeps the first of equal sums, and
    # substitution comes first
    assert M._wer(["a", "b"], ["b", "c"]) == (2.0, 0.0, 0.0)
    assert w(["b c"], ["a b"])["WER-substitutions"] == 100.0
    assert M._wer(["a", "b"], ["b"]) == (0.0, 0.0, 1.0)
    # normalisation: case, punctuation, apostrophe fix-ups, whitespace
    assert M.normalize_for_wer("en", "It' s  A Test, ok?") == "it's a test ok"
    assert w(["It' s a TEST ."], ["it's a test"])["WER"] == 0.0
    assert w.greater_or_eq({"WER": 10.0}, {"WER": 12.0}) and not w.greater_or_eq({"WER": 12.0}, {"WER": 10.0})
    c = M.Wer("zh")
    r = c(["你好 世"], ["你好世界"])                              # per character: one deletion over 4
    assert r["CER"] == 25.0 and r["CER-deletions"] == 25.0


def _edit_distance(ref, hyp):
    # plain Levenshtein distance, one row at a time
    row = list(range(len(hyp) + 1))
    for i, r in enumerate(ref, 1):
        prev, row[0] = row[0], i
        for j, h in enumerate(hyp, 1):
            prev, row[j] = row[j], min(row[j] + 1, row[j - 1] + 1, prev + (r != h))
    return row[-1]


def test_wer_operations_are_a_minimal_edit_script():
    rng = np.random.default_rng(3)
    for _ in range(300):
        ref = [str(x) for x in rng.integers(0, 4, rng.integers(0, 9))]
        hyp = [str(x) for x in rng.integers(0, 4, rng.integers(0, 9))]
        s, i, d = M._wer(ref, hyp)
        assert s + i + d == _edit_distance(ref, hyp) and len(ref) - d + i == len(hyp), (ref, hyp)


def test_tok_bleu_hand_computed():
    b = M.build_metric("tok_bleu", "en")
    hyps, refs = ["a b c d e", "x y"], ["a b c d f", "x y z"]
    # clipped n-gram precisions 6/7, 4/5, 2/3, 1/2; 7 hypothesis words against 8 reference words
    expect = math.exp(1 - 8 / 7) * (6 / 7 * 4 / 5 * 2 / 3 * 1 / 2) ** 0.25 * 100
    res = b(hyps, refs)
    assert res["tok_bleu"] == pytest.approx(expect, rel=1e-12)
    assert b.get_value(res) == res["tok_bleu"]
    # cased, no word matches (a zero precision scores 0); lowercased, every n-gram matches
    lc = M.build_metric("uncased_tok_bleu", "en")
    res = lc(["A B C D"], ["a b c d"])
    assert res["uncased_tok_bleu"] == pytest.approx(100.0) and res["tok_bleu"] == 0.0 and lc.get_value(res) == res["uncased_tok_bleu"]
    # unescape before counting: "&amp;" matches "&"
    assert M.tok_corpus_bleu(["a &amp; b c"], ["a & b c"]) < 1.0
    assert M.unescape("&amp;lt; &#91;x&#93; &quot;") == '< [x] "'          # "&amp;" first, as the reference does
    assert b(["a &amp; b c"], ["a & b c"])["tok_bleu"] == pytest.approx(100.0)


def test_sacre_bleu_13a_hand_computed():
    b = M.build_metric("bleu", "en")
    assert M.tokenize_13a("Hello, world.") == "Hello , world ."
    assert M.tokenize_13a("3.5 and 1,000 x-2 2-x") == "3.5 and 1,000 x-2 2 - x"     # a dash splits after a digit only
    # 3/4, 2/3, 1/2 and no matching 4-gram: the `exp` smoothing turns 0/1 into 100 / (2 * 1)
    expect = (75.0 * (200.0 / 3) * 50.0 * 50.0) ** 0.25
    res = b(["Hello, world."], ["Hello, world!"])
    assert res["sacre_bleu"] == pytest.approx(expect, rel=1e-12) and res["detok_bleu"] == res["sacre_bleu"]
    assert b.get_value(res) == res["sacre_bleu"]                 # eval_metric: bleu ranks by sacre_bleu
    cased = b(["HELLO big wide world"], ["hello big wide world"])
    assert cased["sacre_bleu"] < cased["uncased_sacre_bleu"] == pytest.approx(100.0)
    # brevity penalty: 2 words against 3, no 3- or 4-grams in the hypothesis
    short = M.sacre_corpus_bleu(["a b"], ["a b c"])
    assert short == 0.0
    # a one-word shortfall with all four orders present: brevity penalty exp(1 - 5/4) on 100 % precisions
    assert M.sacre_corpus_bleu(["a b c d"], ["a b c d e"]) == pytest.approx(100.0 * math.exp(1 - 5 / 4), rel=1e-12)
    assert M.sacre_corpus_bleu(["x"], ["y"]) == 0.0
    assert b.greater_or_eq({"sacre_bleu": 30.0}, {"sacre_bleu": 20.0})
    with pytest.raises(ValueError, match="chrf"):
        M.build_metric("uncased_chrf")


def test_criterion_metric():
    m = M.CriterionMetric()
    res = m.reduce(10.0, 4.0, 20.0)
    assert res == {"NLL": 2.5, "PPL": 2.0 ** 0.5}
    assert m.greater_or_eq({"NLL": 1.0}, {"NLL": 2.0}) and not m.greater_or_eq({"NLL": 2.0}, {"NLL": 1.0})


# ------------------------------------------------------------------------------------------------ recorder and savers
def _snapshot(step):
    g = np.random.default_rng(step)
    return {"SpeechTransformer/w": g.standard_normal((3, 4)).astype(np.float32), "SpeechTransformer/b": g.standard_normal(5).astype(np.float32)}


def _best_n(values, n, lower_better):
    order = sorted(values.items(), key=lambda kv: kv[1], reverse=not lower_better)
    return [s for s, _ in order[:n]]


@pytest.mark.parametrize("name, key, values, lower_better", [
    ("wer", "WER", [50.0, 40.0, 45.0, 30.0, 60.0, 35.0, 70.0, 80.0], True),
    ("bleu", "sacre_bleu", [10.0, 20.0, 15.0, 25.0, 5.0, 22.0, 3.0, 2.0], False),
])
def test_recorder_keeps_best_and_averages(tmp_path, name, key, values, lower_better):
    metric = M.build_metric(name, "en")
    written = []
    rec = V.TrainingStatusRecorder(metric, str(tmp_path), estop_patience=3, top_checkpoints_to_keep=3,
                                   model_configs=lambda d: written.append(d))
    assert written == [str(tmp_path / "best"), str(tmp_path / "best_avg")]
    seen, stops = {}, []
    for i, v in enumerate(values):
        step = 4 * (i + 1)
        seen[step] = v
        before = set(os.listdir(tmp_path / "best_avg"))
        stops.append(rec.record(step, {key: v}, lambda: _snapshot(step)))
        added = set(os.listdir(tmp_path / "best_avg")) - before - {"checkpoint"}
        for f in added:                                   # best_avg: np.average over the last 3 evaluated snapshots
            z = np.load(str(tmp_path / "best_avg" / f))
            last = [_snapshot(s) for s in sorted(seen)[-3:]]
            for k in z.files:
                assert np.array_equal(z[k], np.average([s[k] for s in last], axis=0))
            assert f == "ckpt-%d-%.2f.npz" % (step, v)
    best_steps = _best_n(seen, 3, lower_better)
    files = sorted(f for f in os.listdir(tmp_path / "best") if f.endswith(".npz"))
    assert files == sorted("ckpt-%d-%.2f.npz" % (s, seen[s]) for s in best_steps)
    idx = json.load(open(tmp_path / "best" / "checkpoint"))
    assert idx["model_checkpoint_path"] == "ckpt-%d-%.2f.npz" % (best_steps[0], seen[best_steps[0]])
    z = np.load(str(tmp_path / "best" / idx["model_checkpoint_path"]))
    assert all(np.array_equal(z[k], _snapshot(best_steps[0])[k]) for k in z.files)
    # the best value comes at evaluation 4; evaluations 5, 6, 7 bring no improvement: patience 3 stops at the 7th
    assert stops == [False] * 6 + [True, True]
    assert rec.best == {key: seen[best_steps[0]]}
    avg_idx = json.load(open(tmp_path / "best_avg" / "checkpoint"))
    assert avg_idx["model_checkpoint_path"] == "ckpt-%d-%.2f.npz" % (best_steps[0], seen[best_steps[0]])


def test_recorder_without_savers(tmp_path):
    rec = V.TrainingStatusRecorder(M.CriterionMetric())
    assert rec.best_saver is None and rec.avg_saver is None
    assert not rec.record(1, {"NLL": 3.0, "PPL": 4.0}) and not rec.record(2, {"NLL": 4.0, "PPL": 5.0})
    assert rec.best == {"NLL": 3.0, "PPL": 4.0} and rec.bad_count == 1
    V.TrainingStatusRecorder(M.build_metric("wer"), str(tmp_path), top_checkpoints_to_keep=2, auto_average_checkpoints=False)
    assert os.listdir(tmp_path) == ["best"]


def test_restore_from_the_checkpoint_index(tmp_path):
    assert cli.restore_checkpoint(str(tmp_path)) == (None, 0)
    for name in ("ckpt-8-12.34.npz", "ckpt-12-15.00.npz", "ckpt-16.npz"):
        (tmp_path / name).write_bytes(b"")
    (tmp_path / "checkpoint").write_text(json.dumps({"model_checkpoint_path": "ckpt-8-12.34.npz",
                                                     "all_model_checkpoint_paths": ["ckpt-12-15.00.npz", "ckpt-8-12.34.npz"]}))
    p, s = cli.restore_checkpoint(str(tmp_path))
    assert s == 8 and p == str(tmp_path / "ckpt-8-12.34.npz")
    os.remove(str(tmp_path / "ckpt-8-12.34.npz"))                  # the index names a missing file: newest-step glob
    p, s = cli.restore_checkpoint(str(tmp_path))
    assert s == 16 and p.endswith("ckpt-16.npz")
    assert cli.latest_checkpoint(str(tmp_path))[1] == 16             # unchanged
