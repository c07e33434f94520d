"""Validation during training on the device, through the training entry, on the tiny-model TFRecord setup of
tests/test_cli.py: the dev loss against the fp64 oracle on the same checkpoint, the hypotheses against `predict`, the
metric against the host metric, best/ and best_avg/ against the host recorder replayed on the logged metrics, the
training's random streams untouched by validation, restoring from best_avg/, and early stopping."""
import json
import os

import numpy as np
import pytest
import torch

from neurst_b200 import checkpoints as CK
from neurst_b200 import cli
from neurst_b200 import metrics as M
from neurst_b200 import validation as V
from oracle import restatement as R
from tests.test_cli import _write_dataset, _write_yaml

pytestmark = pytest.mark.gpu

TINY = {"encoder.num_layers": 2, "decoder.num_layers": 2, "encoder.hidden_size": 128, "decoder.hidden_size": 128, "modality.dim": 128,
        "encoder.num_attention_heads": 2, "decoder.num_attention_heads": 2, "encoder.filter_size": 256, "decoder.filter_size": 256,
        "modality.source.channels": 64}
ORACLE_CFG = dict(model="speech", d=128, heads=2, enc_layers=2, dec_layers=2, ffn=256, channels=64, feat=80, in_channels=1, vocab=96)
# per-token loss tolerances of the precision modes (smoke(): fp32 at the reference's 1e-4, fp16 on the 16-bit weights 5e-3)
TOL = {"fp32": 1e-4, "fp16": 5e-3}
EVAL_BATCH, BEAM, MAX_LEN = 8, 2, 12


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    root = tmp_path_factory.mktemp("validation")
    _write_dataset(root, vocab=93)                                  # 93 tokens + 3 symbols = 96 (the 16-bit path needs % 8)
    dev = root / "dev"
    dev.mkdir()
    _write_dataset(dev, n_shards=1, per_shard=20, vocab=93)
    return root, _write_yaml(root, data=str(root / "train.tfrecords"), n_tokens=93), str(dev / "train.tfrecords")


def _plan(data, model_dir, dtype, steps, **validator):
    root, y, dev = data
    vp = {"eval_dataset": "AudioTFRecordDataset", "eval_dataset.params": {"data_path": dev, "transcript_key": "translation"},
          "eval_batch_size": EVAL_BATCH, "eval_steps": 4, "eval_criterion": "label_smoothed_cross_entropy",
          "eval_search_method": "beam_search", "eval_search_method.params": {"beam_size": BEAM, "maximum_decode_length": MAX_LEN},
          "eval_metric": "wer", "eval_top_checkpoints_to_keep": 2}
    vp.update(validator)
    ov = [("model_dir", model_dir), ("dtype", dtype), ("task.params.batch_size", 3000), ("task.params.max_src_len", 400),
          ("task.params.max_trg_len", 24), ("task.params.experimental_frame_transcript_ratio", 20), ("save_checkpoint_steps", 4),
          ("summary_steps", 100), ("train_steps", steps)] + [("model.params." + k, v) for k, v in TINY.items()]
    cfg = cli.load_config([y], ov)
    if vp.get("validator", True):
        cfg["validator.class"] = "SeqGenerationValidator"
        cfg["validator.params"] = {k: v for k, v in vp.items() if k != "validator"}
    return cli.resolve(cfg)


def _dev_batches(plan):
    vp = plan["validator"]
    _, ex = cli._examples(dict(plan, dataset=vp["dataset"]), 0, 1, training=False, with_label=True)
    ex = list(ex)
    return ex, [ex[i:i + EVAL_BATCH] for i in range(0, len(ex), EVAL_BATCH)]


def _oracle_nll(plan, ckpt, batches):
    """fp64 restatement on the checkpoint's fp32 weights: sum(nll) / samples and tokens / samples, label smoothing 0 (the
    eval criterion's default)."""
    model = cli._build_model(dict(plan, precision="fp32"))
    CK.load_npz(model.runtime, ckpt)
    P = {k: model.runtime.view(k).detach().cpu().double() for k in model.runtime.table}
    pad = plan["trg_meta"]["pad_id"]
    nll = ntok = n = 0.0
    for g in batches:
        T, Lq = max(int(e["audio_length"]) for e in g), max(e["transcript"].numel() for e in g)
        src = torch.zeros(len(g), T, 80, 1, dtype=torch.float64)
        trg = torch.full((len(g), Lq), pad, dtype=torch.long)
        for j, e in enumerate(g):
            src[j, :int(e["audio_length"]), :, 0] = e["audio"]
            trg[j, :e["transcript"].numel()] = e["transcript"]
        length = torch.tensor([e["transcript"].numel() for e in g])
        trg_input = torch.cat([torch.full((len(g), 1), plan["trg_meta"]["bos_id"]), trg[:, :-1]], 1)
        logits = R.speech_transformer_forward(P, ORACLE_CFG, src, torch.tensor([int(e["audio_length"]) for e in g]), trg_input)
        s, _, t = R.label_smoothed_ce(logits, trg, length, 0.0)
        nll, ntok, n = nll + float(s.sum()), ntok + float(t.sum()), n + len(g)
    return nll / n, ntok / n


def _params(path):
    z = np.load(path)
    return {k: z[k] for k in z.files if "/.OPTIMIZER_SLOT/" not in k}


@pytest.mark.parametrize("dtype, precision", [("float32", "fp32"), ("float16", "fp16")])
def test_validation_during_training(data, tmp_path, dtype, precision):
    root, _, _ = data
    model_dir = str(tmp_path / "run")
    plan = _plan(data, model_dir, dtype, 12)
    res = cli.train(plan)
    vals = res["validations"]
    assert res["global_step"] == 12 and not res["early_stopped"] and [v["step"] for v in vals] == [4, 8, 12]
    examples, batches = _dev_batches(plan)
    tm = plan["trg_meta"]
    refs = [cli.ids_to_text(e["transcript"].tolist(), tm["eos_id"], tm["tokens"]) for e in examples]
    for v in vals:
        ckpt = os.path.join(model_dir, "ckpt-%d.npz" % v["step"])
        # dev loss: the fp64 oracle on the step's regular checkpoint
        nll, tok_per_sentence = _oracle_nll(plan, ckpt, batches)
        assert abs(v["loss"]["NLL"] - nll) <= TOL[precision] * tok_per_sentence, (v["step"], v["loss"], nll)
        assert v["loss"]["PPL"] == pytest.approx(2.0 ** (nll / tok_per_sentence), rel=TOL[precision] * 10)
        # hypotheses: `predict` on the same checkpoint with the same batch settings
        one = tmp_path / ("at%d" % v["step"])
        one.mkdir()
        os.link(ckpt, str(one / os.path.basename(ckpt)))
        vp = plan["validator"]
        got = cli.predict(dict(plan, entry="predict", model_dir=str(one), dataset=vp["dataset"], search_method=vp["search_method"],
                               search=vp["search"], batch_size=EVAL_BATCH, output_file=None))
        assert got["checkpoint_step"] == v["step"]
        assert v["hypotheses"] == [t for t, _ in got["hypotheses"]] and len(v["hypotheses"]) == 20
        # the metric: the host metric over those strings
        assert v["metric"] == M.build_metric("wer", "de")(v["hypotheses"], refs)
    # best/ and best_avg/: the host recorder replayed on the logged metrics and the regular checkpoints' weights
    replay = tmp_path / "replay"
    rec = V.TrainingStatusRecorder(M.build_metric("wer", "de"), str(replay), estop_patience=0, top_checkpoints_to_keep=2)
    for v in vals:
        rec.record(v["step"], v["metric"], lambda: _params(os.path.join(model_dir, "ckpt-%d.npz" % v["step"])))
    for sub in ("best", "best_avg"):
        mine, theirs = os.path.join(model_dir, sub), str(replay / sub)
        assert sorted(os.listdir(mine)) == sorted(os.listdir(theirs) + ["model_configs.yml"])
        assert json.load(open(os.path.join(mine, "checkpoint"))) == json.load(open(os.path.join(theirs, "checkpoint")))
        for f in os.listdir(theirs):
            if f.endswith(".npz"):
                a, b = np.load(os.path.join(mine, f)), np.load(os.path.join(theirs, f))
                assert sorted(a.files) == sorted(b.files) and all(np.array_equal(a[k], b[k]) for k in a.files)
    # best_avg's newest file: np.average over the regular checkpoints of the last two evaluations
    idx = json.load(open(os.path.join(model_dir, "best_avg", "checkpoint")))
    for f in idx["all_model_checkpoint_paths"]:
        step = int(f.split("-")[1])
        prev = [s for s in (4, 8, 12) if s <= step][-2:]
        z = np.load(os.path.join(model_dir, "best_avg", f))
        snaps = [_params(os.path.join(model_dir, "ckpt-%d.npz" % s)) for s in prev]
        assert all(np.array_equal(z[k], np.average([s[k] for s in snaps], axis=0)) for k in z.files)
    torch.cuda.synchronize()


def test_validation_leaves_the_training_streams_alone(data, tmp_path, monkeypatch):
    from neurst_b200.trainer import DataParallelTrainer
    seen = []
    orig = DataParallelTrainer.train_step

    def spy(self, inputs, seed=None):
        seen[-1].append((seed, int(inputs["src_length"].sum()), int(inputs["trg"].sum()), int(inputs["src"].sum().double() * 1e3)))
        return orig(self, inputs, seed)

    monkeypatch.setattr(DataParallelTrainer, "train_step", spy)
    losses = []
    for i, with_validator in enumerate((True, False, False)):
        seen.append([])
        kw = {} if with_validator else {"validator": False}
        res = cli.train(_plan(data, str(tmp_path / ("run%d" % i)), "float32", 12, **kw))
        assert ("validations" in res) == with_validator
        losses.append(res["loss"])
    assert seen[0] == seen[1] == seen[2] and len(seen[0]) == 12
    # fp32 training sums with atomics, so two runs of the same steps differ in the last bits; with and without the
    # validator the final losses agree as closely as two runs without it (spread bounded at 1e-5 relative)
    spread = abs(losses[1] - losses[2])
    assert spread <= 1e-5 * abs(losses[1]), losses
    assert abs(losses[0] - losses[1]) <= 1e-5 * abs(losses[1]), losses


def test_restore_from_best_avg_and_early_stop(data, tmp_path, monkeypatch):
    root, y, dev = data
    model_dir = str(tmp_path / "run")
    cli.train(_plan(data, model_dir, "float16", 8))
    best_avg = os.path.join(model_dir, "best_avg")
    named = json.load(open(os.path.join(best_avg, "checkpoint")))["model_checkpoint_path"]
    plan = _plan(data, best_avg, "float16", 8)
    got = cli.predict(dict(plan, entry="predict", dataset=plan["validator"]["dataset"], output_file=None, batch_size=EVAL_BATCH,
                           search_method="beam_search", search=plan["validator"]["search"]))
    assert got["checkpoint_step"] == int(named.split("-")[1]) and len(got["hypotheses"]) == 20
    # a new run initialised from the averaged weights
    res = cli.train(dict(_plan(data, str(tmp_path / "st"), "float16", 2, validator=False), pretrain_model=best_avg))
    assert res["global_step"] == 2 and np.isfinite(res["loss"])
    # early stop: scripted WER 50, 40, 45 with patience 1 stops at the third evaluation (step 12 of 20) and saves it
    script = iter([50.0, 40.0, 45.0, 30.0, 20.0])
    monkeypatch.setattr(M.Wer, "call", lambda self, h, g: {"WER": next(script)})
    from neurst_b200.trainer import DataParallelTrainer
    step_losses = []
    orig = DataParallelTrainer.train_step
    monkeypatch.setattr(DataParallelTrainer, "train_step", lambda self, inputs, seed=None: step_losses.append(orig(self, inputs, seed))
                        or step_losses[-1])
    res = cli.train(_plan(data, str(tmp_path / "es"), "float16", 20, eval_estop_patience=1))
    assert res["early_stopped"] and res["global_step"] == 12 and [v["step"] for v in res["validations"]] == [4, 8, 12]
    assert len(step_losses) == 12 and res["loss"] == float(step_losses[-1])       # the stopping step's loss, not step 11's
    assert cli.latest_checkpoint(str(tmp_path / "es"))[1] == 12
    torch.cuda.synchronize()
