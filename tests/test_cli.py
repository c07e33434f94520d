"""`python -m neurst_b200.cli`: the yaml-driven trainer / predict entries (SURVEY.md 8b iii).  CPU part: configuration merge,
flat and dotted command-line overrides, vocabulary meta and the resolved plan for a config shaped like the reference's
examples/speech_transformer/must-c/st_training_args.yml.  GPU part (-m gpu): TFRecords -> 6 training steps with checkpoints
-> resume -> greedy predictions, all through the entry."""
import json
import os

import numpy as np
import pytest
import torch

from neurst_b200 import cli

TRAIN_YAML = """
entry.class: trainer
entry.params:
  train_steps: 200000
  summary_steps: 200
  save_checkpoint_steps: 2000
  criterion.class: label_smoothed_cross_entropy
  criterion.params:
    label_smoothing: 0.1
  optimizer.class: adam
  optimizer.params:
    epsilon: 1.e-9
    beta_1: 0.9
    beta_2: 0.98
  lr_schedule.class: noam
  lr_schedule.params:
    initial_factor: 3.5
    end_factor: 1.5
    dmodel: 256
    warmup_steps: 25000
    start_decay_at: 50000
    decay_steps: 50000
dataset.class: AudioTFRecordDataset
dataset.params:
  data_path: %(data)s
  shuffle_dataset: True
  feature_key: audio
  transcript_key: translation
task.class: SpeechToText
task.params:
  audio_feature_dim: 80
  transcript_data_pipeline.class: TranscriptDataPipeline
  transcript_data_pipeline.params:
    language: de
    vocab_path: %(vocab)s
  batch_by_frames: True
  batch_size: 80000
  max_src_len: 3000
  max_trg_len: 150
  truncate_src: True
  experimental_frame_transcript_ratio: 12
"""


def _write_yaml(tmp_path, data="DATA", n_tokens=90):
    vocab = tmp_path / "vocab.de"
    vocab.write_text("".join("tok%d\t%d\n" % (i, 1000 - i) for i in range(n_tokens)), encoding="utf-8")
    y = tmp_path / "train.yml"
    y.write_text(TRAIN_YAML % {"data": data, "vocab": str(vocab)})
    return str(y)


def test_config_merge_overrides_and_plan(tmp_path):
    y = _write_yaml(tmp_path)
    extra = tmp_path / "extra.yml"
    extra.write_text("entry.params:\n  train_steps: 500\n  clip_norm: 1.0\nmodel_dir: /tmp/m\nhparams_set: speech_transformer_m\n")
    paths, ov = cli.parse_command_line(["--config_paths", "%s,%s" % (y, extra), "--summary_steps", "50",
                                        "--task.params.max_src_len", "2000", "--entry.class", "predict", "--dtype=bfloat16"])
    cfg = cli.load_config(paths, ov)
    assert cfg["entry.params"]["train_steps"] == 500 and cfg["entry.params"]["optimizer.params"]["beta_2"] == 0.98   # merged, not replaced
    assert cfg["entry.params"]["summary_steps"] == 50 and cfg["task.params"]["max_src_len"] == 2000
    plan = cli.resolve(cfg, world=8)
    assert plan["entry"] == "predict" and plan["precision"] == "bf16" and plan["model_dir"] == "/tmp/m"
    assert plan["task"]["batch_size_per_gpu"] == 10000 and plan["task"]["frame_transcript_ratio"] == 12       # 80000 frames / 8 replicas
    assert plan["model_params"]["encoder.hidden_size"] == 512 and plan["lr_schedule"]["dmodel"] == 256        # hparams_set < yaml
    assert plan["clip_norm"] == 1.0 and plan["label_smoothing"] == 0.1
    tm = plan["trg_meta"]
    assert (tm["vocab_size"], tm["unk_id"], tm["bos_id"], tm["eos_id"], tm["pad_id"]) == (93, 90, 91, 92, 92) and tm["tokens"][3] == "tok3"
    assert plan["dataset"] == {"data_path": "DATA", "feature_key": "audio", "transcript_key": "translation"}
    assert cli.ids_to_text([3, 4, 92, 5], 92, ["a", "b", "c", "he@@", "llo"]) == "hello"
    assert cli.ids_to_text([3, 4, 92, 5], 92, None) == "3 4"
    with pytest.raises(SystemExit):
        cli.resolve(dict(cfg, **{"task.class": "Translation"}))
    with pytest.raises(SystemExit):
        cli.parse_command_line(["positional"])


def test_latest_checkpoint(tmp_path):
    assert cli.latest_checkpoint(str(tmp_path)) == (None, 0)
    for s in (3, 12, 7):
        (tmp_path / ("ckpt-%d.npz" % s)).write_bytes(b"")
    p, s = cli.latest_checkpoint(str(tmp_path))
    assert s == 12 and p.endswith("ckpt-12.npz")


def _write_dataset(root, n_shards=3, per_shard=70, vocab=90):
    from neurst_b200 import tfrecord as R
    rng = np.random.default_rng(11)
    n = 0
    for s in range(n_shards):
        with R.TFRecordWriter(str(root / ("train.tfrecords-%05d-of-%05d" % (s, n_shards)))) as w:
            for i in range(per_shard):
                frames = int(rng.integers(100, 400))
                l = max(3, frames // 25)
                ids = np.concatenate([rng.integers(0, vocab, l - 1), [vocab + 2]])          # ... <SEQ_END>
                w.write(R.encode_example({"audio": rng.standard_normal(frames * 80).astype(np.float32), "translation": ids,
                                          "src_lang": "en", "uuid": "utt_%d_%d" % (s, i)}))
                n += 1
    return n


@pytest.mark.gpu
def test_train_resume_predict_through_the_entry(tmp_path, monkeypatch):
    from neurst_b200 import checkpoints as CK
    from neurst_b200.runtime import Runtime
    states = []              # the fp16 loss-scale state (scale, finite steps, last skipped, skips, applied updates) around each update
    adam_step = Runtime.adam_step

    def recording(rt, *a, **kw):
        before = rt.loss_scale_state[:5].tolist()
        adam_step(rt, *a, **kw)
        states.append((before, rt.loss_scale_state[:5].tolist()))
    monkeypatch.setattr(Runtime, "adam_step", recording)
    n = _write_dataset(tmp_path, vocab=93)                          # 93 tokens + 3 symbols = 96: the 16-bit path needs vocab % 8 == 0
    y = _write_yaml(tmp_path, data=str(tmp_path / "train.tfrecords"), n_tokens=93)
    model_dir = str(tmp_path / "model")
    tiny = ["--model.params.encoder.num_layers", "2", "--model.params.decoder.num_layers", "2",
            "--model.params.encoder.hidden_size", "128", "--model.params.decoder.hidden_size", "128", "--model.params.modality.dim", "128",
            "--model.params.encoder.num_attention_heads", "2", "--model.params.decoder.num_attention_heads", "2",
            "--model.params.encoder.filter_size", "256", "--model.params.decoder.filter_size", "256",
            "--model.params.modality.source.channels", "64"]
    common = ["--config_paths", y, "--model_dir", model_dir, "--task.params.batch_size", "3000", "--task.params.max_src_len", "400",
              "--task.params.max_trg_len", "24", "--task.params.min_src_bucket_boundary", "128",
              "--task.params.experimental_frame_transcript_ratio", "20", "--save_checkpoint_steps", "3", "--summary_steps", "2"] + tiny
    res = cli.main(common + ["--train_steps", "6"])
    assert res["global_step"] == 6 and res["loss"] is not None and np.isfinite(res["loss"])
    assert os.path.exists(os.path.join(model_dir, "ckpt-3.npz")) and os.path.exists(os.path.join(model_dir, "ckpt-6.npz"))
    idx = json.load(open(os.path.join(model_dir, "checkpoint")))
    assert idx["model_checkpoint_path"] == "ckpt-6.npz"
    z = np.load(os.path.join(model_dir, "ckpt-6.npz"))
    assert any(k.startswith("SpeechTransformer/TransformerEncoder/layer_0/") for k in z.files) and any("/.OPTIMIZER_SLOT/m" in k for k in z.files)
    saved = [float(z[k][0]) for k in CK.LOSS_SCALE_KEYS]         # the default dtype float16: scale, finite steps, applied updates
    assert len(states) == 6 and [states[5][1][i] for i in (0, 1, 4)] == saved
    res = cli.main(common + ["--train_steps", "8"])                 # resumes at 6 (parameters, Adam slots, schedule position)
    assert res["global_step"] == 8 and os.path.exists(os.path.join(model_dir, "ckpt-8.npz"))
    # ... and the loss-scale state: the resumed run's first update starts from the one ckpt-6 saved
    assert len(states) == 8 and [states[6][0][i] for i in (0, 1, 4)] == saved, (states[6][0], saved)
    out = str(tmp_path / "hyp.txt")
    one = tmp_path / "one"
    one.mkdir()
    os.link(str(tmp_path / "train.tfrecords-00000-of-00003"), str(one / "train.tfrecords-00000-of-00001"))
    res = cli.main(common + ["--entry.class", "predict", "--output_file", out, "--dataset.params.data_path", str(one / "train.tfrecords"),
                             "--maximum_decode_length", "12"])
    assert res["checkpoint_step"] == 8 and res["n_hypotheses"] == 70
    lines = open(out, encoding="utf-8").read().split("\n")
    assert len(lines) == 71 and all(all(t.startswith("tok") or t == "<UNK>" for t in l.split()) for l in lines[:-1])
    torch.cuda.synchronize()


def test_rank_shards_are_disjoint_and_complete(tmp_path):
    """Each rank streams its own TFRecord files (dataset_utils.load_tfrecords auto-shard under Horovod); with fewer files than
    ranks every rank reads everything."""
    n = _write_dataset(tmp_path, n_shards=4, per_shard=9)
    y = _write_yaml(tmp_path, data=str(tmp_path / "train.tfrecords"))
    plan = cli.resolve(cli.load_config([y], [("task.params.batch_size", 3000), ("task.params.max_src_len", 400),
                                             ("task.params.max_trg_len", 24)]))
    seen = []
    for rank in range(2):
        _, ex = cli._examples(plan, rank, 2, training=False)
        seen.append([int(e["audio_length"]) for e in ex])
    assert len(seen[0]) == len(seen[1]) == 18 and len(seen[0]) + len(seen[1]) == n
    _, ex = cli._examples(plan, 0, 1, training=False)
    assert sorted(seen[0] + seen[1]) == sorted(int(e["audio_length"]) for e in ex)
    _, ex = cli._examples(plan, 3, 8, training=False)              # 4 files, 8 ranks: no sharding
    assert sum(1 for _ in ex) == n
