"""Cost of one validation pass against one training step: speech_transformer_s, fp16, random-init weights.

The dev set is synthetic: 1,400 utterances (about the size of a MuST-C dev set) written as a TFRecord file in a temporary
directory, 300-1,500 frames of 80 features each, transcripts of frames // 25 token ids ending in <SEQ_END>, vocabulary 8,192.
The validator is the recipes' SeqGenerationValidator: eval_batch_size 64, label_smoothed_cross_entropy, beam_search with
beam 4, length_penalty -1, maximum_decode_length 150, wer, 10 checkpoints kept in best/ and best_avg/.  Random weights
rarely emit <SEQ_END>, so most hypotheses run to the length limit: the generation time is close to its worst case.

The training step is bench.py's cfg2 shape (B 32, T 1000, L 88) replayed from its CUDA graph.  One untimed validation
runs first (dev-set read, graph captures); the second is timed with a host clock (validate() synchronises the device
before it starts and reads every result back before it returns).  Prints the card's name and power limit read in the
same run and writes <out>/validation_bench.json.

    python tools/validation_bench.py [--out bench_out]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_DEV, V, STEPS = 1400, 8192, 20


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # noqa
        return {"error": str(e)}


def write_dev_set(root):
    import numpy as np
    from neurst_b200 import tfrecord as R
    rng = np.random.default_rng(7)
    with open(os.path.join(root, "vocab.txt"), "w") as f:
        f.write("".join("w%d\n" % i for i in range(V - 3)))
    with R.TFRecordWriter(os.path.join(root, "dev.tfrecords-00000-of-00001")) as w:
        for i in range(N_DEV):
            frames = int(rng.integers(300, 1501))
            ids = np.concatenate([rng.integers(0, V - 3, frames // 25 - 1), [V - 1]])
            w.write(R.encode_example({"audio": rng.standard_normal(frames * 80).astype(np.float32), "transcript": ids}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "bench_out"))
    args = ap.parse_args()
    import logging
    logging.basicConfig(level=logging.INFO, format="%(asctime)s %(message)s")
    import torch
    from neurst_b200 import cli
    from neurst_b200.trainer import build_speech_transformer_trainer, synthetic_batch
    from neurst_b200.validation import Validator
    if not torch.cuda.is_available():
        raise SystemExit("validation_bench.py needs a CUDA device")
    info = gpu_info()
    with tempfile.TemporaryDirectory() as tmp:
        write_dev_set(tmp)
        cfg = {"hparams_set": "speech_transformer_s", "dtype": "float16", "model_dir": os.path.join(tmp, "model"),
               "task.params": {"batch_size": 24000, "max_src_len": 3000, "max_trg_len": 150,
                               "transcript_data_pipeline.params": {"vocab_path": os.path.join(tmp, "vocab.txt"), "language": "en"}},
               "dataset.params": {"data_path": os.path.join(tmp, "dev.tfrecords")},
               "validator.class": "SeqGenerationValidator",
               "validator.params": {"eval_dataset": "AudioTFRecordDataset", "eval_dataset.params": {"data_path": os.path.join(tmp, "dev.tfrecords")},
                                    "eval_batch_size": 64, "eval_criterion": "label_smoothed_cross_entropy",
                                    "eval_search_method": "beam_search",
                                    "eval_search_method.params": {"beam_size": 4, "length_penalty": -1, "maximum_decode_length": 150},
                                    "eval_metric": "wer", "eval_top_checkpoints_to_keep": 10}}
        plan = cli.resolve(cfg)
        model = cli._build_model(plan)
        model.init_parameters(1234)
        validator = Validator(plan, model)
        validator.validate(0)                               # dev-set read, graph captures, first saves
        t0 = time.perf_counter()
        rec, _ = validator.validate(1)
        validation_s = time.perf_counter() - t0
    del model, validator
    torch.cuda.empty_cache()
    trainer, _ = build_speech_transformer_trainer("speech_transformer_s", V, precision="fp16", label_smoothing=0.1, seed=1234,
                                                  use_cuda_graph=True)
    batch = synthetic_batch(32, 1000, 88, V, seed=1234, device="cuda")
    for _ in range(3):
        trainer.train_step(batch)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(STEPS):
        trainer.train_step(batch)
    torch.cuda.synchronize()
    step_s = (time.perf_counter() - t0) / STEPS
    out = {"gpu": info, "dev_utterances": N_DEV, "validation_s": validation_s, "validation_parts_s": rec["elapsed"], "train_step_ms": step_s * 1e3,
           "validation_in_train_steps": validation_s / step_s, "NLL": float(rec["loss"]["NLL"]), "WER": float(rec["metric"]["WER"]),
           "mean_hypothesis_words": sum(len(h.split()) for h in rec["hypotheses"]) / len(rec["hypotheses"])}
    print("GPU: %s, power limit %s" % (info.get("name"), info.get("power.limit")))
    print(json.dumps(out))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "validation_bench.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
