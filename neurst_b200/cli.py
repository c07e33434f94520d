"""`neurst-run`-style entries over the C-ABI step loop (SURVEY.md 8b iii): a thin `trainer` / `predict` pair that consumes
the reference's yaml configuration for the speech-to-text path and drives libb200st.

    python -m neurst_b200.cli --config_paths train.yml[,more.yml] [--model_dir DIR] [--hparams_set speech_transformer_s]
                              [--entry.class predict] [--train_steps 1000] [--task.params.max_src_len 2000] ...
    python -m torch.distributed.run --nproc-per-node 8 -m neurst_b200.cli --config_paths train.yml      # data parallel

Host mirror of
  neurst/cli/run_exp.py + neurst/utils/flags_core.py:207-330   config files merged in order, command line on top
  neurst/exps/trainer.py:180-315 (Trainer.run)                 model + optimizer + schedule + dataset -> fit loop, checkpoints
  neurst/exps/sequence_generator.py:62-137                     restore -> search -> hypotheses file
  neurst/tasks/speech2text.py                                  task parameters (data side: neurst_b200/data.py)
  neurst/data/data_pipelines/text_data_pipeline.py:83-93       target vocabulary meta: tokens + <UNK>, <SEQ_BEG>, <SEQ_END>

Keys understood (the ones of examples/speech_transformer/*/st_training_args.yml): entry.class / entry.params {train_steps,
summary_steps, save_checkpoint_steps, update_cycle, clip_value, clip_norm, criterion.params.label_smoothing, optimizer.params,
lr_schedule.params, pretrain_model, initial_global_step, pruning_schedule / pruning_schedule.params {initial_sparsity,
target_sparsity, begin_pruning_step, end_pruning_step, pruning_frequency, polynomial_power} (or the same names as flat
flags), pruning_variable_pattern, nopruning_variable_pattern}, `entry: prune_tune_train` (`train` with the Prune-Tune recipe's
partial_tuning (a bare --partial_tuning) and mask_pkl, and <model_dir>/mask.pkl written after a pruning or partial-tuning
run; --include is accepted and ignored), `entry: mask_predict` / `mask_generation` (`predict` with the weights multiplied
by the masks of mask_pkl), dataset.class AudioTFRecordDataset / dataset.params, task.class SpeechToText /
task.params, model.class / model.params / hparams_set, model_dir, dtype, and for `predict` the keys of the prediction
recipes: `entry: predict` (the alias of entry.class) and search_method beam_search / search_method.params {beam_size,
length_penalty, top_k, maximum_decode_length, extra_decode_length, minimum_decode_length, enable_unk} or search_method
top_sampling / search_method.params {sample_num, top_k, top_p, maximum_decode_length, extra_decode_length,
minimum_decode_length} (sample_num lines per utterance, drawn with entry.params random_seed), and the top-level
batch_size (utterances per call; with a 16-bit dtype decoded from the 16-bit weights).  Several model_dirs (a yaml list or a
comma-separated string) make `predict` decode with their ensemble, weighted by search_method.params / entry.params
ensemble_weights ("average" or comma-separated numbers); each member is rebuilt from its model_configs.yml, which `train`
writes.  validator.class / validator.params (CriterionValidator, SeqGenerationValidator) validate during `train`
(neurst_b200/validation.py).  Transcripts must already be token ids (the
reference's `create_tfrecords` with a projected transcript): its tokenizers / BPE are outside this path and raw text is
refused with that message.  Checkpoints are NumPy archives keyed by the reference's variable names (checkpoints.py).
"""
import copy
import glob
import json
import logging
import os
import re
import sys
import time

import torch

LOG = logging.getLogger("neurst_b200")

SECTIONS = ("entry.params", "task.params", "dataset.params", "model.params", "search_method.params", "validator.params")
TOP_LEVEL = ("model_dir", "hparams_set", "dtype", "output_file", "entry", "search_method", "validator")
# the validators' flags (neurst/training/validator.py, criterion_validator.py, seq_generation_validator.py): a flat
# `--eval_steps 500` lands in validator.params, as the reference's registered flags do
TEXT_TASKS = ("seqtoseq", "seq2seq")                       # registered as seq_to_seq and Seq2Seq
WAITK_TASKS = ("waitktranslation",)                        # registered as WaitkTranslation and waitk_translation
TEXT_DATASETS = ("paralleltextdataset", "paralleltext")
TEXT_MODELS = ("transformer",)
WAITK_MODELS = ("waitktransformer",)
SPEECH_MODELS = ("speechtransformer", "b200speechtransformer", "b200st")
# the reference's boolean flags that stand alone on its command lines (`--partial_tuning`, examples/prune_tune/README.md):
# they take no value unless written `--flag=value`; every other flag takes the values that follow it
BARE_FLAGS = ("partial_tuning",)
# flags of the reference's launcher that have nothing to do here (`--include examples/prune_tune/src/` loads its plugins)
IGNORED_FLAGS = ("include",)
TRAIN_ENTRIES = ("trainer", "train", "prune_tune_train")
MASK_PREDICT_ENTRIES = ("mask_predict", "mask_generation")
PREDICT_ENTRIES = ("predict", "sequencegenerator", "sequence_generator") + MASK_PREDICT_ENTRIES
VALIDATOR_FLAGS = ("eval_steps", "eval_start_at", "eval_on_begin", "eval_dataset", "eval_dataset.params", "eval_batch_size",
                   "eval_task_args", "eval_criterion", "eval_criterion.params", "eval_search_method", "eval_search_method.params",
                   "eval_metric", "eval_metric.params", "eval_estop_patience", "eval_best_checkpoint_path",
                   "eval_auto_average_checkpoints", "eval_best_avg_checkpoint_path", "eval_top_checkpoints_to_keep")


# ------------------------------------------------------------------------------------------------ configuration
def deep_merge(base, new):
    """Later files win; `*.params` dictionaries are merged key by key (flags_core.py: deep_merge_dict)."""
    out = copy.deepcopy(base)
    for k, v in (new or {}).items():
        if isinstance(v, dict) and isinstance(out.get(k), dict):
            out[k] = deep_merge(out[k], v)
        else:
            out[k] = copy.deepcopy(v)
    return out


def _coerce(text):
    import yaml
    try:
        return yaml.safe_load(text)
    except Exception:
        return text


def parse_command_line(argv):
    """--config_paths a,b  plus any number of `--key value` overrides.  A dotted key addresses the nested dictionary
    (`--task.params.max_src_len 2000`, `--entry.class predict`); a plain key is matched against the parameter sections, as
    the reference's flat flags are (`--train_steps 10` -> entry.params.train_steps)."""
    paths, overrides = [], []
    i = 0
    while i < len(argv):
        a = argv[i]
        if not a.startswith("--"):
            raise SystemExit("unexpected argument %r" % a)
        key = a[2:]
        if "=" in key:
            key, val = key.split("=", 1)
        elif key in BARE_FLAGS:
            overrides.append((key, True))
            i += 1
            continue
        else:
            i += 1
            if i >= len(argv):
                raise SystemExit("flag --%s needs a value" % key)
            val = argv[i]
            # several values before the next flag make a list (`--pretrain_model asr/best_avg mt/best_avg`)
            more = []
            while i + 1 < len(argv) and not argv[i + 1].startswith("--"):
                i += 1
                more.append(argv[i])
            if more:
                if key == "config_paths":
                    raise SystemExit("unexpected argument %r" % more[0])
                overrides.append((key, [_coerce(v) for v in [val] + more]))
                i += 1
                continue
        if key == "config_paths":
            paths.extend(p for p in val.split(",") if p)
        else:
            overrides.append((key, _coerce(val)))
        i += 1
    return paths, [(k, v) for k, v in overrides if k not in IGNORED_FLAGS]


def _set_dotted(cfg, key, val):
    # "a.params.b.c" -> cfg["a.params"]["b.c"]; "entry.class" -> cfg["entry.class"]
    m = re.match(r"^([a-z_]+\.params)\.(.+)$", key)
    if m:
        cfg.setdefault(m.group(1), {})[m.group(2)] = val
    else:
        cfg[key] = val


def load_config(paths, overrides=()):
    import yaml
    cfg = {}
    for p in paths:
        with open(p) as f:
            cfg = deep_merge(cfg, yaml.safe_load(f) or {})
    for key, val in overrides:
        if key in ("entry", "search_method", "validator") and (key + ".class") in cfg:
            # `--entry` is the command-line alias of `entry.class` (flags_core.py: ModuleFlag): it overrides the file's class
            cfg[key + ".class"] = val
            continue
        if "." in key or key in TOP_LEVEL:
            _set_dotted(cfg, key, val)
            continue
        hits = [s for s in SECTIONS if isinstance(cfg.get(s), dict) and key in cfg[s]]
        if len(hits) > 1:
            raise SystemExit("flag --%s is ambiguous (%s): use the dotted form" % (key, ", ".join(hits)))
        if not hits and key in VALIDATOR_FLAGS:
            hits = ["validator.params"]
        cfg.setdefault(hits[0] if hits else "entry.params", {})[key] = val
    return cfg


def _vocab_meta(n, path):
    """Vocabulary meta (text_data_pipeline.py:83-93, data/text/vocab.py): ids 0..n-1 are the file's tokens, then <UNK>,
    <SEQ_BEG>, <SEQ_END>; padding = EOS."""
    tokens = None
    if path and os.path.exists(path):
        with open(path, encoding="utf-8") as f:
            tokens = [l.rstrip("\n").split("\t")[0].split(" ")[0] for l in f if l.strip()]
        n = len(tokens) + 3
    if n is None:
        return None
    n = int(n)
    return {"vocab_size": n, "unk_id": n - 3, "bos_id": n - 2, "eos_id": n - 1, "pad_id": n - 1, "padding_mode": "eos_as_padding",
            "tokens": tokens}


def target_meta(task_params):
    """Vocabulary meta of the target side: task.params.vocab_size, or the *_data_pipeline.params.vocab_path file."""
    tp = task_params
    path = None
    for k in ("transcript_data_pipeline.params", "trg_data_pipeline.params", "translation_data_pipeline.params"):
        if isinstance(tp.get(k), dict) and tp[k].get("vocab_path"):
            path = tp[k]["vocab_path"]
    meta = _vocab_meta(tp.get("vocab_size"), path)
    if meta is None:
        raise SystemExit("the target vocabulary is unknown: give task.params.vocab_size or a readable *_data_pipeline.params.vocab_path")
    return meta


def text_vocab_metas(task_params):
    """(source, target) vocabulary metas of the seq2seq task, read from src_data_pipeline.params.vocab_path and
    trg_data_pipeline.params.vocab_path: the text path maps tokens to ids itself, so both files must be readable."""
    metas = []
    for side in ("src", "trg"):
        params = task_params.get(side + "_data_pipeline.params")
        path = params.get("vocab_path") if isinstance(params, dict) else None
        if not path or not os.path.isfile(path):
            raise SystemExit("task.params.%s_data_pipeline.params.vocab_path must name a readable vocabulary file, got %r"
                             % (side, path))
        metas.append(_vocab_meta(None, path))
    return tuple(metas)


def _module_name(cfg, name):
    """`name.class` or its alias `name` (flags_core.py:293-299: the `.class` key wins when both are given)."""
    v = cfg.get(name + ".class", cfg.get(name))
    if isinstance(v, dict):
        v = v.get("class")
    return v


def resolve_search(cfg, ep, tp):
    """Search settings of `predict`.  Without search_method: greedy with the lengths of entry.params (as before).  With
    search_method BeamSearch: its parameters (search_method.params, then entry.params) with BeamSearch's defaults
    (beam_search.py:465-490).  With TopSampling (registered as TopSampling, topsampling and top_sampling): its parameters
    from the same places with Sampling's defaults (sampling.py:290-313) and its two refusals."""
    length_default = int(ep.get("maximum_decode_length", tp.get("max_trg_len") or 256))
    method = _module_name(cfg, "search_method")
    if method is None:
        return None, {"maximum_decode_length": length_default, "extra_decode_length": int(ep.get("extra_decode_length", 50)),
                      "minimum_decode_length": int(ep.get("minimum_decode_length", 0))}
    name = str(method).lower().replace("_", "")
    if name not in ("beamsearch", "topsampling"):
        raise SystemExit("search_method %r is outside this path (beam_search, top_sampling)" % method)
    sp = dict(cfg.get("search_method.params") or {})

    def get(key, default):
        v = sp.get(key, ep.get(key))
        return default if v is None else v

    if name == "topsampling":
        search = {"maximum_decode_length": int(get("maximum_decode_length", length_default)),
                  "extra_decode_length": int(get("extra_decode_length", 50)),
                  "minimum_decode_length": int(get("minimum_decode_length", 0) or 0),
                  "sample_num": int(get("sample_num", 1)), "top_k": int(get("top_k", 0)), "top_p": float(get("top_p", 1.0))}
        if search["top_k"] > 0 and search["top_p"] < 1:               # Sampling.__init__
            raise SystemExit("top_sampling: Not implemented search logic when top_k > 0 and top_p < 1.")
        if search["minimum_decode_length"] >= search["maximum_decode_length"]:       # Sampling.call
            raise SystemExit("top_sampling: `minimum_decode_length` must be less than maximum decode length.")
        if not 1 <= search["sample_num"] <= 8:
            raise SystemExit("top_sampling: sample_num must be in 1..8 (the samples of an utterance share a decoding step), "
                             "got %d" % search["sample_num"])
        if search["top_k"] < 0 or search["top_p"] != search["top_p"] or abs(search["top_p"]) == float("inf"):
            raise SystemExit("top_sampling: top_k must be >= 0 and top_p finite, got top_k %d, top_p %r"
                             % (search["top_k"], search["top_p"]))
        return "top_sampling", search

    lp = sp.get("length_penalty", ep.get("length_penalty", 0.6))
    return "beam_search", {"maximum_decode_length": int(get("maximum_decode_length", length_default)),
                           "extra_decode_length": int(get("extra_decode_length", 50)),
                           "minimum_decode_length": int(get("minimum_decode_length", 0)),
                           "beam_size": int(get("beam_size", 4)), "length_penalty": -1.0 if lp is None else float(lp),
                           "top_k": int(get("top_k", 1)), "enable_unk": bool(get("enable_unk", False))}


def _as_dict(v, what):
    if v is None:
        return {}
    if not isinstance(v, dict):
        raise SystemExit("%s must be a mapping, got %r" % (what, v))
    return dict(v)


def _text_dataset(dsp, what):
    """dataset.params of a ParallelTextDataset: BPE'd, line-aligned source and target files."""
    if not dsp.get("src_file"):
        raise SystemExit("%s ParallelTextDataset needs src_file" % what)
    if not dsp.get("data_is_processed"):
        raise SystemExit("%s ParallelTextDataset with raw text is outside this path: the tokenizer and BPE (moses, "
                         "subword-nmt, sentencepiece) are not applied here; give BPE'd files with data_is_processed: True" % what)
    return {"src_file": dsp["src_file"], "trg_file": dsp.get("trg_file"), "data_is_processed": True}


def resolve_validator(cfg, tp, text=False):
    """validator.class (or its alias `validator`) with validator.params, the flags and defaults of Validator,
    CriterionValidator and SeqGenerationValidator; None without a validator.  `text`: the seq2seq task, whose eval
    dataset is a ParallelTextDataset."""
    cls = _module_name(cfg, "validator")
    if cls is None:
        return None
    name = {"criterionvalidator": "CriterionValidator", "seqgenerationvalidator": "SeqGenerationValidator"}.get(
        str(cls).lower().replace("_", ""))
    if name is None:
        raise SystemExit("validator.class %r is outside this path (CriterionValidator, SeqGenerationValidator)" % cls)
    vp = _as_dict(cfg.get("validator.params"), "validator.params")
    for k in VALIDATOR_FLAGS:               # dotted command-line keys such as --eval_dataset.params.data_path
        if k in cfg:
            vp = deep_merge(vp, {k: cfg[k]})

    def module(key):
        return vp.get(key + ".class", vp.get(key)), _as_dict(vp.get(key + ".params"), "validator.params." + key + ".params")

    ds_cls, dsp = module("eval_dataset")
    if text:
        if str(ds_cls).lower().replace("_", "") not in TEXT_DATASETS:
            raise SystemExit("eval_dataset %r is outside this path for the seq2seq task (ParallelTextDataset only)" % ds_cls)
        if not dsp.get("trg_file"):
            raise SystemExit("validator %s needs eval_dataset.params.trg_file" % name)
    elif ds_cls is None or not dsp.get("data_path"):
        raise SystemExit("validator %s needs eval_dataset with eval_dataset.params.data_path" % name)
    elif str(ds_cls).lower().replace("_", "") not in ("audiotfrecorddataset", "audiotfrecord"):
        raise SystemExit("eval_dataset %r is outside this path (AudioTFRecordDataset only)" % ds_cls)
    task_args = _as_dict(vp.get("eval_task_args"), "eval_task_args")
    unknown = sorted(set(task_args) - {"batch_size", "truncate_src", "max_src_len"})
    if unknown:
        raise SystemExit("eval_task_args %s are outside this path (batch_size, truncate_src, max_src_len)" % ", ".join(unknown))
    crit_cls, critp = module("eval_criterion")
    if crit_cls is not None and str(crit_cls).lower().replace("_", "") != "labelsmoothedcrossentropy":
        raise SystemExit("eval_criterion %r is outside this path (label_smoothed_cross_entropy only)" % crit_cls)
    plan = {"class": name, "eval_steps": int(vp.get("eval_steps", 1000)), "eval_start_at": int(vp.get("eval_start_at", 0)),
            "eval_on_begin": bool(vp.get("eval_on_begin", False)),
            "dataset": _text_dataset(dsp, "eval_dataset") if text else
            {"data_path": dsp["data_path"], "feature_key": dsp.get("feature_key", "audio"),
             "transcript_key": dsp.get("transcript_key", "transcript")},
            "batch_size": int(vp.get("eval_batch_size", 32)),
            "task_args": {k: v for k, v in task_args.items() if k != "batch_size"},
            # the reference builds the eval criterion from its own params: label_smoothing defaults to 0
            "criterion": crit_cls is not None, "label_smoothing": float(critp.get("label_smoothing", 0.0)),
            "search_method": None, "search": None, "metric": None}
    if plan["eval_steps"] <= 0 or plan["batch_size"] <= 0:
        raise SystemExit("eval_steps and eval_batch_size must be positive")
    if name == "SeqGenerationValidator":
        method, sp = module("eval_search_method")
        metric, metric_params = module("eval_metric")
        if metric_params:
            # the restated metrics take no parameters; their language is the target data pipeline's
            raise SystemExit("eval_metric.params %s are outside this path (the metrics take no parameters; the language "
                             "is task.params' *_data_pipeline.params.language)" % ", ".join(sorted(metric_params)))
        if method is not None:
            plan["search_method"], plan["search"] = resolve_search({"search_method": method, "search_method.params": sp}, {}, tp)
            if plan["search_method"] != "beam_search":
                raise SystemExit("eval_search_method %r is outside this path for validation (beam_search only)" % method)
        language = "en"                     # the metric's language: the target data pipeline's (get_eval_metric)
        for k in ("transcript_data_pipeline.params", "trg_data_pipeline.params", "translation_data_pipeline.params"):
            if isinstance(tp.get(k), dict) and tp[k].get("language"):
                language = tp[k]["language"]
        if metric is not None:
            from neurst_b200.metrics import build_metric
            try:
                build_metric(metric, language)
            except ValueError as e:
                raise SystemExit(str(e))
            plan["metric"] = str(metric)
        plan.update(language=language, estop_patience=int(vp.get("eval_estop_patience", 0) or 0),
                    best_checkpoint_path=vp.get("eval_best_checkpoint_path"),
                    auto_average_checkpoints=bool(vp.get("eval_auto_average_checkpoints", True)),
                    best_avg_checkpoint_path=vp.get("eval_best_avg_checkpoint_path"),
                    top_checkpoints_to_keep=int(vp.get("eval_top_checkpoints_to_keep", 10)))
    return plan


def resolve(cfg, world=1):
    """Everything the entries need, as plain dictionaries (also what the CPU test checks)."""
    from neurst_b200.models import speech_transformer_hparams, transformer_hparams, waitk_transformer_hparams
    if str(_module_name(cfg, "entry") or "").lower().replace("_", "") == "cascadest":
        return resolve_cascade(cfg, world)
    if str(_module_name(cfg, "entry") or "").lower().replace("_", "") == "simuleval":
        return resolve_simuleval(cfg, world)
    ep, tp = dict(cfg.get("entry.params") or {}), dict(cfg.get("task.params") or {})
    task_cls = str(cfg.get("task.class", "SpeechToText")).lower().replace("_", "")
    waitk = task_cls in WAITK_TASKS
    text = task_cls in TEXT_TASKS or waitk
    if task_cls not in ("speechtotext", "speech2text") and not text:
        raise SystemExit("task.class %r is outside this path (SpeechToText, Seq2Seq, WaitkTranslation)" % cfg.get("task.class"))
    if not text and (tp.get("wait_k") is not None or cfg.get("wait_k", ep.get("wait_k")) is not None):
        raise SystemExit("wait_k is outside this path for the SpeechToText task: wait-k decoding is the text WaitkTranslation "
                         "task's (the reference has no simultaneous speech model)")
    ds_cls = str(cfg.get("dataset.class", "ParallelTextDataset" if text else "AudioTFRecordDataset")).lower().replace("_", "")
    if text and ds_cls not in TEXT_DATASETS:
        raise SystemExit("dataset.class %r is outside this path for the seq2seq task (ParallelTextDataset only)" % cfg.get("dataset.class"))
    if not text and ds_cls not in ("audiotfrecorddataset", "audiotfrecord"):
        raise SystemExit("dataset.class %r is outside this path (AudioTFRecordDataset only)" % cfg.get("dataset.class"))
    # the hparams_set's name picks the speech or the text table
    hp_name = cfg.get("hparams_set") or ("waitk_transformer_s" if waitk else "transformer_s" if text else "speech_transformer_s")
    try:
        hp = speech_transformer_hparams(hp_name) or transformer_hparams(hp_name) or waitk_transformer_hparams(hp_name)
    except ValueError as e:
        raise SystemExit(str(e))
    if hp is None:
        raise SystemExit("unknown hparams_set %r" % cfg.get("hparams_set"))
    if hp["model.class"] not in (("Transformer", "WaitkTransformer") if text else ("SpeechTransformer",)):
        raise SystemExit("hparams_set %r is a %s preset, outside this path for the %s task" % (
            hp_name, hp["model.class"], "seq2seq" if text else "SpeechToText"))
    model_cls = str(cfg.get("model.class", hp["model.class"])).lower().replace("_", "")
    if waitk and model_cls not in WAITK_MODELS:
        raise SystemExit("model.class %r is outside this path for the WaitkTranslation task (WaitkTransformer only)"
                         % cfg.get("model.class", hp["model.class"]))
    if text and not waitk and model_cls in WAITK_MODELS:
        raise SystemExit("model.class WaitkTransformer needs task.class WaitkTranslation (the task supplies wait_k)")
    if text and not waitk and model_cls not in TEXT_MODELS:
        raise SystemExit("model.class %r is outside this path for the seq2seq task (Transformer only)"
                         % cfg.get("model.class", hp["model.class"]))
    if not text and model_cls not in SPEECH_MODELS:
        raise SystemExit("model.class %r is outside this path (SpeechTransformer only)" % cfg.get("model.class", hp["model.class"]))
    model_params = dict(hp["model.params"])
    model_params.update(cfg.get("model.params") or {})
    opt = dict(hp["optimizer.params"]); opt.update(ep.get("optimizer.params") or {})
    lr = dict(hp["lr_schedule.params"]); lr.update(ep.get("lr_schedule.params") or {})
    if str(ep.get("lr_schedule.class", "noam")).lower() != "noam" or str(ep.get("optimizer.class", "adam")).lower() != "adam":
        raise SystemExit("this path implements the presets' Adam + noam schedule")
    crit = ep.get("criterion.params") or {}
    entry = str(_module_name(cfg, "entry") or "trainer").lower()
    if text:
        return _resolve_text(cfg, ep, tp, world, entry, model_params, opt, lr, crit, waitk)
    # batch_size counts frames when batch_by_frames (speech2text.py:296-310): per-GPU budget = batch_size // replicas
    per_gpu = tp.get("batch_size_per_gpu")
    if per_gpu is None:
        if tp.get("batch_size") is None:
            raise SystemExit("task.params needs batch_size or batch_size_per_gpu (frames)")
        per_gpu = int(tp["batch_size"]) // max(1, world)
    task = dict(max_src_len=tp.get("max_src_len"), max_trg_len=tp.get("max_trg_len"), batch_size_per_gpu=int(per_gpu),
                audio_feature_dim=int(tp.get("audio_feature_dim", 80)), audio_feature_channels=int(tp.get("audio_feature_channels", 1)),
                truncate_src=bool(tp.get("truncate_src", False)), truncate_trg=bool(tp.get("truncate_trg", False)),
                min_src_bucket_boundary=tp.get("min_src_bucket_boundary", 128),
                frame_transcript_ratio=tp.get("experimental_frame_transcript_ratio"),
                disable_batch_efficiency=bool(tp.get("disable_batch_efficiency", False)), specaug=tp.get("specaug"))
    dsp = dict(cfg.get("dataset.params") or {})
    dataset = {"data_path": dsp.get("data_path"), "feature_key": dsp.get("feature_key", "audio"),
               "transcript_key": dsp.get("transcript_key", "transcript")}
    search_method, search = resolve_search(cfg, ep, tp)
    model_dirs = flatten_string_list(cfg.get("model_dir") or ep.get("model_dir") or "./b200st_model")
    if not model_dirs:
        raise SystemExit("model_dir names no directory")
    if len(model_dirs) > 1 and entry in TRAIN_ENTRIES:
        raise SystemExit("training writes one model_dir, got %d: %s" % (len(model_dirs), ", ".join(model_dirs)))
    plan = {
        "entry": entry, "model_class": "SpeechTransformer",
        # several directories: `predict` decodes with the ensemble of their models (SequenceGenerator._build_and_restore_model)
        "model_dir": model_dirs[0] if len(model_dirs) == 1 else model_dirs,
        "precision": {"float16": "fp16", "fp16": "fp16", "bfloat16": "bf16", "bf16": "bf16", "float32": "fp32", "fp32": "fp32"}[
            str(cfg.get("dtype", "float16")).lower()],
        "model_params": model_params, "optimizer": opt, "lr_schedule": lr,
        "label_smoothing": float(crit.get("label_smoothing", 0.1)),
        "train_steps": int(ep.get("train_steps", 10000000)), "summary_steps": int(ep.get("summary_steps", 200)),
        "save_checkpoint_steps": int(ep.get("save_checkpoint_steps", 1000)), "update_cycle": int(ep.get("update_cycle", 1)),
        "clip_value": ep.get("clip_value"), "clip_norm": ep.get("clip_norm"), "pretrain_model": ep.get("pretrain_model"),
        "seed": int(ep.get("random_seed", 1234) or 1234), "max_to_keep": int(ep.get("checkpoints_max_to_keep", 8)),
        "task": task, "dataset": dataset, "trg_meta": target_meta(tp),
        "search": search,
        "output_file": cfg.get("output_file") or ep.get("output_file"),
    }
    return _finish_plan(plan, cfg, ep, tp, search_method, model_dirs)


def _model_dir_configs(model_dir, what):
    """model_configs.yml of a trained model directory: model class and parameters, and the task with its vocabularies."""
    import yaml
    path = os.path.join(model_dir, MODEL_CONFIGS)
    if not os.path.isfile(path):
        raise SystemExit("%s: %s has no %s" % (what, model_dir, MODEL_CONFIGS))
    with open(path) as f:
        configs = yaml.safe_load(f) or {}
    if not isinstance(configs.get("task.params"), dict):
        raise SystemExit("%s: %s records no task.params (the vocabularies); train it with this version or add them" % (what, path))
    return configs


def resolve_cascade(cfg, world=1):
    """The `cascade_st` entry (neurst/cli/cascade_st.py): ASR search, then MT search on the ASR top-1 hypotheses.  Each
    model is rebuilt from its directory's model_configs.yml (model and task, as ModelConfigs.load); the audio dataset is
    AudioTripleTFRecordDataset (feature_key, transcript_key, translation_key)."""
    if world > 1:
        raise SystemExit("cascade_st runs on one device (WORLD_SIZE 1)")
    ep = dict(cfg.get("entry.params") or {})

    def get(key, default=None):
        v = cfg.get(key, ep.get(key))
        return default if v is None else v

    dirs = {side: get(side + "_model_dir") for side in ("asr", "mt")}
    for side, d in dirs.items():
        if not d:
            raise SystemExit("cascade_st needs %s_model_dir" % side)
    ds_cls = str(cfg.get("dataset.class", "AudioTripleTFRecordDataset")).lower().replace("_", "")
    if ds_cls not in ("audiotripletfrecorddataset", "audiotripletfrecord"):
        raise SystemExit("dataset.class %r is outside this path for cascade_st (AudioTripleTFRecordDataset only)" % cfg.get("dataset.class"))
    dsp = dict(cfg.get("dataset.params") or {})
    if not dsp.get("data_path"):
        raise SystemExit("cascade_st needs dataset.params.data_path")
    if str(_model_dir_configs(dirs["mt"], "mt_model_dir").get("model.class")) == "WaitkTransformer":
        raise SystemExit("mt_model_dir %s holds a wait-k model (WaitkTransformer): wait-k decoding in cascade_st is outside "
                         "this path" % dirs["mt"])
    batch_size = int(get("batch_size", 32))
    plans = {}
    for side, want in (("asr", "SpeechTransformer"), ("mt", "Transformer")):
        configs = _model_dir_configs(dirs[side], side + "_model_dir")
        if str(configs.get("model.class")) != want:
            raise SystemExit("%s_model_dir %s holds a %s, not a %s" % (side, dirs[side], configs.get("model.class"), want))
        method = cfg.get(side + "_search_method.class", cfg.get(side + "_search_method", "beam_search"))
        sub = {"entry.class": "predict", "model_dir": dirs[side], "dtype": cfg.get("dtype", "float16"), "batch_size": batch_size,
               "task.class": configs.get("task.class"), "task.params": configs["task.params"],
               "model.class": want, "model.params": configs.get("model.params") or {},
               "hparams_set": "speech_transformer_s" if side == "asr" else "transformer_s",
               "search_method": method, "search_method.params": cfg.get(side + "_search_method.params") or {}}
        if side == "asr":
            sub["dataset.params"] = {"data_path": dsp["data_path"], "feature_key": dsp.get("feature_key", "audio"),
                                     "transcript_key": dsp.get("transcript_key", "transcript")}
        else:
            sub["dataset.class"], sub["dataset.params"] = "ParallelTextDataset", {"src_file": "-", "data_is_processed": True}
        plans[side] = resolve(sub)
        if plans[side].get("search_method") not in ("beam_search", None):
            raise SystemExit("%s_search_method %r is outside this path for cascade_st (beam_search)" % (side, method))
    if plans["asr"]["search"].get("top_k", 1) != 1:
        raise SystemExit("asr_search_method.params.top_k must be 1: the MT stage reads the ASR top-1 hypothesis")
    metrics = {side: str(get(side + "_metric.class", get(side + "_metric", default))) for side, default in (("asr", "wer"), ("mt", "bleu"))}
    from neurst_b200.metrics import build_metric
    for side, m in metrics.items():
        try:
            build_metric(m, "en")
        except ValueError as e:
            raise SystemExit("%s_metric: %s" % (side, e))
    return {"entry": "cascade_st", "asr": plans["asr"], "mt": plans["mt"], "batch_size": batch_size,
            "translation_key": dsp.get("translation_key", "translation"), "metrics": metrics,
            "asr_output_file": get("asr_output_file"), "mt_output_file": get("mt_output_file")}


def resolve_simuleval(cfg, world=1):
    """The `simuleval` entry: SimulEval's text-to-text evaluation of SimulTransTextAgent, replayed offline on the device
    (neurst/utils/simuleval_agents/simul_trans_text_agent.py; examples/iwslt21/SIMUL_TRANS.md).  model_dir: one or more
    WaitkTransformer directories (an ensemble mixed as the agent mixes it); wait_k (source words) from the command line
    overrides model_configs.yml, as build_task_and_model does; source: pre-tokenised (BPE) source lines; target: reference
    lines; output: the directory of instances.log and scores."""
    if world > 1:
        raise SystemExit("simuleval runs on one device (WORLD_SIZE 1)")
    ep = dict(cfg.get("entry.params") or {})

    def get(key, default=None):
        v = cfg.get(key, ep.get(key))
        return default if v is None else v

    model_dirs = flatten_string_list(get("model_dir"))
    if not model_dirs:
        raise SystemExit("simuleval needs --model_dir (one or more WaitkTransformer directories)")
    if len(model_dirs) > 8:
        raise SystemExit("simuleval mixes at most 8 models, got %d" % len(model_dirs))
    k = get("wait_k")
    if k is None or isinstance(k, bool) or not str(k).strip().isdigit() or int(k) < 1:
        raise SystemExit("simuleval needs --wait_k, a positive number of source words, got %r" % (k,))
    for key in ("source", "output"):
        if not get(key):
            raise SystemExit("simuleval needs --%s" % key)
    members, trg_tokens = [], None
    for d in model_dirs:
        configs = _model_dir_configs(d, "model_dir")
        if str(configs.get("model.class")) != "WaitkTransformer":
            raise SystemExit("model_dir %s holds a %s, not a wait-k model (WaitkTransformer): the agent streams a monotonic "
                             "encoder" % (d, configs.get("model.class")))
        tp = dict(configs["task.params"], wait_k=int(k))
        lang = (tp.get("trg_data_pipeline.params") or {}).get("language")
        if str(lang).lower() == "ja":
            raise SystemExit("simuleval: the agent's Japanese target branch (one character per segment) is outside this path")
        sub = {"entry.class": "predict", "model_dir": d, "dtype": get("dtype", "float32"), "task.class": "WaitkTranslation",
               "task.params": tp, "model.class": "WaitkTransformer", "model.params": configs.get("model.params") or {},
               "hparams_set": "waitk_transformer_s", "wait_k": int(k),
               "dataset.params": {"src_file": get("source"), "data_is_processed": True}}
        plan = resolve(sub)
        if trg_tokens is None:
            trg_tokens = plan["trg_meta"]["tokens"]
        elif plan["trg_meta"]["tokens"] != trg_tokens:
            raise SystemExit("model_dir %s has a target vocabulary that differs from %s's: the agent mixes the members' "
                             "distributions over one vocabulary" % (d, model_dirs[0]))
        members.append(plan)
    force = get("force_segment", False)
    if isinstance(force, str):
        force = force.strip().lower() in ("1", "true", "yes", "on")
    return {"entry": "simuleval", "members": members, "wait_k": int(k), "force_segment": bool(force),
            "max_len": int(get("max_len", 200)), "source": get("source"), "target": get("target"), "output": get("output")}


def _pretrain_patterns(ep):
    """pretrain_variable_pattern beside pretrain_model (exps/trainer.py:52-72): one regular expression (or None) per
    archive; None without patterns."""
    patterns = ep.get("pretrain_variable_pattern")
    if patterns is None:
        return None
    models = flatten_string_list(ep.get("pretrain_model"))
    patterns = [patterns] if isinstance(patterns, str) else list(patterns)
    if not models or len(models) != len(patterns):
        raise SystemExit("`pretrain_variable_pattern` must match with `pretrain_model`: %d archive(s), %d pattern(s)"
                         % (len(models or []), len(patterns)))
    for p in patterns:
        if p is not None:
            try:
                re.compile(p)
            except re.error as e:
                raise SystemExit("pretrain_variable_pattern %r: %s" % (p, e))
    return [None if p is None else str(p) for p in patterns]


def _resolve_wait_k(cfg, ep, tp, entry, model_dirs):
    """The lag of a WaitkTranslation run, parsed as WaitkTranslation does (an int, a list or a YAML string of either).
    `predict` takes it from the model directory's model_configs.yml unless a command-line --wait_k or task.params.wait_k
    overrides it (the reference's eval_task_args use); training takes task.params.wait_k."""
    from neurst_b200.models import parse_wait_k
    k = cfg.get("wait_k", ep.get("wait_k"))
    if k is None:
        k = tp.get("wait_k")
    if k is None and entry not in TRAIN_ENTRIES and len(model_dirs) == 1:
        path = os.path.join(model_dirs[0], MODEL_CONFIGS)
        if os.path.isfile(path):
            k = (_model_dir_configs(model_dirs[0], "model_dir").get("task.params") or {}).get("wait_k")
    if k is None:
        raise SystemExit("WaitkTranslation needs wait_k (task.params.wait_k, or --wait_k): the decode lagging")
    try:
        return parse_wait_k(k)
    except ValueError as e:
        raise SystemExit(str(e))


def _resolve_text(cfg, ep, tp, world, entry, model_params, opt, lr, crit, waitk=False):
    """The plan of the seq2seq task over a text Transformer (Seq2Seq, ParallelTextDataset), or of the WaitkTranslation task
    over a WaitkTransformer (plan["wait_k"] set)."""
    src_meta, trg_meta = text_vocab_metas(tp)
    if model_params.get("modality.share_source_target_embedding") and src_meta["tokens"] != trg_meta["tokens"]:
        raise SystemExit("modality.share_source_target_embedding needs identical source and target vocabularies (%d vs %d "
                         "entries)" % (src_meta["vocab_size"], trg_meta["vocab_size"]))
    if entry in TRAIN_ENTRIES and tp.get("batch_size") is None and tp.get("batch_size_per_gpu") is None:
        raise SystemExit("task.params needs batch_size or batch_size_per_gpu (tokens with batch_by_tokens, else pairs)")
    task = dict(max_src_len=tp.get("max_src_len"), max_trg_len=tp.get("max_trg_len"),
                truncate_src=bool(tp.get("truncate_src") or False), truncate_trg=bool(tp.get("truncate_trg") or False),
                batch_size=tp.get("batch_size"), batch_size_per_gpu=tp.get("batch_size_per_gpu"),
                batch_by_tokens=bool(tp.get("batch_by_tokens") or False))
    search_method, search = resolve_search(cfg, ep, tp)
    model_dirs = flatten_string_list(cfg.get("model_dir") or ep.get("model_dir") or "./b200st_model")
    if not model_dirs:
        raise SystemExit("model_dir names no directory")
    if len(model_dirs) > 1 and entry in TRAIN_ENTRIES:
        raise SystemExit("training writes one model_dir, got %d: %s" % (len(model_dirs), ", ".join(model_dirs)))
    plan = {
        "entry": entry, "model_class": "Transformer",
        "model_dir": model_dirs[0] if len(model_dirs) == 1 else model_dirs,
        "precision": {"float16": "fp16", "fp16": "fp16", "bfloat16": "bf16", "bf16": "bf16", "float32": "fp32", "fp32": "fp32"}[
            str(cfg.get("dtype", "float16")).lower()],
        "model_params": model_params, "optimizer": opt, "lr_schedule": lr,
        "label_smoothing": float(crit.get("label_smoothing", 0.1)),
        "train_steps": int(ep.get("train_steps", 10000000)), "summary_steps": int(ep.get("summary_steps", 200)),
        "save_checkpoint_steps": int(ep.get("save_checkpoint_steps", 1000)), "update_cycle": int(ep.get("update_cycle", 1)),
        "clip_value": ep.get("clip_value"), "clip_norm": ep.get("clip_norm"), "pretrain_model": ep.get("pretrain_model"),
        "seed": int(ep.get("random_seed", 1234) or 1234), "max_to_keep": int(ep.get("checkpoints_max_to_keep", 8)),
        "task": task, "dataset": _text_dataset(dict(cfg.get("dataset.params") or {}), "dataset"),
        "src_meta": src_meta, "trg_meta": trg_meta,
        "search": search,
        "output_file": cfg.get("output_file") or ep.get("output_file"),
    }
    if waitk:
        if len(model_dirs) > 1:
            raise SystemExit("an ensemble of %d model_dirs with a wait-k model is outside this path (one WaitkTransformer per "
                             "predict)" % len(model_dirs))
        plan["wait_k"] = _resolve_wait_k(cfg, ep, tp, entry, model_dirs)
        tp = dict(tp, wait_k=plan["wait_k"])
    plan = _finish_plan(plan, cfg, ep, tp, search_method, model_dirs, text=True)
    if waitk:
        plan["task_config"]["task.class"] = "WaitkTranslation"
    return plan


def _entry_key(cfg, ep, key):
    """A trainer flag from entry.params, else from the top level of the configuration."""
    v = ep.get(key)
    return cfg.get(key) if v is None else v


def resolve_pruning(cfg, ep):
    """The trainer's weight pruning (exps/trainer.py:91-93,102-103,136-140): pruning_schedule (class, PolynomialDecay by
    default) with pruning_schedule.params or the flat flags --initial_sparsity --target_sparsity --begin_pruning_step
    --end_pruning_step --pruning_frequency --polynomial_power (a flat flag wins over the same key of the params), and
    pruning_variable_pattern / nopruning_variable_pattern.  None when target_sparsity is 0 (PruningSchedule.new): the
    trainer then runs the plain optimizer step."""
    from neurst_b200 import pruning as PR
    name = _entry_key(cfg, ep, "pruning_schedule.class") or _entry_key(cfg, ep, "pruning_schedule")
    params = _entry_key(cfg, ep, "pruning_schedule.params")
    if isinstance(name, dict):                 # pruning_schedule: {class: ..., params: {...}}
        params = dict(name.get("params") or {}, **(params or {}))
        name = name.get("class")
    params = _as_dict(params, "pruning_schedule.params")
    for k in PR.SCHEDULE_FLAGS:
        v = _entry_key(cfg, ep, k)
        if v is not None:
            params[k] = v
    try:
        cls = PR.schedule_class(name or "PolynomialDecay")
        if cls is PR.ConstantSparsity:
            params = {k: v for k, v in params.items() if k not in ("initial_sparsity", "polynomial_power")}
        schedule = PR.build_schedule(cls.__name__, params)
    except (ValueError, TypeError) as e:
        raise SystemExit("pruning_schedule: %s" % e)
    if schedule is None:
        return None
    patterns = {k: _entry_key(cfg, ep, k) for k in ("pruning_variable_pattern", "nopruning_variable_pattern")}
    for k, p in patterns.items():
        if p is not None:
            try:
                re.compile(p)
            except re.error as e:
                raise SystemExit("%s %r: %s" % (k, p, e))
    return dict(schedule=schedule, **patterns)


def resolve_prune_tune(cfg, ep, entry, pruning, model_dirs):
    """The Prune-Tune entries' flags (examples/prune_tune/src/partial_trainer.py:50-58, mask_sequence_generator.py:40-45):
    prune_tune_train's partial_tuning and mask_pkl, mask_predict's / mask_generation's mask_pkl; None for the other entries."""
    mask_pkl = _entry_key(cfg, ep, "mask_pkl") or None
    if entry not in ("prune_tune_train",) + MASK_PREDICT_ENTRIES:
        return None
    if mask_pkl is not None and not os.path.isfile(str(mask_pkl)):
        raise SystemExit("mask_pkl %s: no such file" % mask_pkl)
    if entry in MASK_PREDICT_ENTRIES:
        if mask_pkl is not None and len(model_dirs) > 1:
            # the reference zips one model's masks against the ensemble's weights
            raise SystemExit("%s with mask_pkl takes one model_dir, got %d: the masks belong to one model" % (entry, len(model_dirs)))
        return {"mask_pkl": mask_pkl}
    partial = bool(_entry_key(cfg, ep, "partial_tuning") or False)
    if partial and pruning is not None:
        # the recipe prunes in one run and tunes in the next; in one run the two writes of mask.pkl would collide
        raise SystemExit("prune_tune_train: partial_tuning together with a pruning schedule is outside this path (prune in one run, "
                         "tune the pruned weights in the next)")
    return {"partial_tuning": partial, "mask_pkl": mask_pkl}


def _finish_plan(plan, cfg, ep, tp, search_method, model_dirs, text=False):
    """Prediction batch size, search, validator and ensemble settings shared by the speech and text plans, and the trainer's
    weight pruning, Prune-Tune flags and initial_global_step."""
    plan["pruning"] = resolve_pruning(cfg, ep)
    plan["prune_tune"] = resolve_prune_tune(cfg, ep, plan["entry"], plan["pruning"], model_dirs)
    igs = _entry_key(cfg, ep, "initial_global_step")
    plan["initial_global_step"] = None if igs is None else int(igs)
    if plan["initial_global_step"] is not None and plan["initial_global_step"] < 0:
        raise SystemExit("initial_global_step must be >= 0")
    # the task's configuration, recorded in model_configs.yml so that a model directory names its vocabularies
    plan["task_config"] = {"task.class": "Seq2Seq" if text else "SpeechToText", "task.params": dict(tp)}
    if ep.get("pretrain_variable_pattern") is not None:
        plan["pretrain_variable_pattern"] = _pretrain_patterns(ep)
    if cfg.get("batch_size") is not None:     # prediction recipes: utterances per batch (SequenceGenerator)
        plan["batch_size"] = int(cfg["batch_size"])
    if search_method:
        plan["search_method"] = search_method
    validator = resolve_validator(cfg, tp, text=text)
    if validator is not None:
        plan["validator"] = validator
        if validator["search_method"]:
            # eval_batch_size x beam_size must fit a decoding step: refused now, not at the first validation
            from neurst_b200.validation import generation_plan
            decode_settings(generation_plan(plan))
    if len(model_dirs) > 1 and search_method == "top_sampling":
        # EncoderDecoderEnsembleModel hands TopSampling one logits tensor per member, which its search cannot take
        raise SystemExit("search_method top_sampling is outside this path for an ensemble of %d model_dirs (beam_search only)"
                         % len(model_dirs))
    if len(model_dirs) > 1:
        # BeamSearch's ensemble_weights: search_method.params, then entry.params (where the flat --ensemble_weights lands)
        sp = cfg.get("search_method.params") or {}
        spec = sp.get("ensemble_weights", ep.get("ensemble_weights"))
        from neurst_b200.decode import ensemble_weights
        try:
            plan["ensemble_weights"] = ensemble_weights("average" if spec is None else spec, len(model_dirs))
        except ValueError as e:
            raise SystemExit("ensemble_weights %r for %d models: %s" % (spec, len(model_dirs), e))
    return plan


def flatten_string_list(arg):
    """A string or a list of strings, each of which may hold comma-separated items -> the list of items (the reference's
    neurst/utils/misc.py:64-74)."""
    if arg is None:
        return None
    items = arg if isinstance(arg, (list, tuple)) else [arg]
    return [c.strip() for cs in items for c in str(cs).split(",") if c.strip()]


# ------------------------------------------------------------------------------------------------ checkpoints
def latest_checkpoint(model_dir):
    """(path, step) of the newest `ckpt-<step>.npz` under model_dir (tf.train.latest_checkpoint's role), or (None, 0)."""
    best = (None, 0)
    for p in glob.glob(os.path.join(model_dir, "ckpt-*.npz")):
        m = re.search(r"ckpt-(\d+)\.npz$", p)
        if m and int(m.group(1)) >= best[1]:
            best = (p, int(m.group(1)))
    return best


def restore_checkpoint(model_dir):
    """(path, step) of the archive to restore from a directory: the one the `checkpoint` index names as
    model_checkpoint_path when it exists (the kept-best `ckpt-<step>-<metric>.npz` of best/ and best_avg/), else the
    newest `ckpt-<step>.npz`.  In a directory `train` wrote the index names the newest archive, so both agree."""
    try:
        with open(os.path.join(model_dir, "checkpoint")) as f:
            name = json.load(f)["model_checkpoint_path"]
    except (OSError, ValueError, KeyError, TypeError):
        name = None
    if name:
        path = os.path.join(model_dir, os.path.basename(name))
        m = re.match(r"ckpt-(\d+)(-[^/]*)?\.npz$", os.path.basename(path))
        if m and os.path.isfile(path):
            return path, int(m.group(1))
    return latest_checkpoint(model_dir)


def save_checkpoint(rt, model_dir, step, max_to_keep=8):
    from neurst_b200 import checkpoints as CK
    os.makedirs(model_dir, exist_ok=True)
    path = os.path.join(model_dir, "ckpt-%d.npz" % step)
    tmp = path + ".tmp.npz"
    CK.save_npz(rt, tmp)
    os.replace(tmp, path)
    kept = sorted((int(re.search(r"ckpt-(\d+)\.npz$", p).group(1)), p) for p in glob.glob(os.path.join(model_dir, "ckpt-*.npz")))
    for _, p in kept[:-max_to_keep] if max_to_keep > 0 else []:
        os.remove(p)
    with open(os.path.join(model_dir, "checkpoint"), "w") as f:          # the index file the reference's managers keep
        json.dump({"model_checkpoint_path": os.path.basename(path), "all_model_checkpoint_paths": [os.path.basename(p) for _, p in kept[-max_to_keep:]]}, f)
    return path


MODEL_CONFIGS = "model_configs.yml"


def write_model_configs(plan):
    """<model_dir>/model_configs.yml with the model's class and parameters (ModelConfigs.dump, written when training begins as
    the reference's checkpoint callback does, neurst/training/callbacks.py:81): what an ensemble member is rebuilt from."""
    import yaml
    os.makedirs(plan["model_dir"], exist_ok=True)
    path = os.path.join(plan["model_dir"], MODEL_CONFIGS)
    with open(path + ".tmp", "w") as f:
        cls = "WaitkTransformer" if plan.get("wait_k") is not None else plan.get("model_class", "SpeechTransformer")
        configs = {"model.class": cls, "model.params": dict(plan["model_params"])}
        configs.update(plan.get("task_config") or {})
        yaml.safe_dump(configs, f, default_flow_style=False)
    os.replace(path + ".tmp", path)


def member_model_params(plan, model_dir):
    """Architecture of one ensemble member: <model_dir>/model_configs.yml when it exists (ModelConfigs.load), else the run's
    model.params / hparams_set."""
    import yaml
    path = os.path.join(model_dir, MODEL_CONFIGS)
    if not os.path.exists(path):
        return plan["model_params"]
    with open(path) as f:
        cfg = yaml.safe_load(f) or {}
    cls = str(cfg.get("model.class", "SpeechTransformer")).lower().replace("_", "")
    if cls in WAITK_MODELS:
        raise SystemExit("%s: a wait-k model (WaitkTransformer) in an ensemble of model_dirs is outside this path" % path)
    if plan.get("model_class") == "Transformer":
        if cls not in TEXT_MODELS:
            raise SystemExit("%s: model.class %r is outside this path for the seq2seq task (Transformer only)"
                             % (path, cfg.get("model.class")))
    elif cls not in SPEECH_MODELS:
        raise SystemExit("%s: model.class %r is outside this path (SpeechTransformer only)" % (path, cfg.get("model.class")))
    return dict(cfg.get("model.params") or {})


# ------------------------------------------------------------------------------------------------ entries
def _dist_setup():
    world, rank, local = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("neurst_b200.cli needs a CUDA device: the product path has no CPU fallback")
    torch.cuda.set_device(local)
    if world > 1 and not torch.distributed.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        torch.distributed.init_process_group("nccl", device_id=torch.device("cuda", local))
    return world, rank, local


def _build_model(plan):
    from neurst_b200.models import SpeechTransformer, Transformer, WaitkTransformer
    tm = {k: v for k, v in plan["trg_meta"].items() if k != "tokens"}
    # only the target table feeds the tensor cores (logits GEMM and its gradient); the source table is gathered and
    # scatter-added in fp32, so a source vocabulary of any size runs on the 16-bit path
    if plan["precision"] != "fp32" and tm["vocab_size"] % 8 != 0:
        raise SystemExit("the 16-bit tensor-core path needs a target vocabulary size that is a multiple of 8 (TMA row alignment of the "
                         "logits gradient); this vocabulary has %d entries (tokens + <UNK>, <SEQ_BEG>, <SEQ_END>): pad the vocabulary file "
                         "with %d unused tokens or run with --dtype float32" % (tm["vocab_size"], -tm["vocab_size"] % 8))
    if plan.get("model_class") == "Transformer":
        sm = {k: v for k, v in plan["src_meta"].items() if k != "tokens"}
        try:
            if plan.get("wait_k") is not None:
                return WaitkTransformer.new(plan["model_params"], sm, tm, precision=plan["precision"],
                                            label_smoothing=plan["label_smoothing"], wait_k=plan["wait_k"], random_seed=plan["seed"])
            return Transformer.new(plan["model_params"], sm, tm, precision=plan["precision"], label_smoothing=plan["label_smoothing"])
        except (NotImplementedError, ValueError) as e:
            raise SystemExit(str(e))
    src_meta = {"audio_feature_dim": plan["task"]["audio_feature_dim"], "audio_feature_channels": plan["task"]["audio_feature_channels"]}
    return SpeechTransformer.new(plan["model_params"], src_meta, tm, precision=plan["precision"], label_smoothing=plan["label_smoothing"])


def _examples(plan, rank, world, training, with_label=None):
    """Endless (training) or single-pass stream of preprocessed samples of this rank's file shard (with the transcripts
    when training or `with_label`).  The text task reads the whole corpus on every rank: its batches are global and
    each rank takes its share of every one (Seq2Seq.train_batches), so all ranks run the same shape at each step.  Text
    `predict` is single-rank: with WORLD_SIZE > 1 every rank decodes the whole file and rank 0 writes it."""
    if plan.get("model_class") == "Transformer":
        from neurst_b200.data import Seq2Seq
        from neurst_b200.text import ParallelTextDataset
        ds = ParallelTextDataset(plan["dataset"])
        task = Seq2Seq(plan["src_meta"], plan["trg_meta"], world=world, **plan["task"])
        proc = task.preprocess_fn(ds.status, training=training, with_label=training if with_label is None else with_label)

        def text_stream():
            while True:
                n = 0
                for ex in ds.build_iterator(map_func=proc)():
                    n += 1
                    yield ex
                if not training or n == 0:
                    return
        return task, text_stream()
    from neurst_b200.data import SpeechToText
    from neurst_b200.tfrecord import AudioTFRecordDataset
    ds = AudioTFRecordDataset(plan["dataset"])
    tk = dict(plan["task"])
    task = SpeechToText({k: v for k, v in plan["trg_meta"].items() if k != "tokens"}, world=1,
                        padding_mode=plan["trg_meta"]["padding_mode"], **tk)
    proc = task.preprocess_fn(ds.status, training=training, with_label=training if with_label is None else with_label)
    from neurst_b200.tfrecord import glob_tfrecords
    shards = world if len(glob_tfrecords(plan["dataset"]["data_path"])) >= world else 1     # fewer files than ranks: every rank reads all

    def stream():
        while True:
            n = 0
            for ex in ds.build_iterator(map_func=proc, shard_id=rank if shards > 1 else 0, total_shards=shards)():
                n += 1
                yield ex
            if not training or n == 0:
                return
    return task, stream()


def initialise(model, plan):
    """The model's starting weights: the newest checkpoint of model_dir (resume), else pretrain_model, else its own
    initialisation.  -> the step to resume from."""
    from neurst_b200 import checkpoints as CK
    start_path, start_step = latest_checkpoint(plan["model_dir"])
    if start_path:
        CK.load_npz(model.runtime, start_path)
        LOG.info("restored %s", start_path)
    elif plan["pretrain_model"] and plan.get("pretrain_variable_pattern"):
        # restore_checkpoint_if_possible per (archive, pattern): the model's own initialisation stays everywhere else
        model.init_parameters(plan["seed"])
        for src, pattern in zip(flatten_string_list(plan["pretrain_model"]), plan["pretrain_variable_pattern"]):
            src = restore_checkpoint(src)[0] if os.path.isdir(src) else src
            if not src:
                raise SystemExit("pretrain_model: no checkpoint to restore")
            got = CK.load_npz(model.runtime, src, strict=False, pattern=pattern, slots=False)
            LOG.info("initialised %d tensors from %s (pattern %r)", len(got), src, pattern)
    elif plan["pretrain_model"]:
        src = plan["pretrain_model"][0] if isinstance(plan["pretrain_model"], (list, tuple)) else plan["pretrain_model"]
        src = restore_checkpoint(src)[0] if os.path.isdir(src) else src
        CK.load_npz(model.runtime, src, strict=False, slots=False)
        LOG.info("initialised from %s", src)
    else:
        model.init_parameters(plan["seed"])
    return start_step


def train(plan):
    from neurst_b200 import prune_tune as PT
    from neurst_b200.trainer import DataParallelTrainer, HostPipeline
    world, rank, local = _dist_setup()
    model = _build_model(plan)
    resumed = latest_checkpoint(plan["model_dir"])[0] is not None
    start_step = initialise(model, plan)
    # initial_global_step wins over a restored checkpoint's step (exps/trainer.py:172-178): the noam position, the checkpoint
    # numbers and the validation steps count from it, and the run makes train_steps updates (the reference's steps_per_epoch)
    igs = plan.get("initial_global_step")
    end_step = plan["train_steps"] if igs is None else igs + plan["train_steps"]
    if igs is not None:
        start_step = igs
    pruning = plan.get("pruning")
    schedule = names = None
    if pruning:
        from neurst_b200.pruning import pruned_parameters
        schedule = pruning["schedule"]
        names = pruned_parameters(model.runtime.table, pruning["pruning_variable_pattern"], pruning["nopruning_variable_pattern"])
        if not names:
            raise SystemExit("pruning: the variable patterns select no parameter tensor")
        LOG.info("Pruning: %s, %d of %d parameter tensors will be pruned", type(schedule).__name__, len(names),
                 len(model.runtime.table))
    prune_tune = plan.get("prune_tune") or {}
    partial = _partial_tuning_masks(model, plan, resumed) if prune_tune.get("partial_tuning") else None
    trainer = DataParallelTrainer(model, plan["optimizer"], plan["lr_schedule"], update_cycle=plan["update_cycle"],
                                  use_cuda_graph=True, clip_value=plan["clip_value"], clip_norm=plan["clip_norm"],
                                  summary_steps=plan["summary_steps"] if rank == 0 else 0, logger=LOG.info,
                                  pruning_schedule=schedule, pruning_variables=names, partial_tuning_mask=partial)
    trainer.global_step = start_step
    if igs is not None:
        # only the lr schedule, the checkpoints and validation read the initial step (compat.register_initial_step); the
        # optimizer's iterations start at 0 in this run, so Adam's bias correction counts this run's updates from t = 1
        trainer.adam_step_base = igs
        if model.runtime.loss_scale_state is not None:
            model.runtime.loss_scale_state[4] = 0.0       # the dynamic loss scale's t: the updates applied in this run

    def log_sparsity():
        if schedule is not None and trainer._pruning_ready:
            zeros, total = model.runtime.prune_sparsity()
            LOG.info("Pruning: %d of %d weights of the pruned tensors are zero (sparsity %.4f)", zeros, total, zeros / total)
            return zeros, total
        return None
    trainer.broadcast_parameters()
    if rank == 0:
        write_model_configs(plan)
    mask_path = os.path.join(plan["model_dir"], PT.MASK_FILE)
    if partial is not None:
        tuned, frozen = trainer.setup_partial_tuning()
        LOG.info("Partial tuning: %d weights are tuned, %d frozen (masks from %s)", tuned, frozen,
                 "the non-zero weights" if isinstance(partial, str) else prune_tune.get("mask_pkl") or mask_path)
        if rank == 0:
            # the reference writes the loaded masks (None without mask_pkl) at the end only; this path writes the masks it
            # tunes with before the first update, so that a resumed run finds them, and again at the end
            os.makedirs(plan["model_dir"], exist_ok=True)
            PT.save_masks(model.runtime, mask_path, model.runtime.partial_frozen)
    validator = None
    if plan.get("validator"):
        from neurst_b200.validation import Validator
        validator = Validator(plan, model, rank, world)
        if plan["validator"]["eval_on_begin"]:
            validator.validate(start_step)
    task, examples = _examples(plan, rank, world, training=True)
    gen = torch.Generator().manual_seed(plan["seed"] + rank)
    from neurst_b200.data import Prefetcher
    import itertools
    last = None
    early_stopped = False
    micro_target = (end_step - start_step) * plan["update_cycle"]
    if micro_target > 0:
        # reading, parsing, padding and pinning of the next batches run in a background thread (tf.data prefetch's role)
        share = rank if plan.get("model_class") == "Transformer" else 0      # the text task's batches are global
        batches = Prefetcher(itertools.islice((per_rank[share] for per_rank in task.train_batches(examples, generator=gen, pin=True)),
                                              micro_target), depth=4, init=lambda: torch.cuda.set_device(local))
        try:
            pipeline = HostPipeline(trainer)
            losses = pipeline.run(batches, seed0=start_step * plan["update_cycle"] + 1)
            saved_at = validated_at = start_step
            for loss in losses:
                if loss is not None:
                    last = loss
                step = trainer.global_step
                if rank == 0 and step > saved_at and step % plan["save_checkpoint_steps"] == 0:
                    torch.cuda.synchronize()
                    save_checkpoint(model.runtime, plan["model_dir"], step, plan["max_to_keep"])
                    saved_at = step
                    log_sparsity()
                # the step's kernels (and its optimizer update) are done once validate() synchronises; the next step is
                # launched only when this generator resumes, so every rank validates the same weights
                if validator is not None and step > validated_at and validator.due(step):
                    validated_at = step
                    if validator.validate(step)[1]:
                        early_stopped = True
                        last = pipeline.latest_loss()      # the losses arrive one step late: read the stopping step's
                        break
        finally:
            batches.close()
    torch.cuda.synchronize()
    if rank == 0 and trainer.global_step > start_step:
        save_checkpoint(model.runtime, plan["model_dir"], trainer.global_step, plan["max_to_keep"])
    if rank == 0 and plan["entry"] == "prune_tune_train" and (partial is not None or schedule is not None):
        # partial_trainer.py:188-206: after a pruning run weight != 0 over every variable, after a partial tuning its masks
        rt = model.runtime
        PT.save_masks(rt, mask_path, rt.partial_frozen if partial is not None else rt.derive_prune_mask(list(rt.table)))
        LOG.info("wrote the masks to %s", mask_path)
    sparsity = log_sparsity() if rank == 0 else None
    if world > 1:
        trainer.close()
        torch.distributed.barrier()
    res = {"global_step": trainer.global_step, "loss": last}
    if partial is not None:
        res["partial_tuning"] = {"tuned": trainer.partial_counts[0], "frozen": trainer.partial_counts[1]}
    if sparsity is not None:
        # the schedule's device state: updates applied in this run, pruning turns, the last turn's sparsity
        import struct
        st = [int(x) for x in model.runtime.prune_state.cpu()]
        res["pruning"] = {"zeros": sparsity[0], "weights": sparsity[1], "sparsity": sparsity[0] / sparsity[1],
                          "updates": st[0], "turns": st[2], "turn_sparsity": struct.unpack("<f", struct.pack("<i", st[3]))[0],
                          "tensors": len(names)}
    if validator is not None:
        res.update(early_stopped=early_stopped, validations=validator.history)
    return res


def _partial_tuning_masks(model, plan, resumed):
    """The masks of a partial-tuning run (partial_tuning_optimizer.py:50-80): those of mask_pkl; else "weights", i.e.
    weight != 0 of the restored or pretrained weights.  One deliberate deviation: a run that resumes from a checkpoint of its
    own model_dir without mask_pkl reads <model_dir>/mask.pkl, which the run wrote before its first update: the reference
    would re-derive the masks from the tuned weights, in which nearly every weight is non-zero, and freeze them all."""
    from neurst_b200 import prune_tune as PT
    path = plan["prune_tune"]["mask_pkl"]
    if path is None and resumed:
        path = os.path.join(plan["model_dir"], PT.MASK_FILE)
        if not os.path.isfile(path):
            raise SystemExit("partial tuning resumes from a checkpoint of %s, which holds no %s: give --mask_pkl (masks "
                             "derived from the tuned weights would freeze nearly every weight)" % (plan["model_dir"], PT.MASK_FILE))
    if path is None:
        return "weights"
    try:
        return PT.load_masks(model.runtime, path)
    except PT.MaskFileError as e:
        raise SystemExit(str(e))


def ids_to_text(ids, eos_id, tokens):
    out = []
    for i in ids:
        if i == eos_id:
            break
        out.append(int(i))
    if tokens is None:
        return " ".join(str(i) for i in out)
    words = [tokens[i] if i < len(tokens) else "<UNK>" for i in out]
    return " ".join(words).replace("@@ ", "")                            # BPE continuation marks (subword-nmt convention)


def _restore(plan, model_dir):
    from neurst_b200 import checkpoints as CK
    model = _build_model(plan)
    path, step = restore_checkpoint(model_dir)
    if not path:
        raise SystemExit("no ckpt-*.npz under %s" % model_dir)
    CK.load_npz(model.runtime, path)
    return model, step


def decode_settings(plan):
    """(utterances per search call, search keyword arguments) of `predict` and the validators' generation.  The recipes'
    batch_size (utterances per batch): with 16-bit weights the batch is decoded in one call from the 16-bit shadow, up
    to MAX_ROWS_SHADOW rows (utterances x beam) per step; the fp32 weights hold MAX_ROWS rows per step."""
    from neurst_b200.decode import MAX_ROWS, MAX_ROWS_SHADOW
    beam = plan.get("search_method") == "beam_search"
    sampling = plan.get("search_method") == "top_sampling"
    width = plan["search"]["beam_size"] if beam else plan["search"]["sample_num"] if sampling else 1
    what = "sample_num" if sampling else "beam_size"
    per_call = MAX_ROWS // width
    if per_call < 1:
        raise SystemExit("%s %d exceeds the %d rows a decoding step holds" % (what, width, MAX_ROWS))
    search_kw = dict(plan["search"])
    if plan.get("batch_size") is not None:
        if plan["precision"] == "fp32":
            LOG.info("dtype float32 decodes %d utterance(s) per call (at most %d rows per step), not batch_size %d",
                     min(per_call, plan["batch_size"]), MAX_ROWS, plan["batch_size"])
            per_call = min(per_call, plan["batch_size"])
        else:
            if not 1 <= plan["batch_size"] * width <= MAX_ROWS_SHADOW:
                raise SystemExit("batch_size %d x %s %d exceeds the %d rows a decoding step holds"
                                 % (plan["batch_size"], what, width, MAX_ROWS_SHADOW))
            per_call = plan["batch_size"]
            search_kw["use_shadow"] = True
    return per_call, search_kw


def sampling_seed(seed, rank):
    """The draws' seed of one rank: the run's random_seed with the rank folded in (rank 0 keeps it)."""
    return (int(seed) + int(rank) * 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF


def search_fn(model, plan):
    """The model's search for the plan's search_method: beam_search, top_sampling, or greedy without one."""
    name = {"beam_search": "beam_search", "top_sampling": "sampling_search"}.get(plan.get("search_method"), "greedy_search")
    return getattr(model, name)


def decode_group(model, task, plan, group, search_kw, first=0, lengths=None):
    """One search call over preprocessed samples -> [(ids_to_text hypothesis, score)], top_k (beam search) or sample_num
    (top_sampling) rows per utterance, consecutive (the reference's [B*top_k] order).  `first`: the position of group[0] in
    the rank's stream of utterances, which keys the samples' draws (row offset first * sample_num), so the samples do not
    depend on how the stream is cut into calls.  `lengths` (a list): receives (source tokens without EOS, hypothesis tokens
    without EOS) per row, the model-token lengths of the wait-k latency."""
    tm = plan["trg_meta"]
    if plan.get("model_class") == "Transformer":
        batch = task.group_to_input(group, infer=True)
        inputs = {"src": batch["src"], "src_padding": batch["src_padding"]}
    else:
        dim = plan["task"]["audio_feature_dim"] * plan["task"]["audio_feature_channels"]
        T = max(int(e["audio_length"]) for e in group)
        src = torch.zeros(len(group), T, dim)
        for j, e in enumerate(group):
            src[j, :int(e["audio_length"])] = e["audio"]
        batch = task.example_to_input({"audio": src, "audio_length": torch.tensor([int(e["audio_length"]) for e in group])}, infer=True)
        inputs = {"src": batch["src"], "src_length": batch["src_length"]}
    if plan.get("search_method") == "top_sampling":
        search_kw = dict(search_kw, row_offset=int(first) * plan["search"]["sample_num"])
    ids, score = search_fn(model, plan)(inputs, **search_kw)
    if lengths is not None:
        per = ids.shape[0] // len(group)
        for r, row in enumerate(ids.cpu().tolist()):
            n = next((i for i, x in enumerate(row) if x == tm["eos_id"]), len(row))
            lengths.append((int(group[r // per]["feature"].numel()) - 1, n))
    return [(ids_to_text(row, tm["eos_id"], tm.get("tokens")), lp) for row, lp in zip(ids.cpu().tolist(), score.cpu().tolist())]


def predict(plan):
    from neurst_b200.models import EncoderDecoderEnsembleModel
    world, rank, _ = _dist_setup()
    ensemble = isinstance(plan["model_dir"], list)
    if ensemble:
        # SequenceGenerator._build_and_restore_model: each member from its own directory, all at the run's dtype
        members = [_restore(dict(plan, model_params=member_model_params(plan, d)), d) for d in plan["model_dir"]]
        model = EncoderDecoderEnsembleModel.new([m for m, _ in members])
        step = [s for _, s in members]
        LOG.info("predict: ensemble of %d models (%s), weights %s", model.model_num, ", ".join(plan["model_dir"]),
                 plan["ensemble_weights"])
    else:
        model, step = _restore(plan, plan["model_dir"])
        mask_pkl = (plan.get("prune_tune") or {}).get("mask_pkl")
        if mask_pkl:
            # mask_sequence_generator.py:74-84: every weight times its mask, on the device, before the search
            from neurst_b200 import prune_tune as PT
            try:
                masks = PT.load_masks(model.runtime, mask_pkl)
            except PT.MaskFileError as e:
                raise SystemExit(str(e))
            model.runtime.apply_mask(PT.mask_bitmap(model.runtime, masks))
            LOG.info("%s: weights masked with %s", plan["entry"], mask_pkl)
    task, examples = _examples(plan, rank, world, training=False)
    per_call, search_kw = decode_settings(plan)
    if ensemble:
        search_kw["ensemble_weights"] = plan["ensemble_weights"]
    if plan.get("search_method") == "top_sampling":
        search_kw["seed"] = sampling_seed(plan["seed"], rank)
    hyps = []
    group = []
    done = 0
    lengths = [] if plan.get("wait_k") is not None else None
    for ex in examples:
        group.append(ex)
        if len(group) == per_call:
            hyps.extend(decode_group(model, task, plan, group, search_kw, first=done, lengths=lengths))
            done += len(group)
            group = []
    if group:
        hyps.extend(decode_group(model, task, plan, group, search_kw, first=done, lengths=lengths))
    out = plan["output_file"]
    if out and rank == 0:
        with open(out, "w", encoding="utf-8") as f:
            for text, _ in hyps:
                f.write(text + "\n")
    result = {"checkpoint_step": step, "hypotheses": hyps}
    if lengths is not None:
        # the offline wait-k schedule's latency, in model (BPE) tokens: not comparable with SimulEval's word-level numbers
        from neurst_b200.metrics import corpus_waitk_latency
        k = model.lag(False)
        result["latency"] = corpus_waitk_latency(k, lengths)
        if result["latency"] is not None:
            LOG.info("predict: wait-k %d latency over %d hypotheses (BPE tokens): AL %.4f AP %.4f DAL %.4f", k, len(lengths),
                     result["latency"]["AL"], result["latency"]["AP"], result["latency"]["DAL"])
    return result


def _cascade_references(plan, key, meta):
    """The reference texts of one key of the audio records (ids -> text), or None when the records do not hold it."""
    from neurst_b200.tfrecord import AudioTFRecordDataset, take_one_record
    asr_ds = plan["asr"]["dataset"]
    kind = take_one_record(asr_ds["data_path"]).get(key, (None, None))[0]
    if kind is None:
        return None
    if kind != "int64":
        raise SystemExit("the %r key holds raw text: the reference's text pipeline (tokenizer / BPE / vocabulary) is outside this "
                         "path; write the TFRecords with projected (int64) ids" % key)
    ds = AudioTFRecordDataset(dict(asr_ds, transcript_key=key))
    return [ids_to_text(list(x["transcript"]), meta["eos_id"], meta.get("tokens")) for x in ds.build_iterator()()]


def cascade_st(plan):
    """ASR search, then, per group of utterances on the same stream, the handoff kernel (b200st_cascade_source: ASR top-1
    ids -> MT source ids through the vocabulary remap table), one copy of the source lengths to the host, and the MT
    encoder and search: no host text between the two models."""
    from neurst_b200 import decode as D
    from neurst_b200.metrics import build_metric
    _dist_setup()
    asr_plan, mt_plan = plan["asr"], plan["mt"]
    asr, _ = _restore(asr_plan, asr_plan["model_dir"])
    mt, _ = _restore(mt_plan, mt_plan["model_dir"])
    task, examples = _examples(asr_plan, 0, 1, training=False, with_label=False)
    asr_meta, src_meta, trg_meta = asr_plan["trg_meta"], mt_plan["src_meta"], mt_plan["trg_meta"]
    if not asr_meta.get("tokens"):
        raise SystemExit("cascade_st maps ASR tokens to MT tokens by string: the ASR model directory needs its vocab_path")
    remap = D.cascade_remap(asr_meta["tokens"], src_meta["tokens"], src_meta["unk_id"], asr_meta["vocab_size"]).cuda()
    asr_per_call, asr_kw = decode_settings(asr_plan)
    mt_per_call, mt_kw = decode_settings(mt_plan)
    per_call = min(asr_per_call, mt_per_call)
    asr_search, mt_search = search_fn(asr, asr_plan), search_fn(mt, mt_plan)
    asr_hyps, mt_hyps = [], []

    def run(group):
        batch = task.example_to_input({"audio": _pad_audio(asr_plan, group), "audio_length": torch.tensor(
            [int(e["audio_length"]) for e in group])}, infer=True)
        ids, _ = asr_search({"src": batch["src"], "src_length": batch["src_length"]}, **asr_kw)
        asr_hyps.extend(ids_to_text(r, asr_meta["eos_id"], asr_meta["tokens"]) for r in ids.cpu().tolist())
        src, padding, _ = D.cascade_source(ids, remap, asr_meta["eos_id"], src_meta["vocab_size"], src_meta["eos_id"],
                                           src_meta["pad_id"], src_meta["unk_id"])
        out, _ = mt_search({"src": src, "src_padding": padding}, **mt_kw)
        mt_hyps.extend(ids_to_text(r, trg_meta["eos_id"], trg_meta["tokens"]) for r in out.cpu().tolist())

    group = []
    for ex in examples:
        group.append(ex)
        if len(group) == per_call:
            run(group)
            group = []
    if group:
        run(group)
    res = {"asr_hypotheses": asr_hyps, "mt_hypotheses": mt_hyps}
    for side, key, meta, hyps in (("asr", asr_plan["dataset"]["transcript_key"], asr_meta, asr_hyps),
                                  ("mt", plan["translation_key"], trg_meta, mt_hyps)):
        out = plan[side + "_output_file"]
        if out:
            with open(out, "w", encoding="utf-8") as f:
                f.write("".join(h + "\n" for h in hyps))
        refs = _cascade_references(plan, key, meta)
        if refs is not None:
            res[side + "_metric"] = build_metric(plan["metrics"][side], "en")(hyps, refs)
            LOG.info("Evaluation Result of %s: %s", side.upper(), res[side + "_metric"])
    return res


def simuleval(plan):
    """Streams every source line through SimulTransTextAgent word by word on the device (simultaneous.py) and writes
    <output>/instances.log (one JSON line per sentence: prediction, delays in source words, the device time of each action)
    and <output>/scores (BLEU from metrics, and AL / AP / DAL of the measured delays from metrics.simul_latency)."""
    from neurst_b200.metrics import build_metric, simul_latency
    from neurst_b200.simultaneous import SimulTransTextAgent, StreamingSession, words_of
    _dist_setup()
    models = [_restore(p, p["model_dir"])[0] for p in plan["members"]]
    first = plan["members"][0]
    with open(plan["source"], encoding="utf-8") as f:
        sources = [l.rstrip("\n") for l in f]
    # the source with the EOS of a forced segment and the final one; the target up to the agent's max_len + 1 units
    max_src = max([len(l.split()) for l in sources] + [1]) + 2
    session = StreamingSession(models, use_shadow=first["precision"] != "fp32", max_src=max_src, max_trg=plan["max_len"] + 2)
    agent = SimulTransTextAgent(session, first["src_meta"], first["trg_meta"], plan["wait_k"], plan["force_segment"], plan["max_len"])
    bow = any(t.startswith("\u2581") for t in first["src_meta"]["tokens"] or [])
    refs = None
    if plan.get("target"):
        with open(plan["target"], encoding="utf-8") as f:
            refs = [l.rstrip("\n") for l in f]

    def clock():
        torch.cuda.synchronize()
        return time.perf_counter()

    os.makedirs(plan["output"], exist_ok=True)
    hyps, lat = [], []
    with open(os.path.join(plan["output"], "instances.log"), "w", encoding="utf-8") as f:
        for i, line in enumerate(sources):
            words = words_of(line, bow)
            r = agent.translate(words, clock=clock)
            hyp = " ".join(r["prediction"])
            hyps.append(hyp)
            row = {"index": i, "prediction": hyp, "delays": r["delays"], "source_length": len(words),
                   "action_seconds": [[a, round(t, 7)] for a, t in r["actions"]]}
            if refs is not None:
                row["reference"] = refs[i]
            m = simul_latency(r["delays"], len(words))
            if m is not None:
                lat.append(m)
                row.update(m)
            f.write(json.dumps(row) + "\n")
    scores = {"n_sentences": len(hyps)}
    for key in ("AL", "AP", "DAL"):
        scores[key] = sum(m[key] for m in lat) / len(lat) if lat else None
    if refs is not None:
        scores["BLEU"] = build_metric("bleu", "en")(hyps, refs)
    with open(os.path.join(plan["output"], "scores"), "w", encoding="utf-8") as f:
        f.write(json.dumps(scores, indent=2) + "\n")
    LOG.info("simuleval: %s", json.dumps(scores))
    return dict(scores, hypotheses=hyps)


def _pad_audio(plan, group):
    dim = plan["task"]["audio_feature_dim"] * plan["task"]["audio_feature_channels"]
    src = torch.zeros(len(group), max(int(e["audio_length"]) for e in group), dim)
    for j, e in enumerate(group):
        src[j, :int(e["audio_length"])] = e["audio"]
    return src


def main(argv=None):
    logging.basicConfig(level=logging.INFO, format="%(asctime)s %(message)s")
    paths, overrides = parse_command_line(list(sys.argv[1:] if argv is None else argv))
    cfg = load_config(paths, overrides)
    plan = resolve(cfg, world=int(os.environ.get("WORLD_SIZE", "1")))
    if plan["entry"] in TRAIN_ENTRIES:
        res = train(plan)
        if "validations" in res:
            res["validations"] = [{k: v for k, v in r.items() if k != "hypotheses"} for r in res["validations"]]
    elif plan["entry"] == "simuleval":
        res = {k: v for k, v in simuleval(plan).items() if k != "hypotheses"}
    elif plan["entry"] == "cascade_st":
        res = cascade_st(plan)
        res = {k: v for k, v in res.items() if not k.endswith("_hypotheses")}
    elif plan["entry"] in PREDICT_ENTRIES:
        res = predict(plan)
        res = {"checkpoint_step": res["checkpoint_step"], "n_hypotheses": len(res["hypotheses"])}
    else:
        raise SystemExit("entry.class %r is outside this path (trainer, prune_tune_train, predict, mask_predict)" % plan["entry"])
    LOG.info("%s", json.dumps(res))
    return res


if __name__ == "__main__":
    main()
