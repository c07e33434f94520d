"""Validation during training: the recipes' CriterionValidator / SeqGenerationValidator with their recorder and
checkpoint savers.

  Validator scheduling               neurst/training/validator.py:52-62
  dev loss (NLL, PPL)                neurst/training/criterion_validator.py:101-134, LabelSmoothedCrossEntropy.reduce_metrics
  dev generation + metric            neurst/training/seq_generation_validator.py:164-233
  TrainingStatusRecorder             neurst/training/training_utils.py:274-370 (early stop ends training cleanly instead of
                                     the reference's SIGUSR1)
  KeepBestCheckpointSaver            neurst/utils/checkpoints.py:186-232   <dir>/best:     ckpt-<step>-<metric %.2f>.npz
  AverageCheckpointSaver             neurst/utils/checkpoints.py:235-305   <dir>/best_avg: np.average of the last N evaluations

The savers and the recorder are host code over a {variable name: ndarray} snapshot; `Validator` runs the dev set on the
device through the model's forward (dev loss) and `cli.decode_group` (the hypotheses `predict` writes).
"""
import functools
import json
import logging
import os
import random
import time

import numpy as np

LOG = logging.getLogger("neurst_b200")


# ------------------------------------------------------------------------------------------------ savers
class _CustomSaver:
    """neurst/utils/checkpoints.py:_CustomSaver: a directory, a bounded list of (name, value) kept in the saver's order
    and the `checkpoint` index naming the last entry (the best) as model_checkpoint_path."""

    def __init__(self, directory, metric, max_to_keep):
        self.directory = directory
        self._metric = metric
        self._max_to_keep = max_to_keep
        self._all_model_checkpoints = []
        os.makedirs(directory, exist_ok=True)

    @property
    def kept(self):
        return list(self._all_model_checkpoints)

    def _should_save(self, metric_value):
        return (0 <= len(self._all_model_checkpoints) < self._max_to_keep
                or self._metric.greater_or_eq(metric_value, self._all_model_checkpoints[0][1]))

    def _write(self, step, metric_value, arrays):
        prefix = "ckpt-%d-%s" % (step, "%.2f" % self._metric.get_value(metric_value))
        path = os.path.join(self.directory, prefix + ".npz")
        tmp = path + ".tmp.npz"
        np.savez(tmp, **arrays)
        os.replace(tmp, path)
        self._all_model_checkpoints.append((prefix, self._metric.get_value(metric_value)))
        # the reference's comparator: y sorts before x only when y is strictly better, so the best ends up last
        self._all_model_checkpoints = sorted(
            self._all_model_checkpoints,
            key=functools.cmp_to_key(lambda x, y: (-int(self._metric.greater_or_eq(y[1], x[1]) and y[1] != x[1]))))
        while len(self._all_model_checkpoints) > self._max_to_keep:
            old, _ = self._all_model_checkpoints.pop(0)
            if os.path.exists(os.path.join(self.directory, old + ".npz")):
                os.remove(os.path.join(self.directory, old + ".npz"))
        names = [p + ".npz" for p, _ in self._all_model_checkpoints]
        index = os.path.join(self.directory, "checkpoint")
        with open(index + ".incomplete", "w") as f:
            json.dump({"model_checkpoint_path": names[-1], "all_model_checkpoint_paths": names}, f)
        os.replace(index + ".incomplete", index)
        return path


class KeepBestCheckpointSaver(_CustomSaver):
    """Saves the current weights when fewer than `max_to_keep` are kept or the value is at least as good as the worst kept."""

    def save(self, step, metric_value, arrays):
        """-> the written path, or None."""
        if not self._should_save(metric_value):
            return None
        return self._write(step, metric_value, arrays)


class AverageCheckpointSaver(_CustomSaver):
    """Keeps the last `max_to_keep` evaluated snapshots; when the value ranks as KeepBestCheckpointSaver's would, saves
    np.average over them (per variable, axis 0)."""

    def __init__(self, directory, metric, max_to_keep):
        super().__init__(directory, metric, max_to_keep)
        self._snapshots = []

    def save(self, step, metric_value, arrays):
        self._snapshots.append(arrays)
        if len(self._snapshots) > self._max_to_keep:
            self._snapshots.pop(0)
        if not self._should_save(metric_value):
            return None
        avg = {k: np.average([s[k] for s in self._snapshots], axis=0) for k in arrays}
        return self._write(step, metric_value, avg)


class TrainingStatusRecorder:
    """training_utils.py:274-370: keeps the best result and a count of evaluations without improvement, drives the two
    savers.  `record` returns True when `estop_patience` evaluations in a row brought no improvement."""

    def __init__(self, metric, model_dir=None, estop_patience=None, best_checkpoint_path=None, auto_average_checkpoints=True,
                 best_avg_checkpoint_path=None, top_checkpoints_to_keep=0, model_configs=None):
        self._metric = metric
        self._estop_patience = estop_patience
        self.best_saver = self.avg_saver = None
        if top_checkpoints_to_keep and top_checkpoints_to_keep > 0:
            self.best_saver = KeepBestCheckpointSaver(best_checkpoint_path or os.path.join(model_dir, "best"), metric,
                                                      top_checkpoints_to_keep)
            dirs = [self.best_saver.directory]
            if auto_average_checkpoints:
                self.avg_saver = AverageCheckpointSaver(best_avg_checkpoint_path or os.path.join(model_dir, "best_avg"),
                                                        metric, top_checkpoints_to_keep)
                dirs.append(self.avg_saver.directory)
            if model_configs is not None:
                for d in dirs:
                    model_configs(d)
        self.best = None
        self.bad_count = 0

    def record(self, step, metric_result, snapshot=None):
        """`snapshot()` -> {variable name: host fp32 ndarray}; called only when a saver exists."""
        if self.best is None or self._metric.greater_or_eq(metric_result, self.best):
            self.bad_count = 0
            self.best = metric_result
        else:
            self.bad_count += 1
        arrays = snapshot() if (self.best_saver is not None and snapshot is not None) else None
        if self.best_saver is not None:
            stat = self.best_saver.save(step, metric_result, arrays)
            LOG.info("Checking the best checkpoints kept and %s.", "a new checkpoint was saved" if stat else "no checkpoint was saved.")
        if self.avg_saver is not None and self.avg_saver.save(step, metric_result, arrays):
            LOG.info("An averaged checkpoint was saved.")
        if self._estop_patience is not None:
            LOG.info("Evaluating %s at step=%d with bad count=%d (early_stop_patience=%s).", self._metric.flag, step,
                     self.bad_count, self._estop_patience)
        if self._estop_patience and self.bad_count >= self._estop_patience > 0:
            LOG.info("Hit maximum patience! Early Stop!!!")
            return True
        return False


# ------------------------------------------------------------------------------------------------ device validator
def _batches(items, size):
    return [items[i:i + size] for i in range(0, len(items), size)]


def generation_plan(plan):
    """The plan `predict` would run for the validator's generation: its search and eval_batch_size utterances per batch."""
    vp = plan["validator"]
    return dict(plan, search_method=vp["search_method"], search=vp["search"], batch_size=vp["batch_size"])


class Validator:
    """One validator of a training run (plan["validator"], resolved by cli.resolve).  Every rank evaluates the batches
    b with b % world == rank; rank 0 gathers them back into dev-set order, computes the metrics and writes best/ and
    best_avg/."""

    def __init__(self, plan, model, rank=0, world=1):
        from neurst_b200.metrics import CriterionMetric, build_metric
        from neurst_b200 import cli
        self.plan, self.vp, self.model = plan, plan["validator"], model
        self.rank, self.world = rank, world
        vp = self.vp
        dev_plan = dict(plan, dataset=vp["dataset"], task=dict(plan["task"], **vp["task_args"]))
        self.task, examples = cli._examples(dev_plan, 0, 1, training=False, with_label=True)
        self.examples = list(examples)          # the reference caches the dev set (dataset.cache()); features are file views
        tm = plan["trg_meta"]
        self.references = [cli.ids_to_text(e["transcript"].tolist(), tm["eos_id"], tm.get("tokens")) for e in self.examples]
        self.criterion_metric = CriterionMetric()
        self.loss_recorder = TrainingStatusRecorder(self.criterion_metric)
        self.gen_metric = self.gen_recorder = None
        if vp["class"] == "SeqGenerationValidator" and vp["metric"] and vp["search_method"]:
            self.gen_metric = build_metric(vp["metric"], vp["language"])
            # predict's batching of eval_batch_size utterances per call (rows checked when the plan was resolved)
            self.gen_plan = generation_plan(plan)
            self.per_call, self.search_kw = cli.decode_settings(self.gen_plan)
            if rank == 0:
                self.gen_recorder = TrainingStatusRecorder(
                    self.gen_metric, plan["model_dir"], vp["estop_patience"], vp["best_checkpoint_path"],
                    vp["auto_average_checkpoints"], vp["best_avg_checkpoint_path"], vp["top_checkpoints_to_keep"],
                    model_configs=lambda d: cli.write_model_configs(dict(plan, model_dir=d)))
        elif vp["class"] == "SeqGenerationValidator":
            LOG.info("WARNING: SeqGenerationValidator without eval_metric or eval_search_method validates the loss only")
        self.t0 = time.time()
        self.history = []

    def due(self, step):
        vp = self.vp
        return step >= vp["eval_start_at"] and step % vp["eval_steps"] == 0

    # ---- device work ------------------------------------------------------------------------------------------
    def _loss_sums(self, mine):
        """[(batch index, nll_sum, n_samples, n_tokens)] over this rank's dev batches: the model's forward without dropout
        (logits), then the eval criterion's label-smoothed CE (b200st_lsce), summed in fp64 on the host."""
        import torch
        from neurst_b200.models import LabelSmoothedCrossEntropy
        crit = LabelSmoothedCrossEntropy({"label_smoothing": self.vp["label_smoothing"]})
        rt = self.model.runtime
        if self.plan.get("model_class") == "Transformer":
            return self._text_loss_sums(mine, crit)
        dim = self.plan["task"]["audio_feature_dim"] * self.plan["task"]["audio_feature_channels"]
        pad = int(self.plan["trg_meta"]["pad_id"])
        out = []
        for bi, group in mine:
            # EVAL-mode padded_batch (speech2text.py:273-279): file order, padded to the longest in the batch
            T = max(int(e["audio_length"]) for e in group)
            Lq = max(int(e["transcript"].numel()) for e in group)
            src = torch.zeros(len(group), T, dim)
            trg = torch.full((len(group), Lq), pad, dtype=torch.long)
            for j, e in enumerate(group):
                src[j, :int(e["audio_length"])] = e["audio"]
                trg[j, :e["transcript"].numel()] = e["transcript"]
            b = self.task.example_to_input({"audio": src, "audio_length": torch.tensor([int(e["audio_length"]) for e in group]),
                                            "transcript": trg})
            b = {k: v.to(rt.device) for k, v in b.items()}
            logits = rt.run({"src": b["src"], "src_length": b["src_length"], "trg_input": b["trg_input"], "training": False,
                             "seed": 0, "want_logits": True}, backward=False)["logits"]
            nll, _, ntok = crit(b, logits)
            out.append((bi, float(nll.double().sum()), float(len(group)), float(ntok.double().sum())))
        return out

    def _text_loss_sums(self, mine, crit):
        """_loss_sums of the text model: EVAL-mode padded_batch (seq2seq.py:236-244, padded to the longest source and
        target of the batch).  A wait-k model is evaluated with its first lag (waitk_transformer.py:106-107)."""
        rt = self.model.runtime
        out = []
        for bi, group in mine:
            b = {k: v.to(rt.device) for k, v in self.task.group_to_input(group, infer=False).items()}
            logits = rt.run({"src": b["src"], "src_padding": b["src_padding"], "trg_input": b["trg_input"], "training": False,
                             "seed": 0, "want_logits": True, "wait_k": self.model.lag(False)}, backward=False)["logits"]
            nll, _, ntok = crit(b, logits)
            out.append((bi, float(nll.double().sum()), float(len(group)), float(ntok.double().sum())))
        return out

    def _gather(self, mine):
        """All ranks' lists -> rank 0's list ordered by batch index (other ranks get None)."""
        if self.world == 1:
            return sorted(mine, key=lambda x: x[0])
        import torch
        got = [None] * self.world if self.rank == 0 else None
        torch.distributed.gather_object(mine, got, dst=0)
        return sorted((x for part in got for x in part), key=lambda x: x[0]) if self.rank == 0 else None

    def validate(self, step):
        """-> (record, stop).  record: {step, loss: {NLL, PPL}, metric: {...}, hypotheses} on rank 0, None elsewhere;
        stop: early stop, agreed by every rank."""
        import torch
        from neurst_b200 import cli
        torch.cuda.synchronize()
        vp, rt = self.vp, self.model.runtime
        rec = {"step": step, "elapsed": {}} if self.rank == 0 else None
        start = time.time()
        stop = False
        if vp["criterion"]:
            loss_batches = _batches(self.examples, vp["batch_size"])
            sums = self._gather(self._loss_sums([(i, g) for i, g in enumerate(loss_batches) if i % self.world == self.rank]))
            elapsed = time.time() - start
        if vp["criterion"] and self.rank == 0:
            tot = np.sum(np.array([s[1:] for s in sums], dtype=np.float64), axis=0)
            res = self.criterion_metric.reduce(*tot)
            self.loss_recorder.record(step, res)
            self._display(self.criterion_metric.flag, res, self.loss_recorder.best, step, elapsed)
            rec["loss"] = res
            rec["elapsed"]["loss"] = elapsed
        if self.gen_metric is not None:
            start = time.time()
            calls = _batches(self.examples, self.per_call)
            mine = [(i, cli.decode_group(self.model, self.task, self.gen_plan, g, self.search_kw))
                    for i, g in enumerate(calls) if i % self.world == self.rank]
            hyps = self._gather(mine)
            elapsed = time.time() - start
            if self.rank == 0:
                rec["elapsed"]["generation"] = elapsed
                start = time.time()
                hyps = [text for _, part in hyps for text, _ in part]
                res = self.gen_metric(hyps, self.references)
                names = None
                if self.gen_recorder.best_saver is not None:
                    from neurst_b200 import checkpoints as CK
                    names = CK.tf_variable_names(rt.table)

                def snapshot():
                    flat = rt.params.detach().cpu().numpy()
                    return {names[k]: flat[off:off + int(np.prod(shp))].reshape(shp) for k, (off, shp) in rt.table.items()}
                stop = self.gen_recorder.record(step, res, snapshot)
                self._display_hypo(hyps)
                self._display(self.gen_metric.flag, res, self.gen_recorder.best, step, elapsed)
                rec.update(metric=res, hypotheses=hyps)
                rec["elapsed"]["metric_and_checkpoints"] = time.time() - start
        if self.world > 1:
            flag = [stop]
            torch.distributed.broadcast_object_list(flag, src=0)
            stop = flag[0]
            torch.distributed.barrier()
        if rec is not None:
            rec["early_stop"] = stop
            self.history.append(rec)
        return rec, stop

    def _display(self, flag, res, best, step, elapsed):
        for k, v in res.items():
            LOG.info("Evaluating (%s) validation set: %s=%.2f (Best %.2f)  step=%d\tElapsed %.2fs  FromSTART %.2fs",
                     flag, k, v, best[k], step, elapsed, time.time() - self.t0)

    def _display_hypo(self, hyps):
        LOG.info("===== Generation examples (Total %d) =====", len(hyps))
        # a private generator: the training's random streams stay untouched
        for i in random.Random(len(hyps)).sample(range(len(hyps)), min(5, len(hyps))):
            LOG.info("Sample %d", i)
            LOG.info("  Reference: %s", self.references[i])
            LOG.info("  Hypothesis: %s", hyps[i])
