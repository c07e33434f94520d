"""Data-parallel training step loop (one process per GPU, NCCL over NVLink only).

Replaces, for the SpeechTransformer hot path, the reference's
  GradAccumKerasModel.train_step / fit loop      neurst/training/gradaccum_keras_model.py:162-260,441-477
  gradient aggregation                           neurst/training/hvd_utils.py:48-62 (hvd.Average),
                                                 neurst/training/distribution_utils.py:73-98 (NcclAllReduce)
  rank-0 weight broadcast                        neurst/exps/trainer.py:285
  Adam + noam schedule                           neurst/optimizers/__init__.py:21, schedules/noam_schedule.py:75-97
  throughput accounting                          neurst/training/callbacks.py:209-238 (src_tokens_per_sec = frames/s)

Semantics kept: each replica normalises its loss by ITS OWN token count (label_smoothed_cross_entropy.py:52-53), the
gradients are averaged over replicas, every replica applies the identical Adam update.
"""
import os
import time

import torch

from neurst_b200.models import SpeechTransformer, speech_transformer_hparams


def noam_learning_rate(step, dmodel, warmup_steps=4000, initial_factor=1.0, end_factor=None, start_decay_at=0,
                       decay_steps=None):
    """neurst/optimizers/schedules/noam_schedule.py:75-97 (global_step counted from 0)."""
    gs = float(step) + 1.0
    if end_factor is None or start_decay_at is None or decay_steps is None:
        end_factor, start_decay_at, decay_steps = initial_factor, 0, 1
    step_factor = max(min(gs - start_decay_at, float(decay_steps)), 0.0)
    lr = end_factor + (initial_factor - end_factor) * (1.0 - step_factor / float(decay_steps))
    lr *= dmodel ** -0.5
    lr *= min(1.0, gs / float(warmup_steps))
    lr /= max(gs, float(warmup_steps)) ** 0.5
    return lr


def allreduce_sum_(flat, dist, buckets=1):
    """In-place SUM all-reduce of the flat gradient arena (NCCL on GPUs; the mean's 1/world is folded into the Adam
    kernel's grad_scale).  `buckets` > 1 splits the arena into contiguous chunks (launch-latency / overlap knob)."""
    if buckets <= 1:
        dist.all_reduce(flat)
        return
    n = flat.numel()
    step = (n + buckets - 1) // buckets
    for i in range(0, n, step):
        dist.all_reduce(flat[i:i + step])


class DataParallelTrainer:
    """One replica of the DP job.  `dist` (torch.distributed, NCCL) is used only for the gradient all-reduce, the
    initial parameter broadcast and scalar metric reduction."""

    def __init__(self, model, optimizer_params=None, lr_schedule_params=None, update_cycle=1, grad_buckets=1,
                 use_cuda_graph=False, clip_value=None, clip_norm=None, summary_steps=0, logger=None, pruning_schedule=None,
                 pruning_variables=None, partial_tuning_mask=None):
        """`pruning_schedule` (neurst_b200.pruning, or None): prune the parameters `pruning_variables` (our names; all of them
        when None) during training, as the reference's pruning optimizer does; a schedule with target_sparsity 0 prunes nothing.  The mask is derived from the weights at the
        first update, after the rank-0 broadcast.
        `partial_tuning_mask` (Prune-Tune's partial tuning, or None): "weights" freezes every weight that is not zero, a
        {our name: 0/1 array} (neurst_b200.prune_tune.load_masks) every element whose mask is 1; only the others are tuned.
        Like the pruning mask it is set up after the rank-0 broadcast (setup_partial_tuning, at the latest at the first
        update), so every rank freezes the same elements.  It cannot be combined with a pruning schedule."""
        self.model = model
        self.rt = model.runtime
        op = optimizer_params or {}
        self.beta1, self.beta2, self.eps = op.get("beta_1", 0.9), op.get("beta_2", 0.98), op.get("epsilon", 1e-9)
        self.lr_params = lr_schedule_params or dict(dmodel=model.runtime.config.d, warmup_steps=4000, initial_factor=1.0)
        self.update_cycle = int(update_cycle)
        self.global_step = 0
        # the global step at which the optimizer's iterations (Adam's t) count from 0: a run started at initial_global_step
        # sets it, as the reference's optimizer starts its own iterations at 0 whatever the registered initial step
        self.adam_step_base = 0
        self._micro = 0
        self.dist = torch.distributed if torch.distributed.is_available() and torch.distributed.is_initialized() else None
        self.world = self.dist.get_world_size() if self.dist else 1
        self.rank = self.dist.get_rank() if self.dist else 0
        self.rt.ensure_grads().zero_()
        self.grad_buckets = max(1, int(grad_buckets))
        self.use_cuda_graph = bool(use_cuda_graph)
        self._graphs = {}
        # gradient clipping of the reference's step (exps/trainer.py:74-75,130-131 -> gradaccum_keras_model.py:228-233)
        self.clip_value, self.clip_norm = clip_value, clip_norm
        # NCCL inside the library when the job runs on GPUs (one communicator per replica); torch.distributed stays the
        # transport only for the gloo / CPU stand-in used by the host-logic tests
        self.lib_comm = bool(self.dist and hasattr(self.rt, "comm_init") and self.dist.get_backend() == "nccl")
        if self.lib_comm:
            self.rt.comm_init(self.dist)
        self.meter = ThroughputMeter(summary_steps, self.world, logger) if summary_steps else None
        # target_sparsity 0 is no pruning (PruningSchedule.new returns None): the plain optimizer step
        self.pruning_schedule = pruning_schedule if pruning_schedule is not None and pruning_schedule.target_sparsity > 0 else None
        self.pruning_variables = None if pruning_variables is None else list(pruning_variables)
        self._pruning_ready = False
        if partial_tuning_mask is not None and not (isinstance(partial_tuning_mask, dict) or partial_tuning_mask == "weights"):
            raise ValueError("partial_tuning_mask is \"weights\" or a {name: 0/1 array} mapping, got %r" % type(partial_tuning_mask))
        if partial_tuning_mask is not None and self.pruning_schedule is not None:
            # the recipe prunes first and tunes afterwards; together, the pruning would re-mask the tuned positions
            raise ValueError("partial tuning cannot be combined with a pruning schedule")
        self.partial_tuning_mask = partial_tuning_mask
        self.partial_counts = None

    def close(self):
        """Collective-ordered shutdown of the in-library communicator (call on every rank before leaving the job)."""
        if self.lib_comm:
            # ncclCommDestroy waits until every CUDA graph that captured one of the communicator's collectives has been
            # destroyed (NCCL keeps a persistent reference per capture): drop the captured steps first
            self._graphs.clear()
            import gc
            gc.collect()
            torch.cuda.synchronize(self.rt.device)
            if self.dist:
                self.dist.barrier()
            self.rt.comm_close()
            self.lib_comm = False

    def broadcast_parameters(self):
        """rank 0 -> all (hvd BroadcastGlobalVariablesCallback, exps/trainer.py:285)."""
        if self.lib_comm:
            self.rt.comm_broadcast_parameters(0)
        elif self.dist:
            self.dist.broadcast(self.rt.params, src=0)
            self.rt._shadow_stale = True

    def setup_partial_tuning(self):
        """Builds the frozen-element bitmap from the current weights or the given masks (once) -> (tuned, frozen) element
        counts, or None without partial tuning.  Call it after broadcast_parameters."""
        if self.partial_tuning_mask is None:
            return None
        if self.partial_counts is None:
            source = None if isinstance(self.partial_tuning_mask, str) else self.partial_tuning_mask
            self.partial_counts = self.rt.partial_setup(self.rt.derive_prune_mask(list(self.rt.table), source))
        return self.partial_counts

    def _allreduce_grads(self):
        if self.dist and not self.lib_comm:        # lib_comm: already reduced inside b200st_train_step, overlapped
            allreduce_sum_(self.rt.grads, self.dist, self.grad_buckets)

    def train_step(self, inputs, seed=None):
        """fwd + bwd (+ all-reduce + Adam every `update_cycle` micro-batches).  Returns the device loss tensor."""
        b = dict(inputs)
        if seed is not None:
            # independent dropout draws per replica (the reference's replicas seed their own RNG streams)
            b["seed"] = int(seed) * self.world + self.rank
        last_micro = (self._micro + 1) % self.update_cycle == 0
        sync_now = self.lib_comm and last_micro          # gradients are all-reduced by the step that completes a cycle
        waitk = getattr(self.model, "wait_k", None) is not None
        if waitk:
            b["wait_k"] = self.model.lag(True)           # the wait-k model's lag of this micro-batch (one draw per call)
        if self.use_cuda_graph:
            from neurst_b200.runtime import GraphedTrainStep
            key = (b["src"].shape[0], b["src"].shape[1], b["trg_input"].shape[1], sync_now)   # one graph per shape bucket
            if key not in self._graphs:
                self._graphs[key] = GraphedTrainStep(self.rt, *key[:3], allreduce=sync_now, wait_k=waitk).capture()
            self._seed_ctr = getattr(self, "_seed_ctr", 0) + 1
            out = self._graphs[key](b, b.get("seed", self._seed_ctr * self.world + self.rank), wait_k=b.get("wait_k", 0))
        else:
            if sync_now:
                b["allreduce"] = True
            out = self.model.forward_backward(b, is_training=True, loss_scale=1.0)
        if self.meter is not None:
            self.meter.add(inputs)
        self._micro += 1
        if self._micro % self.update_cycle == 0:
            self._allreduce_grads()
            lr = noam_learning_rate(self.global_step, **self.lr_params)
            self.global_step += 1
            # GradientAccumulator averages over update_cycle (gradaccum_keras_model.py:62-109); hvd.Average over ranks
            scale = 1.0 / (self.world * self.update_cycle)
            kw = {}
            if self.clip_value or self.clip_norm:
                kw = dict(clip_value=self.clip_value, clip_norm=self.clip_norm)
            if self.pruning_schedule is not None:
                if not self._pruning_ready:
                    names = list(self.rt.table) if self.pruning_variables is None else self.pruning_variables
                    self.rt.prune_setup(self.pruning_schedule, names)
                    self._pruning_ready = True
                kw["prune"] = self.pruning_schedule
            if self.partial_tuning_mask is not None:
                self.setup_partial_tuning()
                kw["frozen"] = self.rt.partial_frozen
            self.rt.adam_step(lr, self.global_step - self.adam_step_base, self.beta1, self.beta2, self.eps, grad_scale=scale, zero_grad=True, **kw)
            if self.meter is not None:
                self.meter.step_end(self.global_step, out["loss"], lr)
        return out["loss"]


class ThroughputMeter:
    """MetricReductionCallback's speed lines (neurst/training/callbacks.py:209-245): every `summary_steps` updates log
    'Update N TrainingLoss=... Speed x secs/step y steps/sec' and a dict with, for every SUM metric of the task
    (src_tokens = input frames, src_real_tokens = sum(src_length), trg_tokens, trg_real_tokens, samples —
    neurst/layers/metric_layers/token_metric_layers.py:59-65), `<metric>_per_step` and `<metric>_per_sec` scaled by the number
    of replicas."""

    def __init__(self, summary_steps, world=1, logger=None):
        import logging
        self.n, self.world = max(1, int(summary_steps)), world
        self.log = logger or logging.getLogger("neurst_b200").info
        self.acc = {}
        self.t0 = time.time()
        self.last = None

    def add(self, inputs):
        src, trg = inputs["src"], inputs["trg_input"]
        m = {"src_tokens": src.shape[0] * src.shape[1], "trg_tokens": trg.shape[0] * trg.shape[1], "samples": src.shape[0]}
        if "src_length" in inputs:
            m["src_real_tokens"] = inputs["src_length"]
        if "trg_length" in inputs:
            m["trg_real_tokens"] = inputs["trg_length"]
        for k, v in m.items():
            self.acc.setdefault(k, []).append(v)

    def step_end(self, step, loss, lr):
        if step % self.n != 0:
            return None
        dt = max(time.time() - self.t0, 1e-9)
        tot = {k: float(sum(float(x.sum()) if torch.is_tensor(x) else x for x in v)) * self.world for k, v in self.acc.items()}
        self.log("Update %d\tTrainingLoss=%.2f\tSpeed %.3f secs/step %.1f steps/sec" % (step, float(loss), dt / self.n, self.n / dt))
        line = {"step": step, "lr": lr}
        for k, v in tot.items():
            line[k + "_per_step"] = v / self.n
            line[k + "_per_sec"] = v / dt
        self.log(str(line))
        self.acc, self.t0, self.last = {}, time.time(), line
        return line


class HostPipeline:
    """Pipelined host loop around `DataParallelTrainer.train_step` — the role of `tf.data` prefetching plus Keras' async
    metric reads in the reference's fit loop (neurst/exps/trainer.py:258-310, training/callbacks.py:209-238).

    Every step still copies its own inputs host->device (from pinned memory) and reads its own loss device->host; the
    copies of step i+1 run on a copy stream under the kernels of step i, and the loss of step i is read while step i+1
    runs, so neither serialises with the GPU work."""

    def __init__(self, trainer):
        self.tr = trainer
        self.dev = trainer.rt.device
        self.copy_stream = torch.cuda.Stream(device=self.dev)
        self.staging = [None, None]                  # device copies of the host batches (double buffer)
        self.ready = [torch.cuda.Event(), torch.cuda.Event()]     # H2D of slot finished
        self.consumed = [torch.cuda.Event(), torch.cuda.Event()]  # compute stream no longer reads slot
        self.loss_host = torch.zeros(2, dtype=torch.float32).pin_memory()
        self.loss_ready = [torch.cuda.Event(), torch.cuda.Event()]
        self.h2d_bytes = 0

    def _upload(self, slot, hb):
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self.consumed[slot])
            st = self.staging[slot]
            if st is None or any(st[k].shape != v.shape for k, v in hb.items()):
                st = self.staging[slot] = {k: torch.empty(v.shape, dtype=v.dtype, device=self.dev) for k, v in hb.items()}
            for k, v in hb.items():
                st[k].copy_(v, non_blocking=True)
            self.ready[slot].record(self.copy_stream)
        self.h2d_bytes = sum(v.numel() * v.element_size() for v in hb.values())

    def run(self, host_batches, seed0=1):
        """Generator over an iterable of pinned host batches: yields the float loss of every step, one step late (the
        first `next()` yields None, `close()`/exhaustion is preceded by the last loss)."""
        it = iter(host_batches)
        cur = torch.cuda.current_stream(self.dev)
        for s in range(2):
            self.consumed[s].record(cur)
        nxt = next(it, None)
        if nxt is None:
            return
        self._upload(0, nxt)
        i = 0
        while nxt is not None:
            slot = i & 1
            nxt = next(it, None)
            if nxt is not None:
                self._upload(slot ^ 1, nxt)                       # H2D of step i+1 under the kernels of step i
            cur.wait_event(self.ready[slot])
            loss = self.tr.train_step(self.staging[slot], seed=seed0 + i)
            self.consumed[slot].record(cur)
            self.loss_host[slot:slot + 1].copy_(loss.reshape(1), non_blocking=True)   # D2H of this step's loss
            self.loss_ready[slot].record(cur)
            self._latest = slot
            prev = None
            if i > 0:
                self.loss_ready[slot ^ 1].synchronize()
                prev = float(self.loss_host[slot ^ 1])
            yield prev
            i += 1
        yield self.latest_loss()

    def latest_loss(self):
        """The loss of the newest step `run` launched, which its generator yields only on the next resume: for a caller
        that stops iterating early."""
        self.loss_ready[self._latest].synchronize()
        return float(self.loss_host[self._latest])


def build_speech_transformer_trainer(hparams_set="speech_transformer_s", vocab_size=8192, feature_dim=80, precision="bf16",
                                     label_smoothing=0.1, dropout=None, seed=1234, update_cycle=1, device=None, use_cuda_graph=False):
    hp = speech_transformer_hparams(hparams_set)
    args = dict(hp["model.params"])
    if dropout is not None:
        for side in ("encoder", "decoder"):
            for k in ("attention_dropout_rate", "ffn_dropout_rate", "layer_postprocess_dropout_rate"):
                args["%s.%s" % (side, k)] = dropout
    src_meta = {"audio_feature_dim": feature_dim, "audio_feature_channels": 1}
    trg_meta = {"vocab_size": vocab_size, "eos_id": vocab_size - 1, "bos_id": vocab_size - 2, "unk_id": vocab_size - 3,
                "pad_id": vocab_size - 1}
    model = SpeechTransformer.new(args, src_meta, trg_meta, precision=precision, label_smoothing=label_smoothing,
                                  device=device or "cuda")
    model.init_parameters(seed)
    tr = DataParallelTrainer(model, hp["optimizer.params"], hp["lr_schedule.params"], update_cycle=update_cycle,
                             use_cuda_graph=use_cuda_graph)
    tr.broadcast_parameters()
    return tr, trg_meta


def synthetic_batch(B, T, Lq, vocab_size, feature_dim=80, seed=1234, lengths="full", device="cpu", pin=False):
    """SURVEY.md §8(d): src ~ N(0,1) (utterance-standardised fbank), zero beyond src_length; trg ~ U{4..V-1} ending in
    EOS then PAD; trg_input = [BOS, trg[:-1]] (neurst/tasks/speech2text.py:149-160)."""
    g = torch.Generator().manual_seed(seed)
    src = torch.randn(B, T, feature_dim, 1, generator=g)
    if lengths == "full":
        src_length = torch.full((B,), T, dtype=torch.long)
    else:
        src_length = (torch.rand(B, generator=g) * 0.4 * T + 0.6 * T).long().clamp(1, T)
        for i in range(B):
            src[i, int(src_length[i]):] = 0.0
    eos, bos = vocab_size - 1, vocab_size - 2
    trg = torch.randint(4, vocab_size - 2, (B, Lq), generator=g)
    trg_length = torch.full((B,), Lq, dtype=torch.long) if lengths == "full" else \
        (torch.rand(B, generator=g) * 0.4 * Lq + 0.6 * Lq).long().clamp(2, Lq)
    for i in range(B):
        n = int(trg_length[i])
        trg[i, n - 1] = eos
        trg[i, n:] = eos
    trg_input = torch.cat([torch.full((B, 1), bos, dtype=torch.long), trg[:, :-1]], dim=1)
    batch = dict(src=src, src_length=src_length, trg=trg, trg_input=trg_input, trg_length=trg_length)
    if pin:
        batch = {k: v.pin_memory() for k, v in batch.items()}
    if device != "cpu":
        batch = {k: v.to(device, non_blocking=True) for k, v in batch.items()}
    return batch
