"""Device-side state of one model replica: the C handle, the flat parameter / gradient / Adam arenas, the
bf16 shadow and the workspace.  PyTorch supplies device memory and streams only; all compute is libb200st."""
import ctypes as C

import torch

from neurst_b200 import lib as L


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


# "mixed16" = the reference's mixed precision (fp16 compute + dynamic loss scaling, training_utils.py:73-81) = "fp16"
PRECISIONS = {"fp32": L.F32, "float32": L.F32, "bf16": L.BF16, "bfloat16": L.BF16, "fp16": L.F16, "float16": L.F16,
              "mixed16": L.F16, "mixed_float16": L.F16}
_TORCH16 = {L.BF16: torch.bfloat16, L.F16: torch.float16}


def make_config(model_type, d, heads, ffn=0, enc_layers=0, dec_layers=0, vocab=0, src_vocab=0, feat=80, in_channels=1,
                channels=0, conv_layer_norm=True, precision="bf16", ln_eps=1e-6, attention_dropout=0.0, ffn_dropout=0.0,
                postprocess_dropout=0.0, label_smoothing=0.0, share_src_trg_embedding=False, mha_self=False, mha_din=0,
                mha_dmem=0, mha_dout=0, with_cross_attention=True, disable_fused_attention=False, deterministic=False,
                encoder_monotonic=False):
    c = L.Config()
    c.model_type = model_type
    c.d, c.heads, c.ffn, c.enc_layers, c.dec_layers = d, heads, ffn, enc_layers, dec_layers
    c.vocab, c.src_vocab = vocab, src_vocab
    c.feat, c.in_channels, c.channels, c.conv_layer_norm = feat, in_channels, channels, int(conv_layer_norm)
    c.precision = PRECISIONS[precision]
    c.ln_eps = ln_eps
    c.attention_dropout, c.ffn_dropout, c.postprocess_dropout = attention_dropout, ffn_dropout, postprocess_dropout
    c.label_smoothing = label_smoothing
    c.share_src_trg_embedding = int(share_src_trg_embedding)
    c.mha_self, c.mha_din, c.mha_dmem, c.mha_dout = int(mha_self), mha_din, mha_dmem, mha_dout
    c.with_cross_attention = int(with_cross_attention)
    c.disable_fused_attention = int(disable_fused_attention)
    c.deterministic = int(deterministic)
    c.encoder_monotonic = int(encoder_monotonic)
    return c


class Runtime:
    """Owns the handle and the flat arenas of one replica on `device`."""

    def __init__(self, config, device="cuda"):
        self.lib = L.load()
        self.config = config
        self.device = torch.device(device)
        if self.device.type != "cuda" or not torch.cuda.is_available():
            raise L.B200STError("neurst_b200 runs on CUDA devices only (no CPU fallback): device=%s, CUDA available=%s" %
                                (self.device, torch.cuda.is_available()))
        h = C.c_void_p()
        L.check(self.lib.b200st_create(C.byref(config), C.byref(h)))
        self.handle = h
        self.prec = int(config.precision)
        self.bf16 = self.prec in _TORCH16          # (historic name) any 16-bit tensor-core precision
        self.fp16 = self.prec == L.F16
        self.numel = int(self.lib.b200st_param_arena_numel(h))
        self.table = {}
        name = C.create_string_buffer(128)
        off, nd, shp = C.c_int64(), C.c_int32(), (C.c_int64 * 4)()
        for i in range(int(self.lib.b200st_param_count(h))):
            L.check(self.lib.b200st_param_info(h, i, name, 128, C.byref(off), C.byref(nd), shp))
            self.table[name.value.decode()] = (int(off.value), tuple(int(shp[k]) for k in range(nd.value)))
        self.params = torch.zeros(self.numel, dtype=torch.float32, device=self.device)
        self.shadow = torch.zeros(self.numel, dtype=_TORCH16[self.prec], device=self.device) if self.bf16 else None
        # dynamic loss scale state of the fp16 precision (b200st_optimizer_step): scale starts at 2^15 like the reference
        # (training_utils.py:413-416); float[8] on the device so CUDA-graph replays follow it
        self.loss_scale_state = None
        self.tensor_sumsq = None
        if self.fp16:
            self.loss_scale_state = torch.zeros(8, dtype=torch.float32, device=self.device)
            self.loss_scale_state[0] = 2.0 ** 15
        self.grads = None
        self.adam_m = None
        self.adam_v = None
        self.workspace = None
        self._shadow_stale = True

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.b200st_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    # ---- parameters ------------------------------------------------------------------------------
    def view(self, name, arena=None):
        off, shp = self.table[name]
        n = 1
        for s in shp:
            n *= s
        a = self.params if arena is None else arena
        return a[off:off + n].view(*shp)

    def named_parameters(self):
        return {k: self.view(k) for k in self.table}

    def load_parameters(self, P):
        """P: dict name -> tensor/ndarray in the reference's TF layouts (oracle.param_shapes naming)."""
        for k in self.table:
            if k not in P:
                raise KeyError("missing parameter %s" % k)
            self.view(k).copy_(torch.as_tensor(P[k]).to(torch.float32).reshape(self.table[k][1]))
        self._shadow_stale = True

    def refresh_shadow(self):
        if self.bf16:
            L.check(self.lib.b200st_refresh_shadow(_ptr(self.params), _ptr(self.shadow), self.prec, self.numel, L._stream()))
        self._shadow_stale = False

    def ensure_grads(self):
        if self.grads is None:
            self.grads = torch.zeros(self.numel, dtype=torch.float32, device=self.device)
        return self.grads

    def grad_view(self, name):
        return self.view(name, self.ensure_grads())

    # ---- execution -------------------------------------------------------------------------------
    def _workspace(self, nbytes):
        if self.workspace is None or self.workspace.numel() < nbytes:
            self.workspace = None
            self.workspace = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=self.device)
        return self.workspace

    def _buffers(self, nbytes, with_grads, ws=None):
        """Buffers struct over the shared (grow-on-demand) workspace, or over a caller-owned tensor `ws` (CUDA-graph
        steps bake the pointer into the captured graph, so each owns its workspace for its whole life)."""
        if ws is None:
            ws = self._workspace(nbytes)
        base = ws.data_ptr()
        aligned = (base + 255) // 256 * 256
        b = L.Buffers()
        b.params = self.params.data_ptr()
        b.shadow = self.shadow.data_ptr() if self.bf16 else None
        b.grads = self.ensure_grads().data_ptr() if with_grads else None
        b.workspace = aligned
        b.workspace_bytes = ws.numel() - (aligned - base)
        return b

    # ---- data parallelism: NCCL communicator owned by the library (b200st_comm_*) ----------------------------------
    def comm_init(self, dist):
        """One communicator per replica: rank 0 creates the NCCL unique id, it travels over the existing process group
        (host channel only), every rank joins.  After this `run(..., allreduce=True)` / graph steps all-reduce the
        gradient arena inside the library, bucketed and overlapped with the backward pass."""
        world, rank = dist.get_world_size(), dist.get_rank()
        buf = C.create_string_buffer(128)
        if rank == 0:
            L.check(self.lib.b200st_comm_unique_id(buf))
        t = torch.tensor(list(buf.raw), dtype=torch.uint8, device=self.device if dist.get_backend() == "nccl" else "cpu")
        dist.broadcast(t, src=0)
        ident = bytes(t.cpu().tolist())
        L.check(self.lib.b200st_comm_init(self.handle, ident, world, rank))
        self.comm_world = world
        return self

    def comm_close(self):
        """Destroys the library's NCCL communicator (every rank, before torch.distributed.destroy_process_group)."""
        if getattr(self, "comm_world", 0):
            torch.cuda.synchronize(self.device)
            L.check(self.lib.b200st_comm_destroy(self.handle))
            self.comm_world = 0

    def comm_broadcast_parameters(self, root=0):
        L.check(self.lib.b200st_comm_broadcast(self.handle, _ptr(self.params), self.numel, int(root), L._stream()))
        self._shadow_stale = True

    def comm_stats(self):
        n, c, w = C.c_int64(0), C.c_int32(0), C.c_int32(0)
        L.check(self.lib.b200st_comm_stats(self.handle, C.byref(n), C.byref(c), C.byref(w)))
        return dict(reduced_elems=n.value, calls=c.value, world=w.value)

    def run(self, batch, backward):
        """batch: dict of CUDA tensors: src|src_ids, src_length|src_padding, trg_input[, trg, trg_length] (+ opts)."""
        if self._shadow_stale:
            self.refresh_shadow()
        bt = L.Batch()
        keep = []

        def put(field, t, dtype):
            if t is None:
                return
            t = t.to(device=self.device, dtype=dtype).contiguous()
            keep.append(t)
            setattr(bt, field, t.data_ptr())

        trg_input = batch["trg_input"]
        B, Lq = trg_input.shape
        if self.config.model_type == L.MODEL_SPEECH:
            src = batch["src"]
            T = src.shape[1]
            put("src", src, torch.float32)
            put("src_length", batch["src_length"], torch.int64)
        else:
            src = batch["src"]
            T = src.shape[1]
            put("src_ids", src, torch.int64)
            put("src_padding", batch["src_padding"], torch.float32)
        put("trg_input", trg_input, torch.int64)
        put("trg", batch.get("trg"), torch.int64)
        put("trg_length", batch.get("trg_length"), torch.int64)
        bt.B, bt.T, bt.L = B, T, Lq
        bt.training = int(batch.get("training", backward))
        bt.seed = int(batch.get("seed", 0))
        bt.loss_scale = float(batch.get("loss_scale", 1.0))
        bt.wait_k = int(batch.get("wait_k", 0))
        if backward and self.fp16 and batch.get("dynamic_loss_scale", True):
            bt.loss_scale_dev = self.loss_scale_state.data_ptr()       # gradients come out multiplied by state[0]
        out = {}
        V = self.config.vocab
        if batch.get("want_logits", not backward):
            out["logits"] = torch.empty(B, Lq, V, dtype=torch.float32, device=self.device)
            bt.logits = out["logits"].data_ptr()
        if batch.get("trg") is not None:
            out["loss"] = torch.zeros(1, dtype=torch.float32, device=self.device)
            out["nll_sum"] = torch.zeros(B, dtype=torch.float32, device=self.device)
            out["n_tokens"] = torch.zeros(B, dtype=torch.float32, device=self.device)
            bt.loss, bt.nll_sum, bt.n_tokens = out["loss"].data_ptr(), out["nll_sum"].data_ptr(), out["n_tokens"].data_ptr()
        if batch.get("want_enc_out", False):
            Ts = ((T + 1) // 2 + 1) // 2 if self.config.model_type == L.MODEL_SPEECH else T
            out["enc_out"] = torch.empty(B, Ts, self.config.d, dtype=torch.float32, device=self.device)
            bt.enc_out = out["enc_out"].data_ptr()
        need = int(self.lib.b200st_workspace_bytes(self.handle, B, T, Lq, int(backward)))
        if need <= 0:
            raise L.B200STError("workspace planning failed: " + self.lib.b200st_last_error().decode())
        bufs = self._buffers(need, backward)
        if backward and batch.get("allreduce", False):
            opts = L.StepOpts()
            opts.allreduce_grads = 1
            L.check(self.lib.b200st_train_step(self.handle, C.byref(bufs), C.byref(bt), C.byref(opts), L._stream()))
            return out
        fn = self.lib.b200st_forward_backward if backward else self.lib.b200st_forward
        L.check(fn(self.handle, C.byref(bufs), C.byref(bt), L._stream()))
        return out

    def adam_step(self, lr, step_t, beta1=0.9, beta2=0.98, eps=1e-9, grad_scale=1.0, zero_grad=True, clip_value=None,
                  clip_norm=None, dynamic_loss_scale=None, growth_steps=2000, multiplier=2.0, prune=None, frozen=None):
        """One optimizer step over the flat arenas (b200st_optimizer_step): unscale -> clip (per gradient tensor, as
        tf.clip_by_value / tf.clip_by_norm in gradaccum_keras_model.py:228-233) -> Keras Adam -> shadow refresh -> g = 0.
        fp16 precision: the gradients carry the dynamic loss scale; a step with non-finite gradients is skipped on the
        device (state in `self.loss_scale_state`).  `prune`: the schedule given to prune_setup(); the step is then
        b200st_optimizer_step_pruned (mask off-turn, selection and new mask on a turn).  `frozen`: the bitmap given to
        partial_setup(); the step is then b200st_optimizer_step_partial (the elements whose bit is 1 keep their weight)."""
        if prune is not None and frozen is not None:
            raise L.B200STError("adam_step takes a pruning schedule or a frozen-element bitmap, not both")
        if self.adam_m is None:
            self.adam_m = torch.zeros_like(self.params)
            self.adam_v = torch.zeros_like(self.params)
        dyn = self.fp16 if dynamic_loss_scale is None else bool(dynamic_loss_scale)
        a = L.OptimArgs()
        a.params, a.grads = self.params.data_ptr(), self.ensure_grads().data_ptr()
        a.m, a.v = self.adam_m.data_ptr(), self.adam_v.data_ptr()
        a.shadow = self.shadow.data_ptr() if self.bf16 else None
        a.shadow_dtype = self.prec if self.bf16 else L.BF16
        a.numel = self.numel
        a.lr, a.beta1, a.beta2, a.eps = lr, beta1, beta2, eps
        a.step_t, a.grad_scale, a.zero_grad = int(step_t), grad_scale, int(zero_grad)
        a.clip_value = abs(float(clip_value or 0.0))      # GradAccumKerasModel takes abs(clip_value)
        a.clip_norm = float(clip_norm or 0.0)
        if dyn or a.clip_norm > 0:
            if self.tensor_sumsq is None:
                self.tensor_sumsq = torch.zeros(len(self.table) + 1, dtype=torch.float32, device=self.device)
            a.tensor_sumsq = self.tensor_sumsq.data_ptr()
        if dyn:
            if self.loss_scale_state is None:
                self.loss_scale_state = torch.zeros(8, dtype=torch.float32, device=self.device)
                self.loss_scale_state[0] = 1.0
            a.loss_scale_state = self.loss_scale_state.data_ptr()
            a.growth_steps, a.multiplier = float(growth_steps), float(multiplier)
        if prune is not None:
            L.check(self.lib.b200st_optimizer_step_pruned(self.handle, C.byref(a), C.byref(self._prune_args(prune)), L._stream()))
        elif frozen is not None:
            if getattr(self, "partial_frozen", None) is not frozen:
                raise L.B200STError("adam_step(frozen=...) needs partial_setup() with that bitmap first")
            L.check(self.lib.b200st_optimizer_step_partial(self.handle, C.byref(a), _ptr(frozen), L._stream()))
        else:
            L.check(self.lib.b200st_optimizer_step(self.handle, C.byref(a), L._stream()))
        self._shadow_stale = False

    # ---- weight pruning (b200st_optimizer_step_pruned) -----------------------------------------------------------------
    def prune_setup(self, schedule, names):
        """Pruning of the parameters `names` under `schedule` (neurst_b200.pruning) for the steps that follow: a fresh device
        state (the schedule's step restarts at 0, as the reference's optimizer iterations do in a new run) and the mask
        derived from the weights now in the arena (weight != 0, keep_prune_property=True): masks are not checkpointed, so
        a resumed or pretrained run finds its pruned weights as zeros."""
        from neurst_b200 import pruning as PR
        if not names:
            raise L.B200STError("pruning selects no parameter tensor")
        if len(names) > L.PRUNE_MAX_TENSORS:
            raise L.B200STError("pruning takes at most %d tensors, got %d" % (L.PRUNE_MAX_TENSORS, len(names)))
        if self.numel % 8:
            raise L.B200STError("pruning needs an arena padded to a multiple of 8 elements")
        index = {k: i for i, k in enumerate(self.table)}
        smax = schedule.max_sparsity()
        for k in names:
            size = self._numel_of(k)
            if PR.k_of(size, smax) < 1:
                raise L.B200STError("pruning %s (%d elements) at sparsity %g keeps no weight (k = 0): lower the sparsity or leave "
                                    "the tensor out" % (k, size, float(smax)))
        self.prune_names = list(names)
        self.prune_schedule = schedule
        self.prune_ids = (C.c_int32 * len(names))(*[index[k] for k in names])
        self.prune_state = torch.zeros(4, dtype=torch.int32, device=self.device)
        self.prune_thresholds = torch.zeros(len(names), dtype=torch.float32, device=self.device)
        nbytes = int(self.lib.b200st_prune_scratch_bytes(len(names)))
        self.prune_scratch = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        self.prune_mask = self.derive_prune_mask()
        return self

    def _numel_of(self, name):
        n = 1
        for s in self.table[name][1]:
            n *= s
        return n

    def derive_prune_mask(self, names=None, source=None):
        """Mask bitmap of the tensors `names` (the pruned set when None) from the current weights: bit j of byte b keeps
        element 8b + j; 1 outside those tensors (and in the alignment padding after each), weight != 0 inside them.  With
        `source` ({name: array in the tensor's shape}, e.g. the masks of a mask file) the bits are source != 0 instead.
        Built tensor by tensor in uint8, so the temporaries are the size of the largest tensor's slot."""
        mask = torch.full((self.numel // 8,), 0xFF, dtype=torch.uint8, device=self.device)
        for k in (self.prune_names if names is None else names):
            off, _ = self.table[k]
            n = self._numel_of(k)
            n8 = (n + 7) // 8 * 8                        # the tensor's slot in the arena
            if source is None:
                nz = (self.params[off:off + n8] != 0).view(-1, 8)
            else:
                nz = torch.empty(n8, dtype=torch.bool, device=self.device)
                nz[:n] = torch.as_tensor(source[k]).to(self.device).reshape(-1) != 0
                nz = nz.view(-1, 8)
            if n8 > n:
                nz[-1, n - n8 + 8:] = True
            byte = torch.zeros(n8 // 8, dtype=torch.uint8, device=self.device)
            for j in range(8):
                byte |= nz[:, j].to(torch.uint8) << j
            mask[off // 8:(off + n8) // 8] = byte
        return mask

    def _prune_args(self, prune):
        from neurst_b200 import pruning as PR
        if getattr(self, "prune_schedule", None) is not prune:
            raise L.B200STError("adam_step(prune=...) needs prune_setup() with that schedule first")
        sc = prune
        p = L.PruneArgs()
        p.mask = self.prune_mask.data_ptr()
        p.tensor_ids = self.prune_ids
        p.n_tensors = len(self.prune_names)
        poly = isinstance(sc, PR.PolynomialDecay)
        p.schedule = L.PRUNE_POLYNOMIAL if poly else L.PRUNE_CONSTANT
        p.initial_sparsity = sc.initial_sparsity if poly else 0.0
        p.target_sparsity = sc.target_sparsity
        p.polynomial_power = sc.polynomial_power if poly else 0.0
        p.begin_step, p.end_step, p.frequency = sc.begin_pruning_step, sc.end_pruning_step, sc.pruning_frequency
        p.state = self.prune_state.data_ptr()
        p.thresholds = self.prune_thresholds.data_ptr()
        p.scratch = self.prune_scratch.data_ptr()
        return p

    def prune_sparsity(self):
        """(zeros, elements) over the pruned tensors: a host reduction, for a point that is already synchronised."""
        zeros = total = 0
        for k in self.prune_names:
            v = self.view(k)
            zeros += int((v == 0).sum())
            total += v.numel()
        return zeros, total

    # ---- partial tuning of a pruned model (b200st_optimizer_step_partial, b200st_apply_mask) ---------------------------
    def partial_setup(self, mask_bitmap):
        """Partial tuning for the steps that follow (adam_step(frozen=self.partial_frozen)): `mask_bitmap` (device uint8
        [numel / 8], derive_prune_mask's layout over every tensor) holds 1 where the weight stays frozen, 0 where it is
        tuned.  -> (tuned, frozen) element counts over the parameter tensors."""
        if self.numel % 8:
            raise L.B200STError("partial tuning needs an arena padded to a multiple of 8 elements")
        m = mask_bitmap
        if not (torch.is_tensor(m) and m.dtype == torch.uint8 and m.device == self.params.device and m.is_contiguous()
                and m.numel() == self.numel // 8):
            raise L.B200STError("partial_setup needs a contiguous uint8 bitmap of %d bytes on %s" % (self.numel // 8, self.device))
        self.partial_frozen = m
        return self.mask_counts(m)

    def mask_counts(self, bitmap):
        """(bits 0, bits 1) over the elements of the parameter tensors of a derive_prune_mask bitmap over every tensor (whose
        bits outside the tensors are 1)."""
        popcount = torch.tensor([bin(i).count("1") for i in range(256)], dtype=torch.int64, device=self.device)
        ones = int(popcount[bitmap.long()].sum())
        elements = sum(self._numel_of(k) for k in self.table)
        frozen = ones - (self.numel - elements)
        return elements - frozen, frozen

    def apply_mask(self, keep):
        """The weights whose bit of `keep` (derive_prune_mask's layout) is 0 -> 0, in the master arena and in the 16-bit
        shadow (b200st_apply_mask)."""
        if not (torch.is_tensor(keep) and keep.dtype == torch.uint8 and keep.numel() == self.numel // 8):
            raise L.B200STError("apply_mask needs a uint8 bitmap of %d bytes" % (self.numel // 8))
        L.check(self.lib.b200st_apply_mask(_ptr(self.params), _ptr(self.shadow), self.prec if self.bf16 else L.BF16, _ptr(keep),
                                           self.numel, L._stream()))

    def dropout_mask(self, site, n, p, seed):
        sid = int(self.lib.b200st_dropout_stream_id(site.encode()))
        out = torch.empty(n, dtype=torch.uint8, device=self.device)
        L.check(self.lib.b200st_dropout_mask(int(seed), sid, n, float(p), _ptr(out), L._stream()))
        return out.bool()


class GraphedTrainStep:
    """CUDA-graph capture of one forward+backward call (b200st_forward_backward) at a fixed (B, T, L).

    All launches of the step (~1800 kernels) are replayed from one graph; inputs live in static device buffers that
    `__call__` refreshes, and the dropout seed is read by the kernels from a device word (`seed_dev`), so every replay
    draws fresh masks.  The wait-k lag of a wait-k model's cross-attention (`wait_k=True`) is a device word too (`wait_k_dev`), so a
    multi-path model draws a fresh k per step and replays the same graph; other models capture no lag at all.  Gradients accumulate into the runtime's gradient arena exactly as in the eager path."""

    def __init__(self, rt, B, T, Lq, allreduce=False, wait_k=False):
        self.allreduce = bool(allreduce)
        cfg = rt.config
        if cfg.model_type not in (L.MODEL_SPEECH, L.MODEL_TEXT):
            raise L.B200STError("GraphedTrainStep supports the SpeechTransformer and text Transformer handles")
        self.rt, self.B, self.T, self.L = rt, B, T, Lq
        self.text = cfg.model_type == L.MODEL_TEXT
        dev = rt.device
        if self.text:            # source ids and their padding (1.0 beyond the source length)
            self.src = torch.zeros(B, T, dtype=torch.int64, device=dev)
            self.src_padding = torch.zeros(B, T, dtype=torch.float32, device=dev)
        else:
            self.src = torch.zeros(B, T, cfg.feat, cfg.in_channels, dtype=torch.float32, device=dev)
            self.src_length = torch.zeros(B, dtype=torch.int64, device=dev)
        self.trg_input = torch.zeros(B, Lq, dtype=torch.int64, device=dev)
        self.trg = torch.zeros(B, Lq, dtype=torch.int64, device=dev)
        self.trg_length = torch.ones(B, dtype=torch.int64, device=dev)
        self.seed = torch.zeros(1, dtype=torch.int64, device=dev)
        self.wait_k = torch.zeros(1, dtype=torch.int32, device=dev) if wait_k else None
        self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
        self.nll_sum = torch.zeros(B, dtype=torch.float32, device=dev)
        self.n_tokens = torch.zeros(B, dtype=torch.float32, device=dev)
        need = int(rt.lib.b200st_workspace_bytes(rt.handle, B, T, Lq, 1))
        if need <= 0:
            raise L.B200STError("workspace planning failed: " + rt.lib.b200st_last_error().decode())
        # the captured graph holds raw pointers into this tensor: owned here, never the runtime's growable workspace
        self.workspace = torch.empty(need + 256, dtype=torch.uint8, device=dev)
        self.bufs = rt._buffers(need, True, ws=self.workspace)
        bt = L.Batch()
        if self.text:
            bt.src_ids, bt.src_padding = self.src.data_ptr(), self.src_padding.data_ptr()
        else:
            bt.src, bt.src_length = self.src.data_ptr(), self.src_length.data_ptr()
        bt.trg_input, bt.trg, bt.trg_length = self.trg_input.data_ptr(), self.trg.data_ptr(), self.trg_length.data_ptr()
        bt.B, bt.T, bt.L, bt.training = B, T, Lq, 1
        bt.seed, bt.seed_dev, bt.loss_scale = 0, self.seed.data_ptr(), 1.0
        if wait_k:
            bt.wait_k_dev = self.wait_k.data_ptr()
        if rt.fp16:
            bt.loss_scale_dev = rt.loss_scale_state.data_ptr()
        bt.loss, bt.nll_sum, bt.n_tokens = self.loss.data_ptr(), self.nll_sum.data_ptr(), self.n_tokens.data_ptr()
        self.bt = bt
        self.graph = None

    def _launch(self):
        if self.allreduce:      # the NCCL all-reduces on the library's communication stream become branches of the graph
            opts = L.StepOpts()
            opts.allreduce_grads = 1
            L.check(self.rt.lib.b200st_train_step(self.rt.handle, C.byref(self.bufs), C.byref(self.bt), C.byref(opts), L._stream()))
            return
        L.check(self.rt.lib.b200st_forward_backward(self.rt.handle, C.byref(self.bufs), C.byref(self.bt), L._stream()))

    def capture(self):
        rt = self.rt
        if rt._shadow_stale:
            rt.refresh_shadow()
        saved = rt.ensure_grads().clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):          # warm-up outside capture (function attributes, tensor-map cache)
            self._launch()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        # thread-local capture mode.  Observed in global mode: the Prefetcher thread of the training entry pins its next batch
        # (Tensor.pin_memory -> cudaHostAlloc) while this thread captures, which invalidates the capture
        # (cudaErrorStreamCaptureInvalidated at capture_end, and torch's graph state stays broken for later captures).
        # The captured region itself issues kernel launches only, so nothing this thread does needs the global check.
        with torch.cuda.graph(g, capture_error_mode="thread_local"):
            self._launch()
        rt.grads.copy_(saved)                  # discard the warm-up / capture-time accumulation
        self.graph = g
        return self

    def __call__(self, batch, seed, wait_k=0):
        if self.graph is None:
            self.capture()
        if self.rt._shadow_stale:
            self.rt.refresh_shadow()
        self.src.copy_(batch["src"], non_blocking=True)
        if self.text:
            self.src_padding.copy_(batch["src_padding"], non_blocking=True)
        else:
            self.src_length.copy_(batch["src_length"], non_blocking=True)
        self.trg_input.copy_(batch["trg_input"], non_blocking=True)
        self.trg.copy_(batch["trg"], non_blocking=True)
        self.trg_length.copy_(batch["trg_length"], non_blocking=True)
        self.seed.fill_(int(seed))
        if self.wait_k is not None:
            self.wait_k.fill_(int(wait_k))
        elif wait_k:
            raise L.B200STError("this GraphedTrainStep was captured without a wait-k lag (wait_k=False)")
        self.graph.replay()
        # fresh tensors, as the eager path returns: the persistent outputs are overwritten by the next replay
        return {"loss": self.loss.clone(), "nll_sum": self.nll_sum.clone(), "n_tokens": self.n_tokens.clone()}
