"""Input-pipeline edge of the speech-to-text task (SURVEY.md 8 f4): frame-budget length bucketing and SpecAugment; and of
the seq2seq (text) task: vocabulary encoding of BPE'd text and token-budget bucketing.

  create_audio_bucket_boundaries / bucket table   neurst/tasks/speech2text.py:38-56,296-384
  SpecAugment                                      neurst/utils/audio_lib.py:24-257 (time warping is a documented no-op there too)
  Seq2Seq / token buckets                          neurst/tasks/seq2seq.py:100-270, neurst/data/dataset_utils.py:125-178,435-560

Bucketing is host logic (which utterance goes into which padded batch); SpecAugment runs on the GPU on the padded batch
(the masks are sampled on the host exactly as `freq_or_time_masking_numpy`, the fill is one masked-select on the device),
so that augmentation does not sit on the critical path of the HostPipeline copy stream.
"""
import math

import torch


def minimal_multiple(val, factor):
    """neurst/training/training_utils.py `minimal_multiple`."""
    return int(math.ceil(val / float(factor)) * factor)


def create_audio_bucket_boundaries(maxlen, minlen=128):
    """Restates neurst/tasks/speech2text.py:38-56 (geometric-ish growth of the bucket width)."""
    if minlen is None:
        minlen = 128
    bounds = [minlen]
    base = minlen
    base_incr = int(2 ** ((math.log2(minlen) + 1) // 2))
    base_incr_mult = 1
    times = len(str(int(minlen)))
    while True:
        for _ in range(times):
            bounds.append(bounds[-1] + base)
            if bounds[-1] > maxlen:
                break
        base += base_incr * base_incr_mult
        base_incr_mult += 1
        if bounds[-1] > maxlen:
            break
    bounds[-1] = maxlen + 1
    return bounds


class FrameBudgetBucketer:
    """The (T bucket -> batch size, transcript bound) table of SpeechToText.create_and_batch_tfds (speech2text.py:296-330):
    batch size per GPU = frame budget // bucket bound, rounded up to a multiple of 8 unless `disable_batch_efficiency`;
    transcript bound from `experimental_frame_transcript_ratio`, multiple of 8.  Every replica takes the same bucket per
    step (SURVEY 8e: no stragglers): `batches()` yields whole global batches of `world` x per-GPU size."""

    def __init__(self, batch_size_per_gpu, max_src_len, max_trg_len, min_src_bucket_boundary=128, world=1,
                 frame_transcript_ratio=None, disable_batch_efficiency=False):
        assert batch_size_per_gpu > max_src_len, "batch size per gpu (%d) must be greater than max_src_len (%d)" % (
            batch_size_per_gpu, max_src_len)
        self.world = world
        self.max_trg_len = minimal_multiple(max_trg_len, 8)
        b = create_audio_bucket_boundaries(max_src_len, min_src_bucket_boundary)
        b[-1] = minimal_multiple(b[-1], 8)
        self.boundaries = b
        if disable_batch_efficiency:
            self.batch_sizes = [int(batch_size_per_gpu // x) for x in b]
        else:
            self.batch_sizes = [int(minimal_multiple(batch_size_per_gpu // x, 8)) for x in b]
        n = len(b)
        if frame_transcript_ratio is None:
            # the reference pads transcripts to the longest of each batch (padded_shapes [None]); a fixed bound keeps the
            # shapes static for CUDA-graph capture and changes no result (padding is masked out of the loss)
            self.trg_bounds = [self.max_trg_len] * n
            self.trg_pairs = [[self.max_trg_len] for _ in range(n)]
        else:
            r = frame_transcript_ratio
            tb = [int(x / (r + i * (max_src_len / self.max_trg_len - r) / n)) for i, x in enumerate(b)]
            self.trg_bounds = [minimal_multiple(min(t, self.max_trg_len), 8) for t in tb]
            # speech2text.py:335-343: every audio bucket accepts its own transcript bound and the next bucket's
            self.trg_pairs = [[self.trg_bounds[i], self.trg_bounds[min(i + 1, n - 1)]] for i in range(n)]

    def bucket_of(self, n_frames, n_trg=0):
        """example_to_bucket_id (speech2text.py:350-360): the first (audio bucket i, transcript slot j) in row-major order
        with n_frames <= bound_i and n_trg <= trans_bound[i][j]; None when nothing matches (the reference filters such
        examples out beforehand with clean_dataset_by_length)."""
        for i, bound in enumerate(self.boundaries):
            if n_frames <= bound:
                for j, tb in enumerate(self.trg_pairs[i]):
                    if n_trg <= tb:
                        return (i, j)
        return None

    def shapes(self):
        """[(T, B per GPU, L)] — the static shape buckets (one captured CUDA graph each in the trainer)."""
        out = []
        for i, (t, bs) in enumerate(zip(self.boundaries, self.batch_sizes)):
            for l in self.trg_pairs[i]:
                if (t, bs, l) not in out:
                    out.append((t, bs, l))
        return out

    def batches(self, examples, pad_id=0, feature_dim=80, groups_only=False):
        """examples: iterable of dict(audio: FloatTensor [n, F], transcript: LongTensor [l]).  Yields per-replica lists of
        padded batches {src [B,T,F,1], src_length, trg [B,L], trg_length}; group_by_window + padded_batch(drop_remainder)
        like the reference: a batch leaves as soon as its bucket holds batch_size x world examples.  `groups_only`: yield
        (bucket key, per-replica example lists) and leave the padding to the caller (SpeechToText pads in worker threads)."""
        pools = {}
        for ex in examples:
            key = self.bucket_of(ex["audio"].shape[0], ex["transcript"].numel())
            if key is None:
                continue
            pool = pools.setdefault(key, [])
            pool.append(ex)
            if len(pool) == self.batch_sizes[key[0]] * self.world:
                pools[key] = []
                if groups_only:
                    yield key, [pool[r::self.world] for r in range(self.world)]
                else:
                    yield [self._pad(pool[r::self.world], key, pad_id, feature_dim) for r in range(self.world)]

    def _pad(self, group, key, pad_id, feature_dim):
        T, L, B = self.boundaries[key[0]], self.trg_pairs[key[0]][key[1]], len(group)
        flat = torch.empty(B, T * feature_dim)
        trg = torch.full((B, L), int(pad_id), dtype=torch.long)
        sl, tl = torch.zeros(B, dtype=torch.long), torch.zeros(B, dtype=torch.long)
        rows = []
        for j, ex in enumerate(group):
            n, l = ex["audio"].shape[0], ex["transcript"].numel()
            a = ex["audio"]
            rows.append(a if (a.dtype == torch.float32 and a.is_contiguous()) else a.to(torch.float32).contiguous())
            trg[j, :l] = ex["transcript"]
            sl[j], tl[j] = n, l
        # padded_batch in C (libb200st_io: one memcpy + one memset per row, outside the GIL): every byte written exactly once
        import ctypes as C
        from neurst_b200.tfrecord import io_lib
        ptrs = (C.c_void_p * B)(*[r.data_ptr() for r in rows])
        lens = (C.c_int64 * B)(*[r.numel() for r in rows])
        io_lib().b200st_pad_rows_f32(flat.data_ptr(), T * feature_dim, ptrs, lens, B)
        return dict(src=flat.view(B, T, feature_dim, 1), src_length=sl, trg=trg, trg_length=tl)


class SpeechToText:
    """Data side of the `SpeechToText` task for already extracted features and tokenised transcripts
    (neurst/tasks/speech2text.py): get_data_preprocess_fn (:163-236), the TRAIN branch of create_and_batch_tfds (:238-384)
    and example_to_input (:135-161).  Raw audio / raw text need the reference's extractor and text pipeline and are refused,
    as the reference refuses raw audio ("We recommend one to preprocess the audio in advance")."""

    def __init__(self, trg_meta, max_src_len, max_trg_len, batch_size_per_gpu, audio_feature_dim=80, audio_feature_channels=1,
                 truncate_src=False, truncate_trg=False, min_src_bucket_boundary=128, frame_transcript_ratio=None,
                 disable_batch_efficiency=False, specaug=None, world=1, padding_mode="default"):
        if max_src_len is None:
            raise RuntimeError("`max_src_len` for SpeechToText task must be provided.")
        if max_trg_len is None:
            raise RuntimeError("`max_trg_len` for SpeechToText task must be provided.")
        self.meta = dict(trg_meta)
        self.dim, self.channels = audio_feature_dim, audio_feature_channels
        self.max_src_len, self.max_trg_len = max_src_len, max_trg_len
        self.truncate_src, self.truncate_trg = truncate_src, truncate_trg
        self.specaug = SpecAugment.build(specaug)
        self.padding_mode = padding_mode
        self.bucketer = FrameBudgetBucketer(batch_size_per_gpu, max_src_len, max_trg_len, min_src_bucket_boundary, world,
                                            frame_transcript_ratio, disable_batch_efficiency)

    def preprocess_fn(self, data_status, training=True, with_label=True):
        if data_status["audio"] != "projected":
            raise RuntimeError("We recommend one to preprocess the audio in advance.")
        if with_label and data_status["transcript"] != "projected":
            raise RuntimeError("raw transcripts need the reference's text pipeline (tokenizer / BPE / vocabulary): "
                               "write the TFRecords with projected (int64) transcripts")
        width = self.dim * self.channels

        def proc(data):
            import warnings
            with warnings.catch_warnings():          # zero-copy view of the read-only file mapping: it is only ever read
                warnings.simplefilter("ignore", UserWarning)
                audio = torch.as_tensor(data["audio"], dtype=torch.float32).reshape(-1)
            if self.truncate_src and self.max_src_len:
                audio = audio[:self.max_src_len * width]
            ret = {"audio": audio.reshape(-1, width), "audio_length": audio.numel() // width}
            if with_label:
                text = torch.as_tensor(data["transcript"], dtype=torch.long).reshape(-1)
                if training and self.truncate_trg and self.max_trg_len and text.numel() > self.max_trg_len:
                    text = torch.cat([text[:self.max_trg_len - 1], text[-1:]])
                ret["transcript"] = text
            return ret
        return proc

    def keep(self, ex):
        """clean_dataset_by_length (dataset_utils.py:326-336): drop empty samples (size <= 1) and samples beyond the maxima."""
        a, t = ex["audio"].numel(), ex["transcript"].numel()
        return 1 < a <= self.max_src_len * self.dim * self.channels and 1 < t <= self.max_trg_len

    def train_batches(self, examples, generator=None, pin=False):
        """examples: preprocessed samples (in the order the dataset yields them; shuffling is the caller's, as
        `shuffle_buffer` is in the reference).  Yields, per step, the list of per-replica model inputs.  Meant to run inside
        a `Prefetcher` thread: 11 ms per 24 000-frame batch on one host core (2.4 M padded frames/s); a thread pool for the
        padding was measured SLOWER (0.6-0.9 M frames/s: the copies already use torch's intra-op threads)."""
        pad = int(self.meta["pad_id"])
        width = self.dim * self.channels
        kept = (e for e in examples if self.keep(e))
        for key, groups in self.bucketer.batches(kept, pad_id=pad, feature_dim=width, groups_only=True):
            # SpecAugment stays reproducible and independent of batching internals: one seed per batch, drawn in order
            seed = int(torch.randint(0, 2 ** 31 - 1, (1,), generator=generator)) if self.specaug is not None else 0
            out = []
            for r, group in enumerate(groups):
                b = self.bucketer._pad(group, key, pad, width)
                B, T = b["src"].shape[0], b["src"].shape[1]
                src = b["src"].reshape(B, T, self.dim, self.channels)
                if self.specaug is not None:       # the reference augments each utterance before padding: same masks, padding untouched
                    src = self.specaug(src, b["src_length"], generator=torch.Generator().manual_seed(seed + r))
                out.append(self.example_to_input(dict(audio=src, audio_length=b["src_length"], transcript=b["trg"]), pin=pin))
            yield out

    def example_to_input(self, batch, infer=False, pin=False):
        B = batch["audio"].shape[0]
        d = {"src": batch["audio"].reshape(B, -1, self.dim, self.channels), "src_length": batch["audio_length"].to(torch.long)}
        bos = torch.full((B,), int(self.meta["bos_id"]), dtype=torch.long)
        if infer:
            d["trg_input"] = bos
        else:
            trg = batch["transcript"]
            pad = int(self.meta["pad_id"])
            if self.padding_mode == "default":                     # deduce_text_length (models/model_utils.py:23-41)
                d["trg_length"] = (trg != pad).sum(1)
            else:                                                  # EOS_AS_PADDING: first pad (= eos) position + 1
                d["trg_length"] = (trg != pad).to(torch.int32).argmin(-1) + 1
            d["trg"] = trg
            d["trg_input"] = torch.cat([bos[:, None], trg[:, :-1]], 1)
        if pin and torch.cuda.is_available():
            d = {k: v.contiguous().pin_memory() for k, v in d.items()}
        return d


# ------------------------------------------------------------------------------------------------ text (seq2seq) side
_MIN_BUCKET_BOUNDARY = 8
_BUCKET_BOUNDARY_SCALE = 1.1


def create_batch_bucket_boundaries(max_length, min_boundary=_MIN_BUCKET_BOUNDARY, boundary_scale=_BUCKET_BOUNDARY_SCALE):
    """neurst/data/dataset_utils.py:125-147: boundaries grown by `boundary_scale` (at least +1), closed by max_length + 1."""
    bounds = []
    x = min_boundary
    while x < max_length:
        bounds.append(x)
        x = max(x + 1, int(x * boundary_scale))
    if not bounds or bounds[-1] < max_length + 1:
        bounds = bounds + [max_length + 1]
    return bounds


def associated_bucket_boundaries(a, b):
    """dataset_utils.py:150-178: two boundary lists resampled to the shorter one's length."""
    la, lb = len(a), len(b)
    if la == lb:
        return a, b
    s1, s2 = (la * 1. / lb, 1) if la > lb else (1, lb * 1. / la)
    return ([a[int(math.ceil(i * s1)) - 1] for i in range(1, min(la, lb) + 1)],
            [b[int(math.ceil(i * s2)) - 1] for i in range(1, min(la, lb) + 1)])


def adjust_batch_size(batch_size=None, batch_size_per_gpu=None, bucket_boundaries=None, num_replicas_in_sync=1):
    """dataset_utils.py:435-464 -> the global batch size in samples (no boundaries) or, by tokens, the list of global
    batch sizes per bucket: tokens // max(bucket boundaries), a multiple of the replica count."""
    if batch_size is None and batch_size_per_gpu is None:
        raise ValueError("At least one of the `batch_size` and `batch_size_per_gpu` should be provided.")
    if batch_size_per_gpu is not None:
        batch_size = int(batch_size_per_gpu * num_replicas_in_sync)
    if bucket_boundaries is None:
        return int(batch_size // num_replicas_in_sync * num_replicas_in_sync)
    n = min(len(v) for v in bucket_boundaries.values())
    return [int(batch_size // max(v[i] for v in bucket_boundaries.values()) // num_replicas_in_sync * num_replicas_in_sync)
            for i in range(n)]


class TokenBucketer:
    """The TRAIN branch of Seq2Seq.create_and_batch_tfds (seq2seq.py:248-270) with batch_examples_by_token
    (dataset_utils.py:467-560): bucket i holds the pairs with len(src) <= src_bounds[i] and len(trg) <= trg_bounds[i]
    (the first such i), is padded to exactly (src_bounds[i], trg_bounds[i]) and leaves as a global batch of
    batch_sizes[i] pairs, drop_remainder.  Each (bucket, per-replica batch) is one static shape, and every replica takes
    the same bucket per step: `batches()` yields whole global batches split into `world` equal parts."""

    def __init__(self, max_src_len, max_trg_len, batch_size=None, batch_size_per_gpu=None, batch_by_tokens=False, world=1):
        if max_src_len is None:
            raise RuntimeError("Must provide `max_src_len` for training.")
        if max_trg_len is None:
            raise RuntimeError("Must provide `max_trg_len` for training.")
        self.world = int(world)
        self.src_bounds, self.trg_bounds = associated_bucket_boundaries(create_batch_bucket_boundaries(int(max_src_len)),
                                                                        create_batch_bucket_boundaries(int(max_trg_len)))
        sizes = adjust_batch_size(batch_size, batch_size_per_gpu, num_replicas_in_sync=self.world,
                                  bucket_boundaries={"feature": self.src_bounds, "label": self.trg_bounds} if batch_by_tokens else None)
        self.batch_sizes = sizes if isinstance(sizes, list) else [sizes] * len(self.src_bounds)
        bad = [i for i, s in enumerate(self.batch_sizes) if s < self.world]
        if bad:
            raise ValueError("batch size %s%s gives bucket (%d, %d) fewer than one pair per replica (%d replicas)" % (
                batch_size if batch_size_per_gpu is None else batch_size_per_gpu,
                " tokens" if batch_by_tokens else "", self.src_bounds[bad[0]], self.trg_bounds[bad[0]], self.world))

    def bucket_of(self, n_src, n_trg):
        for i, (s, t) in enumerate(zip(self.src_bounds, self.trg_bounds)):
            if n_src <= s and n_trg <= t:
                return i
        return None

    def shapes(self):
        """[(T, B per replica, L)]: the static shapes (one captured CUDA graph each in the trainer)."""
        return [(s, b // self.world, t) for s, t, b in zip(self.src_bounds, self.trg_bounds, self.batch_sizes)]

    def batches(self, examples):
        """examples: {feature: LongTensor, transcript: LongTensor} -> (bucket, [per-replica example lists])."""
        pools = {}
        for ex in examples:
            key = self.bucket_of(ex["feature"].numel(), ex["transcript"].numel())
            if key is None:
                continue
            pool = pools.setdefault(key, [])
            pool.append(ex)
            if len(pool) == self.batch_sizes[key]:
                pools[key] = []
                yield key, [pool[r::self.world] for r in range(self.world)]


def _pad_ids(rows, length, pad):
    out = torch.full((len(rows), length), int(pad), dtype=torch.long)
    for j, r in enumerate(rows):
        out[j, :r.numel()] = r
    return out


class Seq2Seq:
    """Data side of the `Seq2Seq` task over BPE'd text (neurst/tasks/seq2seq.py): get_data_preprocess_fn (:165-190) with
    TextDataPipeline.encode(is_processed=True) (tokens -> ids, UNK for a token outside the vocabulary, EOS appended), the
    TRAIN batching of create_and_batch_tfds (TokenBucketer), the EVAL / INFER padded_batch (file order, padded to the
    longest in the batch) and example_to_input (:130-155).  Both sides use EOS as padding.  Raw text needs the
    reference's tokenizer and BPE and is refused."""

    def __init__(self, src_meta, trg_meta, max_src_len=None, max_trg_len=None, truncate_src=False, truncate_trg=False,
                 batch_size=None, batch_size_per_gpu=None, batch_by_tokens=False, world=1):
        self.src_meta, self.meta = dict(src_meta), dict(trg_meta)
        for m in (self.src_meta, self.meta):
            if not m.get("tokens"):
                raise RuntimeError("the text path needs the vocabulary file (*_data_pipeline.params.vocab_path)")
        self._src_vocab = {w: i for i, w in enumerate(self.src_meta["tokens"])}
        self._trg_vocab = {w: i for i, w in enumerate(self.meta["tokens"])}
        self.max_src_len, self.max_trg_len = max_src_len, max_trg_len
        self.truncate_src, self.truncate_trg = truncate_src, truncate_trg
        self._batching = dict(batch_size=batch_size, batch_size_per_gpu=batch_size_per_gpu, batch_by_tokens=batch_by_tokens,
                              world=world)
        self._bucketer = None

    @property
    def bucketer(self):
        if self._bucketer is None:
            self._bucketer = TokenBucketer(self.max_src_len, self.max_trg_len, **self._batching)
        return self._bucketer

    @staticmethod
    def encode(text, vocab, meta):
        """TextDataPipeline.encode(is_processed=True): whitespace tokens -> ids (UNK when missing) + [EOS]."""
        unk = int(meta["unk_id"])
        return [vocab.get(w, unk) for w in text.split()] + [int(meta["eos_id"])]

    @staticmethod
    def truncate(ids, max_len):
        """seq2seq.py:171-176: beyond max_len keep the first max_len - 1 tokens and the last one (EOS)."""
        return ids[:max_len - 1] + ids[-1:] if len(ids) > max_len else ids

    def preprocess_fn(self, data_status, training=True, with_label=True):
        if data_status["feature"] != "processed" or (with_label and data_status.get("label") != "processed"):
            raise RuntimeError("raw text needs the reference's text pipeline (tokenizer / BPE): give BPE'd files with "
                               "dataset.params.data_is_processed: True")

        def side(text, vocab, meta, trunc, max_len):
            ids = self.encode(text, vocab, meta)
            if training and trunc and max_len:
                ids = self.truncate(ids, int(max_len))
            return torch.tensor(ids, dtype=torch.long)

        def proc(data):
            ret = {"feature": side(data["feature"], self._src_vocab, self.src_meta, self.truncate_src, self.max_src_len)}
            if with_label:
                ret["transcript"] = side(data["label"], self._trg_vocab, self.meta, self.truncate_trg, self.max_trg_len)
            return ret
        return proc

    def keep(self, ex):
        """clean_dataset_by_length (dataset_utils.py:328-337): 1 < length <= the maximum, on both sides."""
        s, t = ex["feature"].numel(), ex["transcript"].numel()
        return 1 < s <= int(self.max_src_len) and 1 < t <= int(self.max_trg_len)

    def train_batches(self, examples, generator=None, pin=False):
        """Yields, per step, the list of per-replica model inputs (padded to the bucket's bounds)."""
        b = self.bucketer
        kept = (e for e in examples if self.keep(e))
        for key, groups in b.batches(kept):
            T, Lq = b.src_bounds[key], b.trg_bounds[key]
            yield [self.example_to_input({"feature": _pad_ids([e["feature"] for e in g], T, self.src_meta["pad_id"]),
                                          "transcript": _pad_ids([e["transcript"] for e in g], Lq, self.meta["pad_id"])},
                                         pin=pin) for g in groups]

    def group_to_input(self, group, infer=True):
        """EVAL / INFER padded_batch of a list of samples: file order, padded to the longest source (and target)."""
        batch = {"feature": _pad_ids([e["feature"] for e in group], max(e["feature"].numel() for e in group),
                                     self.src_meta["pad_id"])}
        if not infer:
            batch["transcript"] = _pad_ids([e["transcript"] for e in group], max(e["transcript"].numel() for e in group),
                                           self.meta["pad_id"])
        return self.example_to_input(batch, infer=infer)

    @staticmethod
    def _eos_padded_length(x, pad):
        # deduce_text_length with EOS_AS_PADDING (models/model_utils.py:23-41): first pad (= EOS) position + 1
        return (x != pad).to(torch.int32).argmin(-1) + 1

    def example_to_input(self, batch, infer=False, pin=False):
        src = batch["feature"]
        B, T = src.shape
        src_length = self._eos_padded_length(src, int(self.src_meta["pad_id"])).to(torch.long)
        d = {"src": src, "src_padding": (torch.arange(T)[None, :] >= src_length[:, None]).to(torch.float32)}
        bos = torch.full((B,), int(self.meta["bos_id"]), dtype=torch.long)
        if infer:
            d["trg_input"] = bos
        else:
            trg = batch["transcript"]
            d["trg_length"] = self._eos_padded_length(trg, int(self.meta["pad_id"])).to(torch.long)
            d["trg"] = trg
            d["trg_input"] = torch.cat([bos[:, None], trg[:, :-1]], 1)
        if pin and torch.cuda.is_available():
            d = {k: v.contiguous().pin_memory() for k, v in d.items()}
        return d


class Prefetcher:
    """Runs an iterator in a background thread with a bounded queue — the role of tf.data's prefetch in the reference's
    input pipeline (neurst/exps/trainer.py:258-262): file reads, record parsing, padding and pinning of the next batches
    overlap the GPU step of the current one (the copies and NumPy / torch kernels release the GIL)."""

    _END = object()

    def __init__(self, iterable, depth=3, init=None):
        """`init` runs first inside the thread (e.g. torch.cuda.set_device(local_rank): pinning memory from a thread whose
        current device is 0 would create a context on GPU 0 from every rank)."""
        import queue
        import threading
        self._q = queue.Queue(maxsize=max(1, int(depth)))
        self._exc = None
        self._stop = False

        def work():
            try:
                if init is not None:
                    init()
                for item in iterable:
                    while not self._stop:
                        try:
                            self._q.put(item, timeout=0.1)
                            break
                        except queue.Full:
                            continue
                    if self._stop:
                        return
            except BaseException as e:      # re-raised in the consumer
                self._exc = e
            finally:
                while not self._stop:
                    try:
                        self._q.put(self._END, timeout=0.1)
                        break
                    except queue.Full:
                        continue

        self._t = threading.Thread(target=work, daemon=True)
        self._t.start()
        _LIVE_PREFETCHERS.add(self)

    def __iter__(self):
        return self

    def __next__(self):
        item = self._q.get()
        if item is self._END:
            self._stop = True
            if self._exc is not None:
                raise self._exc
            raise StopIteration
        return item

    def close(self):
        """Stops the producer and waits for it (a thread still inside a torch call while the interpreter finalises aborts
        the process)."""
        self._stop = True
        try:
            while True:
                self._q.get_nowait()
        except Exception:
            pass
        self._t.join(timeout=10.0)
        _LIVE_PREFETCHERS.discard(self)


import atexit
import weakref

_LIVE_PREFETCHERS = weakref.WeakSet()


@atexit.register
def _close_prefetchers():
    for p in list(_LIVE_PREFETCHERS):
        p.close()


class SpecAugment:
    """SpecAugment with the reference's settings table and sampling rule (audio_lib.py:27-66,107-147,231-245):
    repeat n times f ~ U[0, F), f0 ~ U[0, nu - f); positions [f0, f0+f) := mask value (utterance mean unless given); a mask
    starting at 0 is skipped (the reference's `if f0[i] == 0: continue`); time masks are capped at p * frames."""
    SETTINGS = {"LB": dict(freq_mask_n=1, freq_mask_f=27, time_mask_n=1, time_mask_t=100, time_mask_p=1.0),
                "LD": dict(freq_mask_n=2, freq_mask_f=27, time_mask_n=2, time_mask_t=100, time_mask_p=1.0),
                "SM": dict(freq_mask_n=2, freq_mask_f=15, time_mask_n=2, time_mask_t=70, time_mask_p=0.2),
                "SS": dict(freq_mask_n=2, freq_mask_f=27, time_mask_n=2, time_mask_t=70, time_mask_p=0.2)}

    def __init__(self, freq_mask_n, freq_mask_f, time_mask_n, time_mask_t, time_mask_p, mask_value=None, time_wrap_w=0):
        assert time_mask_t > 0 and freq_mask_f > 0
        self.fn, self.ff, self.tn, self.tt, self.tp, self.mask_value = freq_mask_n, freq_mask_f, time_mask_n, time_mask_t, time_mask_p, mask_value

    @classmethod
    def build(cls, setting):
        if setting is None:
            return None
        if isinstance(setting, str):
            setting = cls.SETTINGS.get(setting)
        return cls(**setting) if setting else None

    @staticmethod
    def _ranges(n, F, size, gen, p=None):
        if size < F:
            return []
        if p:
            F = min(F, math.floor(size * p))
        if F <= 0:
            return []
        out = []
        f = torch.randint(0, F, (n,), generator=gen)
        for i in range(n):
            f0 = int(torch.randint(0, size - int(f[i]), (1,), generator=gen))
            if f0 == 0:
                continue
            out.append((f0, f0 + int(f[i])))
        return out

    def masks(self, lengths, n_freq, T, generator=None):
        """Host-sampled boolean masks [B, T] (time) and [B, n_freq] (frequency) for a padded batch."""
        B = len(lengths)
        tm, fm = torch.zeros(B, T, dtype=torch.bool), torch.zeros(B, n_freq, dtype=torch.bool)
        for b in range(B):
            for a, z in self._ranges(self.fn, self.ff, n_freq, generator):
                fm[b, a:z] = True
            for a, z in self._ranges(self.tn, self.tt, int(lengths[b]), generator, self.tp):
                tm[b, a:z] = True
        return tm, fm

    def __call__(self, src, src_length, generator=None):
        """src [B,T,F,1] (any device), src_length [B] -> augmented copy (same device).  Mask value = per-utterance mean over
        the real frames (`spectrogram.mean()` of the unpadded utterance in the reference)."""
        B, T, Fd = src.shape[0], src.shape[1], src.shape[2]
        lens = src_length.to("cpu")
        tm, fm = self.masks(lens, Fd, T, generator)
        dev = src.device
        valid = (torch.arange(T, device=dev)[None, :] < src_length.to(dev)[:, None])
        if self.mask_value is None:
            tot = (src[..., 0] * valid[..., None]).sum((1, 2))
            mv = tot / (src_length.to(dev).clamp(min=1).float() * Fd)
        else:
            mv = torch.full((B,), float(self.mask_value), device=dev)
        m = (tm.to(dev)[:, :, None] | fm.to(dev)[:, None, :]) & valid[..., None]
        return torch.where(m[..., None], mv[:, None, None, None].to(src.dtype), src)
