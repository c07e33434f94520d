"""Streaming simultaneous translation: the wait-k agent's read / write loop on the device.

Host mirror of
  SimulTransTextAgent                 neurst/utils/simuleval_agents/simul_trans_text_agent.py (policy, predict,
                                      segment_to_units, units_to_segment, build_task_and_model)
  WaitkTransformer.incremental_encode / incremental_decode   neurst/models/waitk_transformer.py:119-140

`StreamingSession` owns the device state of one source stream decoded by one or more WaitkTransformer members
(b200st_stream_*): every member's encoder self-attention caches, cross-attention memory and decoder caches grow in
place, a READ encodes only the new source ids, and a WRITE is one captured CUDA graph (every member's decoder step, the
equal-weight mixture, the argmax) followed by one pinned read of the emitted id.

`SimulTransTextAgent` restates the reference agent over pre-tokenised units: a source word (one SimulEval segment) is a
list of BPE tokens, joined by the subword-nmt `@@` convention of `cli.ids_to_text`, or by the reference's `BOW_PREFIX`
rule when the target vocabulary is made of `▁`-prefixed pieces.  Its model side is any object with read(ids),
write() -> int and reset(): a StreamingSession on the device, or a restatement in the tests.  `translate` replays
SimulEval's text-to-text loop offline (the `simuleval` entry of cli.py); SimulEval itself is not needed.
"""
import ctypes as C

import torch

from neurst_b200 import lib as L

BOW_PREFIX = "▁"
DEFAULT_EOS = "</s>"             # simuleval.DEFAULT_EOS
READ_ACTION, WRITE_ACTION = 0, 1
ABBREVIATIONS = ("lbs.", "Dr.", "Prof.", "Mr.", "Mrs.", "Ms.")


class StreamingSession:
    """One source stream decoded by 1..8 WaitkTransformer members sharing the target vocabulary (and d), on the device.

    read(ids): encode the source ids at the next positions for every member; write() -> int: one decoder step of every
    member over all of the memory read so far, the members' log-probabilities mixed as logsumexp - log n, and the argmax,
    which becomes the next decoder input; reset(start_id): empty the stream, with `start_id` (default BOS) as the first
    decoder input.  use_shadow: read the weight matrices from the members' 16-bit shadows (16-bit handles only)."""

    def __init__(self, models, use_shadow=False, max_src=256, max_trg=256, keep_encoder_output=False):
        models = list(models)
        if not 1 <= len(models) <= L.ENSEMBLE_MAX_MODELS:
            raise ValueError("a streaming session has 1..%d members, got %d" % (L.ENSEMBLE_MAX_MODELS, len(models)))
        for i, m in enumerate(models):
            if getattr(m, "wait_k", None) is None or not m.runtime.config.encoder_monotonic:
                raise ValueError("member %d is not a wait-k model with a monotonic encoder (WaitkTransformer): the streaming "
                                 "agent's incremental encoding needs one" % i)
        metas = [m._trg_meta for m in models]
        for i, meta in enumerate(metas[1:], 1):
            if meta["vocab_size"] != metas[0]["vocab_size"] or meta.get("tokens") != metas[0].get("tokens"):
                raise ValueError("member %d's target vocabulary differs from member 0's: the agent mixes the members' "
                                 "distributions over one vocabulary" % i)
        self.models, self.trg_meta = models, metas[0]
        self.max_src, self.max_trg = int(max_src), int(max_trg)
        self.lib = L.load()
        dev = models[0].runtime.device
        self.device = dev
        self._keep = []
        self.states = []
        members = (L.StreamMember * len(models))()
        for i, m in enumerate(models):
            rt = m.runtime
            cfg = rt.config
            from neurst_b200.decode import _bufs
            bufs = _bufs(rt)
            enc_kv = torch.zeros(cfg.enc_layers, 2, self.max_src, cfg.d, dtype=torch.float32, device=dev)
            cross_kv = torch.zeros(cfg.dec_layers, self.max_src, 2 * cfg.d, dtype=torch.float32, device=dev)
            self_kv = torch.zeros(cfg.dec_layers, 2, self.max_trg, cfg.d, dtype=torch.float32, device=dev)
            enc_out = torch.zeros(self.max_src, cfg.d, dtype=torch.float32, device=dev) if keep_encoder_output else None
            scratch = torch.zeros(int(self.lib.b200st_stream_scratch_floats(rt.handle)), dtype=torch.float32, device=dev)
            st = L.StreamState()
            st.max_src, st.max_trg = self.max_src, self.max_trg
            st.enc_kv, st.cross_kv, st.self_kv = enc_kv.data_ptr(), cross_kv.data_ptr(), self_kv.data_ptr()
            st.enc_out = enc_out.data_ptr() if enc_out is not None else None
            st.scratch, st.use_shadow = scratch.data_ptr(), int(bool(use_shadow))
            self.states.append(dict(enc_kv=enc_kv, cross_kv=cross_kv, self_kv=self_kv, enc_out=enc_out))
            self._keep += [bufs, st, scratch]
            members[i].h, members[i].buf, members[i].st = rt.handle, C.pointer(bufs), C.pointer(st)
        self._members = members
        self.lens = torch.zeros(2, dtype=torch.int32, device=dev)
        self.symbol = torch.zeros(1, dtype=torch.int64, device=dev)
        self._host_id = torch.zeros(1, dtype=torch.int64).pin_memory()
        self._stream = torch.cuda.Stream(device=dev)
        self._done = torch.cuda.Event()
        h = C.c_void_p()
        L.check(self.lib.b200st_stream_create(members, len(models), self.lens.data_ptr(), C.byref(h)))
        self._h = h
        self.reset()

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            self.lib.b200st_stream_destroy(h)
            self._h = None

    def _run(self, call):
        cur = torch.cuda.current_stream(self.device)
        self._stream.wait_stream(cur)
        with torch.cuda.stream(self._stream):
            L.check(call(C.c_void_p(self._stream.cuda_stream)))
        cur.wait_stream(self._stream)

    @property
    def lengths(self):
        """(src_len, trg_len): source ids encoded and decoder positions used (the library's host mirrors)."""
        a, b = C.c_int32(), C.c_int32()
        L.check(self.lib.b200st_stream_lengths(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def reset(self, start_id=None):
        start = int(self.trg_meta["bos_id"] if start_id is None else start_id)

        def call(s):
            self.symbol.fill_(start)
            return self.lib.b200st_stream_reset(self._h, s)
        self._run(call)

    def read(self, ids):
        ids = torch.as_tensor(ids, dtype=torch.int64).reshape(-1)
        if ids.numel() == 0:
            return
        dev_ids = ids.to(self.device)
        self._keep_ids = dev_ids
        self._run(lambda s: self.lib.b200st_stream_read(self._h, int(ids.numel()), dev_ids.data_ptr(), s))

    def write(self, weights=None):
        """One WRITE: the emitted id (also the next decoder input).  weights: None = equal (the agent's), else one per member."""
        w = None
        if weights is not None:
            w = (C.c_float * len(self.models))(*[float(x) for x in weights])

        def call(s):
            rc = self.lib.b200st_stream_write(self._h, w, self.symbol.data_ptr(), s)
            if rc == 0:
                self._host_id.copy_(self.symbol, non_blocking=True)
                self._done.record(self._stream)
            return rc
        self._run(call)
        self._done.synchronize()
        return int(self._host_id[0])


class _States:
    """The agent's per-sentence states (SimulEval TextStates, as SimulTransTextAgent.initialize_states fills them)."""

    def __init__(self):
        self.reading = True               # states.status["read"]
        self.units_source, self.units_target = [], []
        self.segments_source, self.segments_target = [], []
        self.queue_source, self.queue_target = [], []
        self.segment = False
        self.encoding_time = 0


class SimulTransTextAgent:
    """The reference agent over pre-tokenised units (see the module docstring).  model: read(ids) / write() / reset();
    src_meta, trg_meta: vocabulary metas (tokens, eos_id); wait_k counts source words (segments)."""

    def __init__(self, model, src_meta, trg_meta, wait_k, force_segment=False, max_len=200):
        if str(trg_meta.get("language", "")).lower() == "ja":
            raise ValueError("the agent's Japanese target branch (one character per segment) is outside this path")
        if not trg_meta.get("tokens"):
            raise ValueError("the agent merges target units into words: the target vocabulary needs its tokens")
        self.model, self.src_meta, self.trg_meta = model, src_meta, trg_meta
        self.wait_k, self.force_segment, self.max_len = int(wait_k), bool(force_segment), int(max_len)
        self.words = list(ABBREVIATIONS)
        self.src_ids = {t: i for i, t in enumerate(src_meta.get("tokens") or [])}
        self.bow = any(t.startswith(BOW_PREFIX) for t in trg_meta["tokens"])
        self.states = None

    # ---- states ----
    def initialize_states(self, states=None):
        """Empty states and an empty stream on the model; a sentence continued after a forced segment keeps reading."""
        if states is None:
            states = _States()
        else:
            reading = states.reading
            states.__init__()
            states.reading = reading
        self.states = states
        self.model.reset()
        return states

    # ---- segments <-> units ----
    def _segment_text(self, segment):
        """The word a list of source tokens spells (the SimulEval segment), for the force-segment punctuation rules."""
        return "".join(t[:-2] if t.endswith("@@") else t.replace(BOW_PREFIX, "") for t in segment)

    def segment_to_units(self, segment, states):
        """A source word (its tokens) -> its unit ids, with the EOS of a forced segment end."""
        if self.force_segment:
            s = self._segment_text(segment)
            if s.endswith('."') or s.endswith('?"') or s.endswith('!"'):
                if s.endswith('..."'):
                    states.segment = True
                elif len(s) > 2 and not s[-3].isupper() and s[:-1] not in self.words:
                    states.segment = True
            if s.endswith('.') or s.endswith('?') or s.endswith('!'):
                if s.endswith('...'):
                    states.segment = True
                elif len(s) > 1 and not s[-2].isupper() and s not in self.words:
                    states.segment = True
        unk = self.src_meta["unk_id"]
        units = [self.src_ids.get(t, unk) for t in segment]
        if self.force_segment and states.segment:
            units.append(self.src_meta["eos_id"])
        return units

    def _finish_forced(self, states):
        """force_segment while reading: the present sentence ends, the next one starts from empty states."""
        states.segment = False
        self.initialize_states(states)

    def units_to_segment(self, units, states):
        """Target units not yet emitted -> the words they complete (and DEFAULT_EOS), or None."""
        eos, tokens = self.trg_meta["eos_id"], self.trg_meta["tokens"]
        tok = (lambda i: tokens[i] if i < len(tokens) else "<UNK>")
        if units[0] == eos or len(states.segments_target) > self.max_len:
            units.pop(0)
            if self.force_segment and states.reading:
                self._finish_forced(states)
                return None
            return [DEFAULT_EOS]
        if self.bow:
            segment = []
            for n, index in enumerate(units):
                if index == eos:
                    break
                token = tok(index)
                if token.startswith(BOW_PREFIX) and segment:
                    del units[:n]
                    out = ["".join(segment)]
                    if units[0] == eos:
                        out.append(DEFAULT_EOS)
                    return out
                segment.append(token.replace(BOW_PREFIX, ""))
        else:
            for n, index in enumerate(units):
                if index == eos:
                    break
                if not tok(index).endswith("@@"):          # the word ends here (subword-nmt: "@@" continues it)
                    word = "".join(tok(i)[:-2] if tok(i).endswith("@@") else tok(i) for i in units[:n + 1])
                    del units[:n + 1]
                    return [word]
        if (units and units[-1] == eos) or len(states.units_target) > self.max_len:
            pieces = [tok(u) for u in units][:-1]
            text = "".join(p[:-2] if p.endswith("@@") else p for p in pieces).replace(BOW_PREFIX, "")
            del units[:]
            if self.force_segment and states.reading:
                self._finish_forced(states)
                return [text] if text else None
            return ([text] if text else []) + [DEFAULT_EOS]
        return None

    # ---- the policy and the prediction ----
    def policy(self, states):
        if self.force_segment and not states.reading:
            return WRITE_ACTION
        if self.force_segment and states.segment:
            return READ_ACTION if states.queue_source else WRITE_ACTION
        if not states.reading and (not states.units_source or states.units_source[-1] != self.src_meta["eos_id"]):
            states.units_source.append(self.src_meta["eos_id"])
        if states.queue_source and states.reading:
            return READ_ACTION
        if len(states.segments_source) - len(states.segments_target) < self.wait_k and states.reading:
            return READ_ACTION
        return WRITE_ACTION

    def predict(self, states):
        eos = self.trg_meta["eos_id"]
        if self.force_segment and not states.reading:
            return eos
        if len(states.units_target) > self.max_len:
            return eos
        new = states.units_source[states.encoding_time:]
        if new:
            self.model.read(new)
        states.encoding_time = len(states.units_source)
        return self.model.write()

    # ---- SimulEval's text-to-text loop, replayed offline ----
    def translate(self, words, clock=None):
        """Streams one sentence of source words (lists of tokens) through the agent.  Returns dict(prediction: the emitted
        target words, delays: source words read when each was emitted, actions: [(READ/WRITE, seconds)] when `clock`
        (a callable returning seconds after the device work of the action) is given)."""
        states = self.initialize_states()
        out, delays, actions = [], [], []
        n_read = 0
        while True:
            t0 = clock() if clock else 0.0
            action = self.policy(states)
            if action == READ_ACTION:
                if not states.queue_source:
                    if n_read < len(words):
                        seg = list(words[n_read])
                        n_read += 1
                        states.segments_source.append(seg)
                        states.queue_source.extend(self.segment_to_units(seg, states))
                    else:
                        states.reading = False
                states.units_source.extend(states.queue_source)
                del states.queue_source[:]
                # a READ encodes on the device when the agent predicts next: nothing to time here
                if clock:
                    actions.append(("R", clock() - t0))
                continue
            unit = self.predict(states)
            if clock:
                actions.append(("W", clock() - t0))
            states.units_target.append(unit)
            states.queue_target.append(unit)
            segs = self.units_to_segment(states.queue_target, states) if states.queue_target else None
            finished = False
            for w in segs or []:
                if w == DEFAULT_EOS:
                    finished = True
                    break
                out.append(w)
                delays.append(n_read)
                self.states.segments_target.append(w)
            if finished:
                break
        return dict(prediction=out, delays=delays, actions=actions)


def words_of(line, bow=False):
    """Source words (lists of tokens) of one pre-tokenised line: subword-nmt `@@` continuations, or `▁`-prefixed
    pieces starting a word (bow)."""
    words, cur = [], []
    for t in line.split():
        if bow:
            if t.startswith(BOW_PREFIX) and cur:
                words.append(cur)
                cur = []
            cur.append(t)
        else:
            cur.append(t)
            if not t.endswith("@@"):
                words.append(cur)
                cur = []
    if cur:
        words.append(cur)
    return words

