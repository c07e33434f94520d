"""Inference on top of libb200st: encoder pass, decoding cache, cached decoder step, greedy search.

Host mirror of
  EncoderDecoderModel.get_symbols_to_logits_fn      neurst/models/encoder_decoder_model.py:211-261
  TransformerDecoder.create_decoding_internal_cache neurst/layers/decoders/transformer_decoder.py:105-147
  sequence_beam_search                              neurst/layers/search/beam_search.py:254-439
  sequence_sampling_search                          neurst/layers/search/sampling.py:103-250
  SequenceGenerator                                 neurst/exps/sequence_generator.py:62-86

Everything numeric is a library call (b200st_encode / b200st_decode_init / b200st_decode_step / b200st_greedy_search /
b200st_beam_search / b200st_ensemble_beam_search / b200st_sampling_search):
the key/value caches are preallocated device buffers owned by `DecodingCache`, the token ids and the position live on the
device, and the greedy loop replays one captured CUDA graph per token inside the library.
"""
import ctypes as C

import torch

from neurst_b200 import lib as L

MAX_ROWS = 8      # rows (batch x beam) per decoding step with the fp32 master weights
MAX_ROWS_SHADOW = 256   # with the 16-bit shadow (use_shadow=True): above 8 rows the step runs on the tensor cores


def max_rows(use_shadow):
    """Rows (utterances x beam) one decoding step holds."""
    return MAX_ROWS_SHADOW if use_shadow else MAX_ROWS


class DecodingCache:
    """`cache` argument of symbols_to_logits_fn: encoder memory (pre-projected per layer) + self-attention K/V.

    beam > 1 (beam search): the memory stays one copy per utterance, the self-attention cache and the step scratch hold
    B * beam rows: at most MAX_ROWS with the fp32 weights, MAX_ROWS_SHADOW with use_shadow.

    wait_k > 0 (a WaitkTransformer): step t attends to the memory keys j < min(Tm, wait_k + t), the offline form of the
    streaming wait-k agent (waitk_transformer.py:102-110); 0 attends to the whole memory."""

    def __init__(self, rt, B, Tm, max_len, memory_bias, use_shadow=False, beam=1, wait_k=0):
        cfg = rt.config
        limit = max_rows(use_shadow)
        if beam < 1 or not 1 <= B * beam <= limit:
            raise L.B200STError("decoding supports 1..%d rows (utterances x beam) per step, got %d x %d" % (limit, B, beam))
        dev = rt.device
        self.rt, self.B, self.Tm, self.max_len, self.beam = rt, B, Tm, max_len, beam
        rows = B * beam
        self.cross_kv = torch.zeros(cfg.dec_layers, B, max(Tm, 1), 2 * cfg.d, dtype=torch.float32, device=dev)
        self.self_kv = torch.zeros(cfg.dec_layers, 2, rows, max_len, cfg.d, dtype=torch.float32, device=dev)
        self.memory_bias = memory_bias
        n = int(rt.lib.b200st_decode_scratch_floats(rt.handle, rows))
        self.scratch = torch.zeros(n, dtype=torch.float32, device=dev)
        self.time = torch.zeros(1, dtype=torch.int32, device=dev)
        st = L.DecodeState()
        st.B, st.Tm, st.max_len = B, Tm, max_len
        st.cross_kv, st.self_kv = self.cross_kv.data_ptr(), self.self_kv.data_ptr()
        st.memory_bias = memory_bias.data_ptr() if memory_bias is not None else None
        st.scratch = self.scratch.data_ptr()
        st.use_shadow = int(bool(use_shadow))
        st.wait_k = int(wait_k)
        self.state = st

    # reference-shaped view of the cache (transformer_decoder.py:119-147) for inspection / tests
    def as_dict(self, upto):
        d, H = self.rt.config.d, self.rt.config.heads
        out = {}
        for i in range(self.rt.config.dec_layers):
            rows = self.self_kv.shape[2]
            out["layer_%d" % i] = {
                "self_attention": {"keys": self.self_kv[i, 0, :, :upto].reshape(rows, upto, H, d // H),
                                   "values": self.self_kv[i, 1, :, :upto].reshape(rows, upto, H, d // H)},
                "memory": {"keys": self.cross_kv[i, :, :, :d], "values": self.cross_kv[i, :, :, d:]}}
        return out


def _bufs(rt, need=0):
    if rt._shadow_stale:
        rt.refresh_shadow()
    return rt._buffers(max(int(need), 256), False)


def encode(rt, inputs):
    """Modality + encoder: returns (encoder_outputs fp32 [B,T',d], memory_bias fp32 [B,T'] additive)."""
    cfg = rt.config
    bt = L.Batch()
    keep = []

    def put(field, t, dtype):
        t = torch.as_tensor(t).to(device=rt.device, dtype=dtype).contiguous()
        keep.append(t)
        setattr(bt, field, t.data_ptr())

    src = inputs["src"]
    B, T = src.shape[0], src.shape[1]
    if cfg.model_type == L.MODEL_SPEECH:
        put("src", src, torch.float32)
        put("src_length", inputs["src_length"], torch.int64)
        Ts = ((T + 1) // 2 + 1) // 2
    else:
        put("src_ids", src, torch.int64)
        put("src_padding", inputs["src_padding"], torch.float32)
        Ts = T
    bt.B, bt.T, bt.L, bt.training = B, T, 1, 0
    enc = torch.empty(B, Ts, cfg.d, dtype=torch.float32, device=rt.device)
    bias = torch.empty(B, Ts, dtype=torch.float32, device=rt.device)
    need = int(rt.lib.b200st_encode_workspace_bytes(rt.handle, B, T))
    if need <= 0:
        raise L.B200STError("workspace planning failed: " + rt.lib.b200st_last_error().decode())
    bufs = _bufs(rt, need)
    L.check(rt.lib.b200st_encode(rt.handle, C.byref(bufs), C.byref(bt), enc.data_ptr(), bias.data_ptr(), L._stream()))
    return enc, bias


def create_decoding_cache(rt, encoder_outputs, memory_bias, max_len, use_shadow=False, beam=1, wait_k=0):
    """create_decoding_internal_cache(is_inference=True) + memorize_memory for every layer."""
    B, Tm, _ = encoder_outputs.shape
    cache = DecodingCache(rt, B, Tm, max_len, memory_bias.contiguous() if memory_bias is not None else None, use_shadow, beam,
                          wait_k)
    bufs = _bufs(rt)
    enc = encoder_outputs.to(torch.float32).contiguous()
    L.check(rt.lib.b200st_decode_init(rt.handle, C.byref(bufs), enc.data_ptr(), C.byref(cache.state), L._stream()))
    cache.memory = enc
    return cache


def decoder_step_logits(rt, symbols, cache, time):
    """symbols_to_logits_fn(symbols [B], cache, time) -> logits [B, V]."""
    if int(time) >= cache.max_len:
        raise L.B200STError("decode position %d beyond the cache length %d" % (int(time), cache.max_len))
    ids = torch.as_tensor(symbols).to(device=rt.device, dtype=torch.int64).reshape(-1).contiguous()
    cache.time.fill_(int(time))
    logits = torch.empty(cache.B, rt.config.vocab, dtype=torch.float32, device=rt.device)
    bufs = _bufs(rt)
    L.check(rt.lib.b200st_decode_step(rt.handle, C.byref(bufs), C.byref(cache.state), ids.data_ptr(), cache.time.data_ptr(),
                                      logits.data_ptr(), L._stream()))
    return logits


def _search_steps(Tm, maximum_decode_length, extra_decode_length, minimum_decode_length):
    """maximum_search_steps = max(min(T' + extra, maximum), minimum) (beam_search.py:366-372)."""
    return max(min(Tm + extra_decode_length, maximum_decode_length), minimum_decode_length)


def _bos(rt, bos_id, B):
    """The first decoder input of each utterance: one id for all, or one per utterance."""
    bos = torch.as_tensor(bos_id).to(device=rt.device, dtype=torch.int64).reshape(-1)
    return (bos.repeat(B) if bos.numel() == 1 else bos).contiguous()


def _state_words(rt, B, width, max_len, search):
    """The search's device state words, b200st_beam_state_bytes(B, width, max_len) of them (>= 512 bytes)."""
    nbytes = int(rt.lib.b200st_beam_state_bytes(rt.handle, B, width, max_len))
    if nbytes <= 0:
        raise L.B200STError("%s state sizing failed: %s" % (search, rt.lib.b200st_last_error().decode()))
    return torch.zeros((nbytes + 7) // 8, dtype=torch.int64, device=rt.device)


def _on_decode_stream(rt, call):
    """L.check(call()) on rt's side stream, ordered after and before the current stream's work: the library captures the
    step into a CUDA graph, which needs a real (non-legacy-default) stream.  `call` reads L._stream() when it runs."""
    cur = torch.cuda.current_stream(rt.device)
    side = getattr(rt, "_decode_stream", None)
    if side is None:
        side = rt._decode_stream = torch.cuda.Stream(device=rt.device)
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        L.check(call())
    cur.wait_stream(side)


def _pad_with_eos(out, steps, maximum_decode_length, eos_id):
    """The first `steps` columns, padded to the fixed output length with EOS (beam_search.py:428-436, sampling.py:253-256)."""
    out = out[:, :steps]
    if steps < maximum_decode_length:
        out = torch.cat([out, torch.full((out.shape[0], maximum_decode_length - steps), int(eos_id), dtype=torch.int64,
                                         device=out.device)], 1)
    return out


def _search_cache(rt, inputs, cache, width, width_name, search, maximum_decode_length, use_shadow, wait_k):
    """The caller's cache, checked to hold B * width rows, or the encoder pass over `inputs` and a new cache of B * width
    rows."""
    if cache is not None:
        if cache.self_kv.shape[2] < cache.B * width:
            raise L.B200STError("the decoding cache holds %d rows, %s needs %d"
                                % (cache.self_kv.shape[2], search, cache.B * width))
        return cache
    B = int(inputs["src"].shape[0])
    if B * width > max_rows(use_shadow):
        raise L.B200STError("%s decodes at most %d rows (utterances x %s) per call, got %d x %d"
                            % (search, max_rows(use_shadow), width_name, B, width))
    enc, bias = encode(rt, inputs)
    return create_decoding_cache(rt, enc, bias, maximum_decode_length, use_shadow, beam=width, wait_k=wait_k)


def greedy_search(rt, inputs, bos_id, eos_id, unk_id=None, maximum_decode_length=256, extra_decode_length=50,
                  minimum_decode_length=0, enable_unk=False, use_shadow=False, use_graph=True, cache=None, persistent=True,
                  wait_k=0):
    """sequence_beam_search(beam_size=1, top_k=1): returns (hypothesis int64 [B, maximum_decode_length] padded with EOS,
    log-probability [B], decoding length [B]).  `maximum_search_steps` = max(min(T' + extra, maximum), minimum)
    (beam_search.py:357-363)."""
    if cache is None:
        enc, bias = encode(rt, inputs)
        cache = create_decoding_cache(rt, enc, bias, maximum_decode_length, use_shadow, wait_k=wait_k)
    B = cache.B
    steps = min(_search_steps(cache.Tm, maximum_decode_length, extra_decode_length, minimum_decode_length), cache.max_len)
    bos = _bos(rt, bos_id, B)
    out = torch.empty(B, steps, dtype=torch.int64, device=rt.device)
    length = torch.zeros(B, dtype=torch.int32, device=rt.device)
    logprob = torch.zeros(B, dtype=torch.float32, device=rt.device)
    words = _state_words(rt, B, 1, cache.max_len, "greedy search")       # holds B rows' words
    a = L.GreedyArgs()
    a.bos_ids, a.eos_id = bos.data_ptr(), int(eos_id)
    a.unk_id = -1 if (enable_unk or unk_id is None) else int(unk_id)
    a.min_len, a.max_steps = int(minimum_decode_length), int(steps)
    a.out_ids, a.out_len, a.out_logprob = out.data_ptr(), length.data_ptr(), logprob.data_ptr()
    # persistent: the whole search is ONE cooperative kernel (grid barriers between the phases of a token); otherwise one
    # captured CUDA graph of ~40 kernels is replayed per token (use_graph) or every kernel is launched eagerly.  Above 8
    # rows there is no persistent kernel: the library replays the captured graph instead
    a.state_words, a.use_graph = words.data_ptr(), (2 if (persistent and use_graph) else int(bool(use_graph)))
    bufs = _bufs(rt)
    _on_decode_stream(rt, lambda: rt.lib.b200st_greedy_search(rt.handle, C.byref(bufs), C.byref(cache.state), C.byref(a),
                                                              L._stream()))
    if use_graph and int(rt.lib.b200st_greedy_used_graph()) < 1:
        raise L.B200STError("greedy search could neither run its persistent kernel nor capture its step graph")
    return _pad_with_eos(out, steps, maximum_decode_length, eos_id), logprob, length


def beam_search(rt, inputs, bos_id, eos_id, unk_id=None, beam_size=4, length_penalty=0.6, top_k=1, maximum_decode_length=256,
                extra_decode_length=50, minimum_decode_length=0, enable_unk=False, use_shadow=False, use_graph=True, cache=None,
                wait_k=0):
    """sequence_beam_search (beam_search.py:254-439) on the device: returns (hypotheses int64 [B*top_k, maximum_decode_length]
    padded with EOS, scores fp32 [B*top_k] = logprob * length penalty, best first per utterance, accumulated log-probabilities
    [B*top_k], decoding lengths [B*top_k]).  length_penalty < 0 (or None) scores by 1/length.  At most
    max_rows(use_shadow) // beam_size utterances per call, and beam_size <= 8.  beam_size 1 is the greedy search (with its persistent kernel when use_graph)."""
    return _beam_search([rt], None, inputs, bos_id, eos_id, unk_id, beam_size, length_penalty, top_k, maximum_decode_length,
                        extra_decode_length, minimum_decode_length, enable_unk, use_shadow, use_graph,
                        None if cache is None else [cache], wait_k)


def ensemble_weights(spec, n):
    """BeamSearch._get_ensemble_weights (beam_search.py:486-515): "average" gives 1/n each; comma-separated numbers (or a
    list of them) must count exactly n and are normalised to sum 1.  Whether the values are usable (finite, >= 0, a positive
    sum) is checked by the library, which normalises them again."""
    if spec is None or (isinstance(spec, str) and spec.strip() == "average"):
        return [1.0 / n] * n
    if isinstance(spec, (int, float)):          # one number, as a yaml or command-line value parses
        spec = [spec]
    eles = [float(x) for x in (spec.strip().split(",") if isinstance(spec, str) else spec)]
    if len(eles) != n:
        raise ValueError("The number of manual weights must have equal to the models.")
    total = sum(eles)
    return [x / total for x in eles] if total > 0 else eles


def ensemble_beam_search(rts, inputs, bos_id, eos_id, unk_id=None, weights="average", beam_size=4, length_penalty=0.6, top_k=1,
                         maximum_decode_length=256, extra_decode_length=50, minimum_decode_length=0, enable_unk=False,
                         use_shadow=False, use_graph=True, caches=None):
    """sequence_beam_search over an ensemble (EncoderDecoderEnsembleModel, beam_search.py:97-115) on the device: every step
    mixes the members' next-token distributions, log(sum_m w_m softmax(logits_m)), and searches on the mixture.  `rts` are
    the members' runtimes (same vocabulary); each runs its own encoder and keeps its own DecodingCache(beam=beam_size)
    (`caches`: one per member, built by create_decoding_cache).  `weights`: "average", comma-separated numbers or a list
    (ensemble_weights).  Returns what beam_search returns.  beam_size 1 is the ensemble's greedy search; one member is
    exactly beam_search."""
    rts = list(rts)
    n = len(rts)
    if not 1 <= n <= L.ENSEMBLE_MAX_MODELS:
        raise L.B200STError("an ensemble has 1..%d members, got %d" % (L.ENSEMBLE_MAX_MODELS, n))
    return _beam_search(rts, ensemble_weights(weights, n), inputs, bos_id, eos_id, unk_id, beam_size, length_penalty, top_k,
                        maximum_decode_length, extra_decode_length, minimum_decode_length, enable_unk, use_shadow, use_graph,
                        caches, 0)


def _beam_search(rts, weights, inputs, bos_id, eos_id, unk_id, beam_size, length_penalty, top_k, maximum_decode_length,
                 extra_decode_length, minimum_decode_length, enable_unk, use_shadow, use_graph, caches, wait_k):
    """beam_search (weights None: b200st_beam_search of rts[0]) and ensemble_beam_search (b200st_ensemble_beam_search)."""
    beam_size, top_k = int(beam_size), int(top_k)
    if beam_size < 1:
        raise L.B200STError("beam_size must be >= 1, got %d" % beam_size)
    if not 1 <= top_k <= beam_size:
        raise L.B200STError("top_k must be in 1..beam_size (%d), got %d" % (beam_size, top_k))
    if minimum_decode_length >= maximum_decode_length:          # BeamSearch.call (beam_search.py:531-532)
        raise L.B200STError("minimum_decode_length must be less than maximum_decode_length")
    n = len(rts)
    caches = [None] * n if caches is None else list(caches)
    if len(caches) != n:
        raise L.B200STError("%d decoding caches for %d ensemble members" % (len(caches), n))
    caches = [_search_cache(rt, inputs, c, beam_size, "beam_size", "beam search", maximum_decode_length, use_shadow, wait_k)
              for rt, c in zip(rts, caches)]
    rt0, c0 = rts[0], caches[0]
    B, dev = c0.B, rt0.device
    steps = _search_steps(c0.Tm, maximum_decode_length, extra_decode_length, minimum_decode_length)
    bos = _bos(rt0, bos_id, B)
    k = B * top_k
    out = torch.empty(k, max(steps, 1), dtype=torch.int64, device=dev)
    scores = torch.zeros(k, dtype=torch.float32, device=dev)
    logprob = torch.zeros(k, dtype=torch.float32, device=dev)
    length = torch.zeros(k, dtype=torch.int32, device=dev)
    words = _state_words(rt0, B, beam_size, c0.max_len, "beam search")
    a = L.BeamArgs()
    a.bos_ids, a.eos_id = bos.data_ptr(), int(eos_id)
    a.unk_id = -1 if (enable_unk or unk_id is None) else int(unk_id)
    a.min_len, a.max_steps = int(minimum_decode_length), int(steps)     # the library refuses steps beyond the cache
    a.beam_size, a.top_k, a.length_penalty = beam_size, top_k, -1.0 if length_penalty is None else float(length_penalty)
    a.out_ids, a.out_scores, a.out_logprob, a.out_len = out.data_ptr(), scores.data_ptr(), logprob.data_ptr(), length.data_ptr()
    a.state_words = words.data_ptr()
    # one model's beam 1 is the greedy search, with its persistent kernel
    a.use_graph = (2 if beam_size == 1 else 1) if use_graph else 0
    bufs = [_bufs(rt) for rt in rts]
    if weights is None:
        _on_decode_stream(rt0, lambda: rt0.lib.b200st_beam_search(rt0.handle, C.byref(bufs[0]), C.byref(c0.state), C.byref(a),
                                                                  L._stream()))
    else:
        members = (L.EnsembleMember * n)()
        for i, (rt, c) in enumerate(zip(rts, caches)):
            members[i].h, members[i].buf, members[i].st = rt.handle, C.pointer(bufs[i]), C.pointer(c.state)
            members[i].weight = weights[i]
        _on_decode_stream(rt0, lambda: rt0.lib.b200st_ensemble_beam_search(members, n, C.byref(a), L._stream()))
    if n == 1 and beam_size == 1 and use_graph and int(rt0.lib.b200st_greedy_used_graph()) < 1:
        raise L.B200STError("greedy search could neither run its persistent kernel nor capture its step graph")
    return _pad_with_eos(out, steps, maximum_decode_length, eos_id), scores, logprob, length


DEFAULT_SAMPLING_SEED = 1234      # the entries' default random_seed


def _check_sampling_filter(top_k, top_p):
    """Sampling.__init__'s refusal (sampling.py:313-314)."""
    if top_k > 0 and top_p < 1:
        raise NotImplementedError("Not implemented search logic when top_k > 0 and top_p < 1.")


def sampling_search(rt, inputs, bos_id, eos_id, unk_id, sample_num=1, top_k=0, top_p=1.0, maximum_decode_length=256,
                    extra_decode_length=50, minimum_decode_length=0, seed=DEFAULT_SAMPLING_SEED, row_offset=0, use_shadow=False,
                    use_graph=True, cache=None, wait_k=0):
    """sequence_sampling_search of TopSampling (neurst/layers/search/sampling.py:103-250) on the device: each utterance is
    decoded `sample_num` times (row b * sample_num + s is sample s of utterance b), every step masks UNK (unk_id None: not
    masked) and, before minimum_decode_length, EOS; keeps the top_k logits (top_k > 0) or the nucleus of mass top_p
    (top_p < 1); and draws one id per row with the keyed Philox draw of include/b200st.h (seed, global row
    row_offset + row, step).  A row that has emitted EOS emits EOS.  Returns (ids int64 [B*sample_num, maximum_decode_length]
    padded with EOS, log-probability fp32 [B*sample_num] of the drawn ids under the masked, unfiltered softmax, decoding
    length int32 [B*sample_num]).  At most max_rows(use_shadow) // sample_num utterances per call, sample_num <= 8."""
    sample_num, top_k, top_p = int(sample_num), int(top_k), float(top_p)
    _check_sampling_filter(top_k, top_p)
    if minimum_decode_length >= maximum_decode_length:          # Sampling.call (sampling.py:330-331)
        raise ValueError("`minimum_decode_length` must be less than maximum decode length.")
    if not 1 <= sample_num <= 8:
        raise L.B200STError("sample_num must be in 1..8, got %d" % sample_num)
    cache = _search_cache(rt, inputs, cache, sample_num, "sample_num", "sampling search", maximum_decode_length, use_shadow,
                          wait_k)
    B, dev = cache.B, rt.device
    steps = _search_steps(cache.Tm, maximum_decode_length, extra_decode_length, minimum_decode_length)
    bos = _bos(rt, bos_id, B)
    n = B * sample_num
    out = torch.empty(n, max(steps, 1), dtype=torch.int64, device=dev)
    logprob = torch.zeros(n, dtype=torch.float32, device=dev)
    length = torch.zeros(n, dtype=torch.int32, device=dev)
    words = _state_words(rt, B, sample_num, cache.max_len, "sampling search")
    a = L.SamplingArgs()
    a.bos_ids, a.eos_id = bos.data_ptr(), int(eos_id)
    a.unk_id = -1 if unk_id is None else int(unk_id)
    a.min_len, a.max_steps = int(minimum_decode_length), int(steps)     # the library refuses steps beyond the cache
    a.sample_num, a.top_k, a.top_p = sample_num, top_k, top_p
    a.seed, a.row_offset = int(seed) & 0xFFFFFFFFFFFFFFFF, int(row_offset)
    a.out_ids, a.out_logprob, a.out_len = out.data_ptr(), logprob.data_ptr(), length.data_ptr()
    a.state_words, a.use_graph = words.data_ptr(), int(bool(use_graph))
    bufs = _bufs(rt)
    _on_decode_stream(rt, lambda: rt.lib.b200st_sampling_search(rt.handle, C.byref(bufs), C.byref(cache.state), C.byref(a),
                                                                L._stream()))
    return _pad_with_eos(out, steps, maximum_decode_length, eos_id), logprob, length


def sample_logits(logits, top_k=0, top_p=1.0, seed=DEFAULT_SAMPLING_SEED, row_offset=0, step=0):
    """top_k_logits / top_p_logits and one draw per row (sampling.py:76-100 + tf.random.categorical) on caller logits fp32
    [rows, V] (CUDA), with the keyed draw of the sampling search: row r draws with (seed, row_offset + r, step).  No masks.
    -> int64 [rows]."""
    top_k, top_p = int(top_k), float(top_p)
    _check_sampling_filter(top_k, top_p)
    z = torch.as_tensor(logits)
    if z.dim() != 2 or not z.is_cuda:
        raise L.B200STError("sample_logits takes CUDA logits [rows, V]")
    z = z.to(torch.float32).contiguous()
    out = torch.empty(z.shape[0], dtype=torch.int64, device=z.device)
    L.check(L.load().b200st_sample_logits(z.data_ptr(), z.shape[0], z.shape[1], top_k, top_p, int(seed) & 0xFFFFFFFFFFFFFFFF,
                                          int(row_offset), int(step), out.data_ptr(), L._stream()))
    return out


def cascade_remap(asr_tokens, mt_src_tokens, mt_unk_id, asr_vocab_size):
    """int32 [asr_vocab_size] table ASR target id -> MT source id, by token string (TextDataPipeline's vocabulary lookup:
    a later duplicate wins); ids past the ASR token list (<UNK>, <SEQ_BEG>, <SEQ_END>) and tokens missing from the MT
    vocabulary map to the MT UNK."""
    index = {w: i for i, w in enumerate(mt_src_tokens)}
    table = torch.full((int(asr_vocab_size),), int(mt_unk_id), dtype=torch.int32)
    for i, w in enumerate(asr_tokens[:int(asr_vocab_size)]):
        table[i] = index.get(w, int(mt_unk_id))
    return table


def cascade_source(hyp_ids, remap, asr_eos_id, mt_vocab, mt_eos_id, mt_pad_id, mt_unk_id, max_src_len=0):
    """b200st_cascade_source: ASR top-1 hypotheses (device int64 [B, hyp_len]) -> the MT source batch on the device
    (src_ids int64 [B, T], src_padding fp32 [B, T], src_len int32 [B]), T the longest source (one copy of the lengths to
    the host sets it, as padded_batch pads to the longest of the batch)."""
    dev = hyp_ids.device
    hyp = hyp_ids.to(torch.int64).contiguous()
    B, n = hyp.shape
    remap = remap.to(device=dev, dtype=torch.int32).contiguous()
    lo, hi = int(remap.min()), int(remap.max())                   # the table is the caller's: checked before the launch
    if lo < 0 or hi >= int(mt_vocab):
        raise L.B200STError("cascade remap table holds ids outside the MT vocabulary of %d (%d..%d)" % (mt_vocab, lo, hi))
    width = min(n + 1, int(max_src_len)) if max_src_len else n + 1
    src = torch.empty(B, width, dtype=torch.int64, device=dev)
    pad = torch.empty(B, width, dtype=torch.float32, device=dev)
    length = torch.empty(B, dtype=torch.int32, device=dev)
    a = L.CascadeSourceArgs()
    a.hyp_ids, a.B, a.hyp_len, a.hyp_stride = hyp.data_ptr(), B, n, n
    a.asr_eos_id, a.asr_vocab, a.remap = int(asr_eos_id), remap.numel(), remap.data_ptr()
    a.mt_vocab, a.mt_eos_id, a.mt_pad_id, a.mt_unk_id = int(mt_vocab), int(mt_eos_id), int(mt_pad_id), int(mt_unk_id)
    a.max_src_len, a.out_stride = int(max_src_len or 0), width
    a.src_ids, a.src_padding, a.src_len = src.data_ptr(), pad.data_ptr(), length.data_ptr()
    L.check(L.load().b200st_cascade_source(C.byref(a), L._stream()))
    T = int(length.max())
    return src[:, :T], pad[:, :T], length
