"""Restatement of the reference's beam search in torch (neurst/layers/search/beam_search.py:24-437), the checker of the
device beam search.  It follows the reference's data flow, not the device's: the decoding cache is tiled per beam
(stack_beam_size) and really gathered by parent beam every step, so the ancestry-table indexing of the CUDA path is checked
by an independent route.  Kept with the tests; the layers it calls are the oracle's (oracle/restatement.py)."""
import math

import torch
import torch.nn.functional as F

from oracle import restatement as R

FLOAT_MIN = R.FLOAT_MIN


def length_penalty(lengths, alpha):
    """_calculate_length_penalty (beam_search.py:24-40), fp32."""
    lengths = lengths.to(torch.float32)
    if alpha is None or alpha < 0.0:
        return torch.tensor(1.0, dtype=torch.float32) / lengths
    return ((5.0 + lengths) / 6.0) ** (-alpha)


def _map(fn, tree):
    if isinstance(tree, dict):
        return {k: _map(fn, v) for k, v in tree.items()}
    if isinstance(tree, (list, tuple)):
        return type(tree)(_map(fn, v) for v in tree)
    return fn(tree) if torch.is_tensor(tree) else tree


def _sorted_desc(x):
    """Descending along the last axis, the lower index first on ties (tf.nn.top_k)."""
    return torch.sort(x, dim=-1, descending=True, stable=True)


def beam_search(symbols_to_logits_fn, initial_ids, cache, eos_id, unk_id=None, beam_size=4, length_penalty_alpha=0.6, top_k=1,
                maximum_decode_length=256, extra_decode_length=50, minimum_decode_length=0, encoder_inputs_maxlen=None):
    """sequence_beam_search over `symbols_to_logits_fn(ids [N], cache, time) -> logits [N, V]` with `cache` a nested
    structure of tensors whose first axis is the batch.  `unk_id` None: UNK allowed.  Returns a dict: hypotheses
    [B*top_k, maximum_decode_length] padded with EOS, scores / logprob / length [B*top_k] best first per utterance, steps,
    and gap: the smallest score difference met between the beam-th and (beam+1)-th candidate of a step and between
    neighbouring final ranks up to top_k (a comparison with another implementation is only meaningful above it)."""
    B = initial_ids.shape[0]
    k = beam_size
    ids = initial_ids.repeat_interleave(k)                                             # stack_beam_size
    cache = _map(lambda x: x.repeat_interleave(k, 0), cache)
    N = B * k
    finished = torch.zeros(N, dtype=torch.bool)
    logprob = torch.zeros(N, dtype=torch.float32)
    length = torch.zeros(N, dtype=torch.long)
    pred = torch.zeros(N, 0, dtype=torch.long)
    steps = maximum_decode_length if encoder_inputs_maxlen is None else min(encoder_inputs_maxlen + extra_decode_length,
                                                                             maximum_decode_length)
    steps = max(steps, minimum_decode_length)                                          # :366-372
    base = torch.arange(B) * k
    gap = math.inf
    t = 0
    while t < steps and not bool(finished.all()):                                      # :417-424
        lp = torch.log_softmax(symbols_to_logits_fn(ids, cache, t).to(torch.float32), -1)     # :97-99
        V = lp.shape[-1]
        fin = finished.to(torch.float32).unsqueeze(1)
        fin_bias = torch.full((V,), FLOAT_MIN, dtype=torch.float32)
        fin_bias[eos_id] = 0.0
        lp = lp * (1.0 - fin) + fin_bias.unsqueeze(0) * fin                            # :113-125
        if unk_id is not None:
            lp[:, unk_id] += FLOAT_MIN                                                 # :128-138
        if t < minimum_decode_length - 1:
            lp[:, eos_id] += FLOAT_MIN                                                 # :380-388
        acc = lp + logprob.unsqueeze(1)                                                # :170
        next_length = length + 1 - finished.long()                                     # :172-173
        scores = (acc * length_penalty(next_length, length_penalty_alpha).unsqueeze(1)).reshape(B, k * V)
        if t == 0:
            scores = scores[:, :V]                                                     # first beam only (:181-186)
        vals, order = _sorted_desc(scores)
        if vals.shape[1] > k:
            gap = min(gap, float((vals[:, k - 1] - vals[:, k]).min()))
        sel = order[:, :k]                                                             # [B, beam]
        word = (sel % V).reshape(-1)
        parent = (sel // V + base.unsqueeze(1)).reshape(-1)
        logprob = acc.reshape(B, k * V).gather(1, sel).reshape(-1)                     # :205-210
        length = next_length[parent]
        pred = torch.cat([pred[parent], word.unsqueeze(1)], 1)                         # :395-404
        cache = _map(lambda x: x.index_select(0, parent), cache)
        ids = word
        finished = word == eos_id
        t += 1
    final = (logprob * length_penalty(length, length_penalty_alpha)).reshape(B, k)    # :217-251
    fvals, forder = _sorted_desc(final)
    for i in range(min(top_k, k - 1)):
        gap = min(gap, float((fvals[:, i] - fvals[:, i + 1]).min()))
    top = (forder[:, :top_k] + base.unsqueeze(1)).reshape(-1)
    hyp = F.pad(pred[top], (0, maximum_decode_length - pred.shape[1]), value=int(eos_id))        # :428-437
    return dict(hypotheses=hyp, scores=fvals[:, :top_k].reshape(-1), logprob=logprob[top], length=length[top], steps=t, gap=gap)


def speech_beam_search(P, cfg, src, src_length, bos_id, eos_id, unk_id=None, beam_size=4, length_penalty_alpha=0.6, top_k=1,
                       maximum_decode_length=256, extra_decode_length=50, minimum_decode_length=0):
    """The SpeechTransformer case: symbols_to_logits_fn of encoder_decoder_model.py:243-253 through the oracle's cached
    decoder; the cache (memory, memory bias, per-layer self-attention keys / values) is tiled and gathered per beam."""
    H = cfg["heads"]
    emb = R.add_position(R.conv_subsample(P, src))
    T2 = emb.shape[1]
    padding = R.input_length_to_padding(R.length_after_conv(src_length), T2, emb.dtype)
    enc = R.encoder(P, emb, padding, cfg["enc_layers"], H)
    B, d = src.shape[0], emb.shape[-1]
    layers = [dict(keys=torch.zeros(B, 0, H, d // H, dtype=emb.dtype), values=torch.zeros(B, 0, H, d // H, dtype=emb.dtype))
              for _ in range(cfg["dec_layers"])]
    cache = dict(memory=enc, memory_bias=R.input_padding_to_bias(padding), layers=layers)

    def symbols_to_logits_fn(ids, cache, time):
        x = R.target_embed(P, ids, time=time).unsqueeze(1)
        y = R.decoder(P, x, cache["memory"], cache["memory_bias"], cfg["dec_layers"], H, caches=cache["layers"])
        return R.logits_layer(P, y[:, 0])

    with torch.no_grad():
        return beam_search(symbols_to_logits_fn, torch.full((B,), int(bos_id), dtype=torch.long), cache, eos_id, unk_id,
                           beam_size, length_penalty_alpha, top_k, maximum_decode_length, extra_decode_length,
                           minimum_decode_length, encoder_inputs_maxlen=T2)
