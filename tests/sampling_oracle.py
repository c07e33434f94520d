"""Restatement of the reference's top-k / nucleus sampling search in fp64 (neurst/layers/search/sampling.py:76-250), the
checker of the device sampling search.  The reference's tf.random.categorical is replaced by the keyed draw the library
defines (include/b200st.h): Philox4x32-7 restated in numpy here, u = (x >> 8) * 2^-24, the first index whose running sum of
kept weights exceeds u * W.  The cache is tiled per sample (stack_beam_size) as the reference does.  Every function also
reports how close the search came to a rounding-sensitive decision, so a comparison can first assert that it met none."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import restatement as R

FLOAT_MIN = R.FLOAT_MIN
_MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32(seed, counter, stream, rounds=7):
    """The four 32-bit words of Philox4x32-`rounds` (Salmon et al. 2011) for key `seed` (64 bits), counter words
    (counter, stream) (64 bits each), as common.cuh's philox4x32.  Arguments broadcast as numpy uint64 arrays."""
    seed, counter, stream = (np.asarray(x, dtype=np.uint64) for x in (seed, counter, stream))
    k0, k1 = seed & _MASK32, seed >> np.uint64(32)
    c0, c1 = counter & _MASK32, counter >> np.uint64(32)
    c2, c3 = stream & _MASK32, stream >> np.uint64(32)
    for _ in range(rounds):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _MASK32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _MASK32
        k0 = (k0 + np.uint64(0x9E3779B9)) & _MASK32
        k1 = (k1 + np.uint64(0xBB67AE85)) & _MASK32
    return c0, c1, c2, c3


def uniforms(seed, step, rows):
    """u of the draws of global rows `rows` at `step`: (x >> 8) * 2^-24 with x the first Philox word (float64, exact)."""
    x = philox4x32(np.uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), np.uint64(step), np.asarray(rows, dtype=np.uint64))[0]
    return (x >> np.uint64(8)).astype(np.float64) * 2.0 ** -24


def filter_keep(z, top_k=0, top_p=1.0):
    """Boolean keep mask of top_p_logits (top_p < 1) or top_k_logits (top_k > 0) on z [N, V] (fp64), and the smallest margin
    of the threshold: for top-k the gap between the k-th and the (k+1)-th largest value; for top-p the distance of p to the
    cumulative probabilities on both sides of the threshold position, and the gap to the next value (inf without filter)."""
    z = torch.as_tensor(z, dtype=torch.float64)
    N, V = z.shape
    if top_p < 1.0:
        s, _ = torch.sort(z, dim=-1, descending=True)
        cum = torch.cumsum(torch.softmax(s, -1), -1)
        reach = cum >= top_p
        has = reach.any(-1)
        first = torch.where(has, reach.to(torch.int64).argmax(-1), torch.full((N,), V - 1, dtype=torch.int64))
        thr = torch.where(has, s.gather(1, first.unsqueeze(1))[:, 0], s[:, -1])
        margin = float("inf")
        for i in range(N):
            f = int(first[i])
            if not bool(has[i]):
                margin = min(margin, top_p - float(cum[i, -1]))
                continue
            margin = min(margin, float(cum[i, f]) - top_p)
            if f > 0:
                margin = min(margin, top_p - float(cum[i, f - 1]))
            if f + 1 < V:
                margin = min(margin, float(s[i, f] - s[i, f + 1]))
        return z >= thr.unsqueeze(1), margin
    if top_k > 0:
        s, _ = torch.sort(z, dim=-1, descending=True)
        thr = s[:, top_k - 1]
        margin = float((s[:, top_k - 1] - s[:, top_k]).min()) if top_k < V else float("inf")
        return z >= thr.unsqueeze(1), margin
    return torch.ones_like(z, dtype=torch.bool), float("inf")


def draw(z, keep, u):
    """The keyed draw on z [N, V] with keep mask and uniforms u [N]: the first index whose running sum of kept weights
    exp(z - max) exceeds u * W, and the smallest relative distance of u * W to a cumulative boundary."""
    z = torch.as_tensor(z, dtype=torch.float64)
    w = torch.where(keep, torch.exp(z - z.max(-1, keepdim=True).values), torch.zeros_like(z))
    cum = torch.cumsum(w, -1)
    W = cum[:, -1:]
    target = torch.as_tensor(u, dtype=torch.float64).unsqueeze(1) * W
    ids = (cum > target).to(torch.int64).argmax(-1)
    margin = float(((cum - target).abs() / W).min())
    return ids, margin


def sampling_search(symbols_to_logits_fn, initial_ids, cache, eos_id, unk_id=None, sample_num=1, top_k=0, top_p=1.0,
                    maximum_decode_length=256, extra_decode_length=50, minimum_decode_length=0, encoder_inputs_maxlen=None,
                    seed=1234, row_offset=0):
    """sequence_sampling_search over `symbols_to_logits_fn(ids [N], cache, time) -> logits [N, V]`.  Returns a dict: ids
    [B*sample_num, maximum_decode_length] padded with EOS (a finished row emits EOS), logprob (masked, unfiltered
    log-softmax of the drawn ids) and length [B*sample_num], steps, and the smallest draw / threshold margins met."""
    B = initial_ids.shape[0]
    ids = initial_ids.repeat_interleave(sample_num)
    cache = _map(lambda x: x.repeat_interleave(sample_num, 0), cache)
    N = B * sample_num
    finished = torch.zeros(N, dtype=torch.bool)
    logprob = torch.zeros(N, dtype=torch.float64)
    length = torch.zeros(N, dtype=torch.long)
    pred = torch.zeros(N, 0, dtype=torch.long)
    steps = maximum_decode_length if encoder_inputs_maxlen is None else min(encoder_inputs_maxlen + extra_decode_length,
                                                                             maximum_decode_length)
    steps = max(steps, minimum_decode_length)
    draw_margin = thr_margin = float("inf")
    t = 0
    while t < steps and not bool(finished.all()):
        z = symbols_to_logits_fn(ids, cache, t).to(torch.float64).clone()
        if unk_id is not None:
            z[:, unk_id] = FLOAT_MIN                                                    # _calculate_logits
        if t < minimum_decode_length - 1:
            z[:, eos_id] = FLOAT_MIN                                                    # :213-221
        lse = torch.logsumexp(z, -1)
        live = ~finished
        keep, m = filter_keep(z[live], top_k, top_p)
        u = uniforms(seed, t, np.arange(N, dtype=np.uint64)[live.numpy()] + np.uint64(row_offset))
        got, dm = draw(z[live], keep, u)
        thr_margin, draw_margin = min(thr_margin, m), min(draw_margin, dm)
        word = torch.full((N,), int(eos_id), dtype=torch.long)
        word[live] = got
        logprob[live] += z[live].gather(1, got.unsqueeze(1))[:, 0] - lse[live]
        length[live] += 1
        pred = torch.cat([pred, word.unsqueeze(1)], 1)
        ids = word
        finished = finished | (word == eos_id)
        t += 1
    hyp = F.pad(pred, (0, maximum_decode_length - pred.shape[1]), value=int(eos_id))
    return dict(ids=hyp, logprob=logprob, length=length, steps=t, draw_margin=draw_margin, threshold_margin=thr_margin)


def _map(fn, tree):
    if isinstance(tree, dict):
        return {k: _map(fn, v) for k, v in tree.items()}
    if isinstance(tree, (list, tuple)):
        return type(tree)(_map(fn, v) for v in tree)
    return fn(tree) if torch.is_tensor(tree) else tree


def _cached_decoder_fn(P, cfg):
    H = cfg["heads"]

    def symbols_to_logits_fn(ids, cache, time):
        x = R.target_embed(P, ids, time=time).unsqueeze(1)
        y = R.decoder(P, x, cache["memory"], cache["memory_bias"], cfg["dec_layers"], H, caches=cache["layers"])
        return R.logits_layer(P, y[:, 0])
    return symbols_to_logits_fn


def _empty_layers(cfg, B, dtype):
    H, d = cfg["heads"], cfg["d"]
    return [dict(keys=torch.zeros(B, 0, H, d // H, dtype=dtype), values=torch.zeros(B, 0, H, d // H, dtype=dtype))
            for _ in range(cfg["dec_layers"])]


def speech_sampling_search(P, cfg, src, src_length, bos_id, eos_id, unk_id=None, **kw):
    """The SpeechTransformer case in fp64: the oracle's encoder, then its cached decoder (encoder_decoder_model.py:243-253)."""
    P = {k: v.double() for k, v in P.items()}
    with torch.no_grad():
        emb = R.add_position(R.conv_subsample(P, src.double()))
        T2 = emb.shape[1]
        padding = R.input_length_to_padding(R.length_after_conv(src_length), T2, emb.dtype)
        enc = R.encoder(P, emb, padding, cfg["enc_layers"], cfg["heads"])
        B = src.shape[0]
        cache = dict(memory=enc, memory_bias=R.input_padding_to_bias(padding), layers=_empty_layers(cfg, B, torch.float64))
        return sampling_search(_cached_decoder_fn(P, cfg), torch.full((B,), int(bos_id), dtype=torch.long), cache, eos_id, unk_id,
                               encoder_inputs_maxlen=T2, **kw)


def decoder_sampling_search(P, cfg, memory, bias, bos_id, eos_id, unk_id=None, **kw):
    """The cached decoder (fp64, parameters as given: e.g. rounded like the 16-bit shadow) on a given memory."""
    B = memory.shape[0]
    cache = dict(memory=memory.double(), memory_bias=bias.double(), layers=_empty_layers(cfg, B, torch.float64))
    with torch.no_grad():
        return sampling_search(_cached_decoder_fn(P, cfg), torch.full((B,), int(bos_id), dtype=torch.long), cache, eos_id, unk_id,
                               encoder_inputs_maxlen=memory.shape[1], **kw)
