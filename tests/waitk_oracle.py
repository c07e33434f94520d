"""fp64 restatement of the wait-k model (neurst/models/waitk_transformer.py) on top of oracle/restatement.py, the checker of
the device's wait-k training and searches: the monotonic encoder's bias (transformer_encoder.py:119-123), the wait-k
cross-attention bias (transformer_decoder.py:194-208, layer_utils.py:56-78), both combined with the padding bias by `min`
as the reference does, the teacher-forced logits, and the cached decoder step with the lag of search step t (k + t,
waitk_transformer.py:102-110) as a `symbols_to_logits_fn` for tests/beam_oracle.py and tests/sampling_oracle.py."""
import torch

from oracle import restatement as R


def monotonic_padding(padding):
    """[B,T,T] 'padding' of the monotonic encoder: 1 where key j is padding or j > i.  restatement.encoder turns it into
    the bias FLOAT_MIN * padding, i.e. min(padding bias, lower-triangle bias) (transformer_encoder.py:119-123)."""
    T = padding.shape[1]
    tri = torch.ones(T, T, dtype=padding.dtype).triu(1)
    return torch.maximum(padding[:, None, :], tri[None])


def waitk_memory_bias(padding, Lq, k, t0=0):
    """[B,Lq,Tm] cross-attention bias of target positions t0..t0+Lq-1 with lag k: min(padding bias, wait-k bias), the
    wait-k bias being FLOAT_MIN outside band_part(ones, -1, k-1) (transformer_decoder.py:194-208, layer_utils.py:56-78).
    k = 0: the padding bias alone."""
    pad = R.input_padding_to_bias(padding)[:, None, :].expand(-1, Lq, -1)
    if not k:
        return pad
    Tm = padding.shape[1]
    i = torch.arange(t0, t0 + Lq)[:, None]
    j = torch.arange(Tm)[None, :]
    lag = torch.where(j < i + k, 0.0, R.FLOAT_MIN).to(padding.dtype)
    return torch.minimum(pad, lag[None])


def waitk_forward(P, cfg, src, src_padding, trg_input, k, monotonic=True):
    """The WaitkTransformer's teacher-forced logits (waitk_transformer.py:88-116) in the restatement's terms."""
    table = P["trg.emb"] if cfg.get("share_src_trg") else P["srcemb.emb"]
    emb = R.add_position(table[src])
    enc = R.encoder(P, emb, monotonic_padding(src_padding) if monotonic else src_padding, cfg["enc_layers"], cfg["heads"])
    dec_in = R.target_embed(P, trg_input)
    dec = R.decoder(P, dec_in, enc, waitk_memory_bias(src_padding, trg_input.shape[1], k), cfg["dec_layers"], cfg["heads"])
    return R.logits_layer(P, dec)


def waitk_greedy(P, cfg, src, src_padding, bos, eos, steps, k, unk=None, enc=None):
    """Greedy search of the wait-k model: step t sees the memory keys j < min(k + t, Tm); the self-attention is cached as in
    restatement.greedy_search.  `enc`: a given encoder memory instead of the monotonic encoding of `src`.  Returns ids
    [B, steps] (EOS after a row finishes) and the per-step logits."""
    if enc is None:
        table = P["trg.emb"] if cfg.get("share_src_trg") else P["srcemb.emb"]
        enc = R.encoder(P, R.add_position(table[src]), monotonic_padding(src_padding), cfg["enc_layers"], cfg["heads"])
    B = enc.shape[0]
    H, dh = cfg["heads"], cfg["d"] // cfg["heads"]
    caches = [dict(keys=torch.zeros(B, 0, H, dh, dtype=enc.dtype), values=torch.zeros(B, 0, H, dh, dtype=enc.dtype))
              for _ in range(cfg["dec_layers"])]
    ids = torch.full((B,), int(bos), dtype=torch.long)
    fin = torch.zeros(B, dtype=torch.bool)
    out, all_logits = [], []
    for t in range(steps):
        x = R.target_embed(P, ids, time=t).unsqueeze(1)
        y = R.decoder(P, x, enc, waitk_memory_bias(src_padding, 1, k, t0=t), cfg["dec_layers"], cfg["heads"], caches=caches)
        logits = R.logits_layer(P, y)[:, 0]
        all_logits.append(logits)
        lp = torch.log_softmax(logits, -1)
        if unk is not None:
            lp[:, unk] = R.FLOAT_MIN
        nxt = torch.where(fin, torch.full_like(ids, eos), lp.argmax(-1))
        fin = fin | (nxt == eos)
        out.append(nxt)
        ids = nxt
    return torch.stack(out, 1), torch.stack(all_logits, 1)


def lagged_bias(memory_bias, k, time):
    """[N,1,Tm] cross-attention bias of search step `time` from the additive padding bias [N,Tm]: the keys j >= k + time get
    FLOAT_MIN too (min, as the reference); k = 0: the padding bias alone."""
    if not k:
        return memory_bias[:, None, :]
    j = torch.arange(memory_bias.shape[1])
    lag = torch.where(j < k + int(time), 0.0, R.FLOAT_MIN).to(memory_bias.dtype)
    return torch.minimum(memory_bias, lag[None])[:, None, :]


def lagged_decoder_fn(P, cfg, k):
    """symbols_to_logits_fn(ids [N], cache, time) -> logits [N, V] of the cached decoder with lag k, over a cache dict(memory,
    memory_bias [N,Tm] additive, layers) as tests/sampling_oracle.py's; the searches tile and gather it per beam."""
    H = cfg["heads"]

    def symbols_to_logits_fn(ids, cache, time):
        x = R.target_embed(P, ids, time=time).unsqueeze(1)
        y = R.decoder(P, x, cache["memory"], lagged_bias(cache["memory_bias"], k, time), cfg["dec_layers"], H,
                      caches=cache["layers"])
        return R.logits_layer(P, y[:, 0])
    return symbols_to_logits_fn


def monotonic_text_cache(P, cfg, src, padding):
    """The search cache of the text model with a monotonic encoder: fp64 memory, its padding bias and empty layer caches."""
    table = P["trg.emb"] if cfg.get("share_src_trg") else P["srcemb.emb"]
    enc = R.encoder(P, R.add_position(table[src]), monotonic_padding(padding), cfg["enc_layers"], cfg["heads"])
    return given_memory_cache(cfg, enc, R.input_padding_to_bias(padding))


def given_memory_cache(cfg, memory, memory_bias):
    B, H, d = memory.shape[0], cfg["heads"], cfg["d"]
    layers = [dict(keys=torch.zeros(B, 0, H, d // H, dtype=torch.float64), values=torch.zeros(B, 0, H, d // H, dtype=torch.float64))
              for _ in range(cfg["dec_layers"])]
    return dict(memory=memory.double(), memory_bias=memory_bias.double(), layers=layers)

