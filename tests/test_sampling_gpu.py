"""Top-k / nucleus sampling on the device (b200st_sampling_search through decode.sampling_search, the model and `predict`;
b200st_sample_logits on fixed logits) against the restated search of tests/sampling_oracle.py, which replays the same keyed
Philox draws in fp64: token ids IDENTICAL, lengths equal, log-probabilities to 1e-4 relative.  Every exact comparison first
asserts that the oracle met no near-tie (every draw's u * W farther than 1e-4 relative from a cumulative boundary, every
threshold farther than 1e-4 from the next value or from p), so a mismatch cannot come from rounding."""
import functools

import numpy as np
import pytest
import torch

from neurst_b200 import decode as D
from neurst_b200 import lib as L
from tests import sampling_oracle as SO
from tests.test_beam_search_gpu import BOS, EOS, SMALL, UNK, _runtime, _small
from tests.test_decode_shadow_gpu import DTYPES, _cache, _chaotic, shadow_rounded
from tests.test_decode_shadow_gpu import _runtime as _shadow_runtime

pytestmark = pytest.mark.gpu

MIN_GAP = 1e-4


def _check(ref, ids, logprob, length):
    assert ref["draw_margin"] > MIN_GAP and ref["threshold_margin"] > MIN_GAP, \
        "near-tie in the oracle's search (draw %.2e, threshold %.2e): pick another case" % (ref["draw_margin"], ref["threshold_margin"])
    assert torch.equal(ids.cpu(), ref["ids"]), [(i, a, b) for i, (a, b) in enumerate(zip(ids.cpu().view(-1).tolist(),
                                                ref["ids"].view(-1).tolist())) if a != b][:5]
    assert torch.equal(length.cpu().long(), ref["length"])
    assert torch.allclose(logprob.cpu().double(), ref["logprob"], rtol=1e-4, atol=1e-5), (logprob.tolist(), ref["logprob"].tolist())


# ---- narrow path: the small model of test_beam_search_gpu, fp32 weights, 2 utterances ---------------------------------------
# (sample_num, top_k, top_p) -> (sampling seed, maximum_decode_length): the first seeds whose fp64 search keeps both margins
# above 1e-4 (CPU; at 24 steps no seed of 1-59 did for 4 samples without a filter or with top_p 0.9)
NARROW = {(1, 0, 1.0): (1, 24), (1, 5, 1.0): (1, 24), (1, 0, 0.9): (38, 24),
          (4, 0, 1.0): (2, 12), (4, 5, 1.0): (1, 24), (4, 0, 0.9): (48, 8)}
MODEL_SEED, MIN_LEN = 4, 3


@functools.lru_cache(maxsize=None)
def _narrow_reference(sample_num, top_k, top_p):
    seed, max_len = NARROW[sample_num, top_k, top_p]
    P, src, lens = _small(MODEL_SEED)
    return SO.speech_sampling_search(P, SMALL, src, lens, BOS, EOS, UNK, sample_num=sample_num, top_k=top_k, top_p=top_p,
                                     maximum_decode_length=max_len, extra_decode_length=8, minimum_decode_length=MIN_LEN, seed=seed)


@pytest.mark.parametrize("sample_num", [1, 4])
@pytest.mark.parametrize("top_k,top_p", [(0, 1.0), (5, 1.0), (0, 0.9)])
@pytest.mark.parametrize("use_graph", [True, False])
def test_sampling_token_ids_exact_small(sample_num, top_k, top_p, use_graph):
    seed, max_len = NARROW[sample_num, top_k, top_p]
    ref = _narrow_reference(sample_num, top_k, top_p)
    _, src, lens = _small(MODEL_SEED)
    ids, logprob, length = D.sampling_search(_runtime(MODEL_SEED), dict(src=src, src_length=lens), BOS, EOS, UNK,
                                             sample_num=sample_num, top_k=top_k, top_p=top_p, maximum_decode_length=max_len,
                                             extra_decode_length=8, minimum_decode_length=MIN_LEN, seed=seed, use_graph=use_graph)
    torch.cuda.synchronize()
    _check(ref, ids, logprob, length)
    assert len(set(ids.view(-1).tolist())) >= 8, "degenerate samples: the test would not exercise the draws"


# ---- wide path: 16-bit shadow weights, 16 x 4 and 64 x 4 rows, against the fp64 decoder on the rounded weights ------------
# utterances -> (sampling seed, maximum_decode_length); top_k 5, minimum length 2, the memory of test_decode_rows_gpu's
# greedy case (seed 2)
WIDE = {("fp16", 16): (2, 8), ("fp16", 64): (1, 4), ("bf16", 16): (3, 8), ("bf16", 64): (1, 4)}


@functools.lru_cache(maxsize=None)
def _wide_reference(precision, B):
    seed, max_len = WIDE[precision, B]
    P, memory, bias = _chaotic("small", B, 61, 4.0, 2)
    return SO.decoder_sampling_search(shadow_rounded(P, DTYPES[precision]), SMALL, memory, bias, 94, 95, 93, sample_num=4, top_k=5,
                                      maximum_decode_length=max_len, extra_decode_length=8, minimum_decode_length=2, seed=seed)


def _wide(precision, B, row_offset=0, rows=None, use_graph=True, **kw):
    seed, max_len = WIDE[precision, B]
    P, memory, bias = _chaotic("small", B, 61, 4.0, 2)
    if rows is not None:
        memory, bias = memory[rows], bias[rows]
    rt = _shadow_runtime(SMALL, precision, P)
    out = D.sampling_search(rt, None, 94, 95, 93, sample_num=4, top_k=kw.get("top_k", 5), top_p=kw.get("top_p", 1.0),
                            maximum_decode_length=max_len, extra_decode_length=8, minimum_decode_length=2, seed=seed,
                            row_offset=row_offset, use_shadow=True, use_graph=use_graph,
                            cache=_cache(rt, memory, bias, max_len, beam=4))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("B", [16, 64])
def test_wide_sampling_token_ids_exact(precision, B):
    ref = _wide_reference(precision, B)
    _check(ref, *_wide(precision, B))


def test_wide_sampling_is_bit_reproducible_and_independent_of_the_call_split():
    """Two calls give bit-identical output; the 64 utterances x 4 samples as one 256-row call and as two 128-row calls with
    row offsets 0 and 128 give identical ids."""
    a, b = _wide("fp16", 64, top_k=0, top_p=0.9), _wide("fp16", 64, top_k=0, top_p=0.9)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    first = _wide("fp16", 64, rows=slice(0, 32), top_k=0, top_p=0.9)
    second = _wide("fp16", 64, row_offset=128, rows=slice(32, 64), top_k=0, top_p=0.9)
    assert torch.equal(a[0], torch.cat([first[0], second[0]])) and torch.equal(a[2], torch.cat([first[2], second[2]]))
    assert torch.equal(a[1], torch.cat([first[1], second[1]]))
    assert len(set(a[0].view(-1).tolist())) >= 8


# ---- top_k 1 and a tiny top_p are the greedy search -----------------------------------------------------------------------
@pytest.mark.parametrize("top_k,top_p", [(1, 1.0), (0, 1e-6)])
def test_top1_is_the_greedy_search(top_k, top_p):
    _, src, lens = _small(MODEL_SEED)
    rt = _runtime(MODEL_SEED)
    inputs = dict(src=src, src_length=lens)
    g_ids, g_lp, g_len = D.greedy_search(rt, inputs, BOS, EOS, UNK, maximum_decode_length=24, extra_decode_length=8)
    ids, lp, length = D.sampling_search(rt, inputs, BOS, EOS, UNK, top_k=top_k, top_p=top_p, maximum_decode_length=24,
                                        extra_decode_length=8)
    torch.cuda.synchronize()
    assert torch.equal(ids, g_ids) and torch.equal(length, g_len)
    # the log-probabilities differ by UNK's share: the sampling search masks UNK in the logits before its softmax
    # (sampling.py:48-73), the beam search after its log_softmax (beam_search.py:128-138)
    assert bool((lp >= g_lp - 1e-5).all()) and float((lp - g_lp).abs().max()) < 0.1, (lp.tolist(), g_lp.tolist())
    # the wide step: 64 utterances of test_decode_rows_gpu's greedy case, sample_num 1 = 64 rows
    P, memory, bias = _chaotic("small", 64, 61, 4.0, 2)
    rt = _shadow_runtime(SMALL, "fp16", P)
    g = D.greedy_search(rt, None, 94, 95, 93, maximum_decode_length=12, extra_decode_length=8, use_shadow=True,
                        cache=_cache(rt, memory, bias, 12))
    s = D.sampling_search(rt, None, 94, 95, 93, top_k=top_k, top_p=top_p, maximum_decode_length=12, extra_decode_length=8,
                          use_shadow=True, cache=_cache(rt, memory, bias, 12))
    torch.cuda.synchronize()
    assert torch.equal(s[0], g[0]) and torch.equal(s[2], g[2])
    assert len(set(s[0].view(-1).tolist())) >= 8


# ---- b200st_sample_logits on fixed logits ---------------------------------------------------------------------------------
def _draws(z, n, **kw):
    """n draws from each row of z (rows repeated with consecutive row offsets) -> ids [n, rows]."""
    rows = z.shape[0]
    zz = z.float().cuda().repeat(n, 1)
    return D.sample_logits(zz, **kw).cpu().view(n, rows)


def test_top_k_keeps_ties_and_draws_nothing_else():
    z = torch.full((1, 64), -2.0)
    z[0, 10], z[0, 3], z[0, 40], z[0, 41], z[0, 63] = 3.0, 2.0, 1.0, 1.0, 1.0       # 3rd largest value 1.0, held three times
    z[0, 20] = 0.5
    got = _draws(z, 4096, top_k=3, seed=11)
    assert set(got.view(-1).tolist()) == {10, 3, 40, 41, 63}
    got = _draws(z, 4096, top_k=1, seed=11)
    assert set(got.view(-1).tolist()) == {10}


@pytest.mark.parametrize("p", [0.3, 0.6, 0.9, 0.99, 0.999, 0.9995])
def test_top_p_kept_set_matches_the_restatement(p):
    g = torch.Generator().manual_seed(5)
    z = torch.randn(1, 24, generator=g, dtype=torch.float64) * 1.5
    z[0, 7] = z[0, 2]                                                                  # a tie
    keep, margin = SO.filter_keep(z, top_p=p)
    assert margin > MIN_GAP, margin
    probs = torch.softmax(z, -1)[0]
    got = set(_draws(z, 20000, top_p=p, seed=3).view(-1).tolist())
    kept = set(torch.nonzero(keep[0]).view(-1).tolist())
    assert got <= kept and {v for v in kept if probs[v] > 1e-3} <= got, (sorted(got), sorted(kept))
    assert (7 in kept) == (2 in kept)


@pytest.mark.parametrize("V", [8192, 32768])
@pytest.mark.parametrize("top_k,top_p", [(0, 1.0), (10, 1.0), (0, 0.9)])
def test_draws_match_the_restated_draw_at_large_vocabularies(V, top_k, top_p):
    """Every row's id equals the restated draw (the same Philox uniform, fp64 running sums) where that draw is not within
    1e-4 of a boundary; the rows' logits differ, so the filter's threshold is found anew for each.  With thousands of kept
    tokens the cumulative boundaries lie ~1e-4 apart, so about a quarter of the rows are left out of the exact comparison."""
    rows = 256
    g = torch.Generator().manual_seed(V + top_k)
    z = torch.randn(rows, V, generator=g, dtype=torch.float64) * 3.0
    z32 = z.float()
    ids = D.sample_logits(z32.cuda(), top_k=top_k, top_p=top_p, seed=99, row_offset=1000, step=7).cpu()
    z64 = z32.double()
    keep, margin = SO.filter_keep(z64, top_k=top_k, top_p=top_p)
    u = SO.uniforms(99, 7, np.arange(rows, dtype=np.uint64) + np.uint64(1000))
    w = torch.where(keep, torch.exp(z64 - z64.max(-1, keepdim=True).values), torch.zeros_like(z64))
    cum = torch.cumsum(w, -1)
    target = torch.as_tensor(u).unsqueeze(1) * cum[:, -1:]
    want = (cum > target).to(torch.int64).argmax(-1)
    near = ((cum - target).abs() / cum[:, -1:]).min(-1).values <= MIN_GAP
    assert int(near.sum()) <= rows // 2, int(near.sum())
    assert bool(keep.gather(1, ids.unsqueeze(1)).all()), "a filtered-out token was drawn"
    assert torch.equal(ids[~near], want[~near]), [(i, int(a), int(b)) for i, (a, b) in enumerate(zip(ids, want)) if a != b][:5]


@pytest.mark.parametrize("top_k,top_p", [(0, 1.0), (5, 1.0), (0, 0.8)])
def test_frequencies_follow_the_filtered_softmax(top_k, top_p):
    """Fixed seed, 40000 keys over one row of logits: a chi-square test against the filtered softmax (deterministic)."""
    from scipy.stats import chisquare
    z = torch.tensor([[2.0, 1.5, 1.5, 1.0, 0.5, 0.0, -0.5, -1.0, 0.7, 1.2]], dtype=torch.float64)
    keep, _ = SO.filter_keep(z, top_k=top_k, top_p=top_p)
    w = torch.where(keep, torch.exp(z - z.max()), torch.zeros_like(z))[0]
    probs = (w / w.sum()).numpy()
    n = 40000
    got = _draws(z, n, top_k=top_k, top_p=top_p, seed=2024).view(-1).numpy()
    counts = np.bincount(got, minlength=z.shape[1])
    assert counts[probs == 0].sum() == 0
    stat, pval = chisquare(counts[probs > 0], probs[probs > 0] * n)
    print("\n[sampling chi-square top_k %d top_p %.2f] statistic %.2f, p %.3g" % (top_k, top_p, stat, pval))
    assert pval > 1e-4, (counts.tolist(), (probs * n).round(1).tolist())


# ---- invalid arguments are refused before anything is launched ------------------------------------------------------------
def test_invalid_arguments_raise_before_any_launch():
    _, src, lens = _small(MODEL_SEED)
    rt = _runtime(MODEL_SEED)
    enc, bias = D.encode(rt, dict(src=src, src_length=lens))
    cache = D.create_decoding_cache(rt, enc, bias, 24, beam=4)
    short = D.create_decoding_cache(rt, enc, bias, 8, beam=2)
    torch.cuda.synchronize()
    before = L.launch_count()
    kw = dict(maximum_decode_length=24, extra_decode_length=8)
    with pytest.raises(NotImplementedError, match="top_k > 0 and top_p < 1"):
        D.sampling_search(rt, None, BOS, EOS, UNK, sample_num=4, top_k=5, top_p=0.9, cache=cache, **kw)
    with pytest.raises(ValueError, match="minimum_decode_length"):
        D.sampling_search(rt, None, BOS, EOS, UNK, sample_num=4, minimum_decode_length=24, cache=cache, **kw)
    with pytest.raises(L.B200STError, match="top_k"):
        D.sampling_search(rt, None, BOS, EOS, UNK, sample_num=4, top_k=-1, cache=cache, **kw)
    with pytest.raises(L.B200STError, match="exceeds the vocabulary"):
        D.sampling_search(rt, None, BOS, EOS, UNK, sample_num=4, top_k=97, cache=cache, **kw)
    with pytest.raises(L.B200STError, match="top_p"):
        D.sampling_search(rt, None, BOS, EOS, UNK, sample_num=4, top_p=float("nan"), cache=cache, **kw)
    with pytest.raises(L.B200STError, match="cache length"):
        D.sampling_search(rt, None, BOS, EOS, UNK, sample_num=2, cache=short, **kw)
    cache.state.B = 3                                                  # 3 x 4 rows with the fp32 weights
    with pytest.raises(L.B200STError, match="rows"):
        D.sampling_search(rt, None, BOS, EOS, UNK, sample_num=4, cache=cache, **kw)
    with pytest.raises(L.B200STError, match="sample_num"):
        D.sampling_search(rt, dict(src=src, src_length=lens), BOS, EOS, UNK, sample_num=9, **kw)
    with pytest.raises(L.B200STError, match="rows"):
        D.sampling_search(rt, dict(src=src, src_length=lens), BOS, EOS, UNK, sample_num=8, **kw)
    z = torch.zeros(2, 16, device="cuda")
    with pytest.raises(L.B200STError, match="exceeds the vocabulary"):
        D.sample_logits(z, top_k=17)
    with pytest.raises(L.B200STError, match="null"):
        L.check(L.load().b200st_sample_logits(None, 2, 16, 0, 1.0, 0, 0, 0, None, L._stream()))
    assert L.launch_count() == before
    torch.cuda.synchronize()


# ---- predict through the entry --------------------------------------------------------------------------------------------
def test_predict_with_top_sampling_through_the_entry(tmp_path):
    import os

    from neurst_b200 import cli
    from tests import test_cli as T
    T._write_dataset(tmp_path, vocab=93)
    y = T._write_yaml(tmp_path, data=str(tmp_path / "train.tfrecords"), n_tokens=93)
    tiny = ["--model.params.encoder.num_layers", "2", "--model.params.decoder.num_layers", "2",
            "--model.params.encoder.hidden_size", "128", "--model.params.decoder.hidden_size", "128", "--model.params.modality.dim", "128",
            "--model.params.encoder.num_attention_heads", "2", "--model.params.decoder.num_attention_heads", "2",
            "--model.params.encoder.filter_size", "256", "--model.params.decoder.filter_size", "256",
            "--model.params.modality.source.channels", "64"]
    common = ["--model_dir", str(tmp_path / "model"), "--task.params.batch_size", "3000", "--task.params.max_src_len", "400",
              "--task.params.max_trg_len", "24", "--task.params.min_src_bucket_boundary", "128",
              "--task.params.experimental_frame_transcript_ratio", "20", "--save_checkpoint_steps", "3", "--summary_steps", "2"] + tiny
    assert cli.main(["--config_paths", y] + common + ["--train_steps", "4"])["global_step"] == 4
    one = tmp_path / "one"
    one.mkdir()
    os.link(str(tmp_path / "train.tfrecords-00000-of-00003"), str(one / "train.tfrecords-00000-of-00001"))
    texts = {}
    for bs in (16, 32):
        extra = tmp_path / ("bs%d.yml" % bs)
        extra.write_text("batch_size: %d\n" % bs)
        out = str(tmp_path / ("samples_%d.txt" % bs))
        res = cli.main(["--config_paths", y + "," + str(extra)] + common + [
            "--entry.class", "predict", "--output_file", out, "--dataset.params.data_path", str(one / "train.tfrecords"),
            "--search_method", "top_sampling", "--search_method.params.sample_num", "2", "--search_method.params.top_p", "0.9",
            "--search_method.params.maximum_decode_length", "12"])
        assert res["n_hypotheses"] == 140                              # two lines per utterance
        texts[bs] = open(out, encoding="utf-8").read()
    lines = texts[16].split("\n")
    assert len(lines) == 141 and all(all(t.startswith("tok") or t == "<UNK>" for t in l.split()) for l in lines[:-1])
    assert texts[16] == texts[32]
    torch.cuda.synchronize()
