"""Wait-k simultaneous translation on the device: forward / loss / gradient parity of a monotonic-encoder wait-k model with
the fp64 restatement (fp32 / fp16 / bf16, k = 1, 3 and k >= T, masks crossing 128-row tiles), the fused 16-bit attention
against the materialised path, a lag of k >= T as a bit-exact no-op in training and in every decoding kernel, greedy token
ids against the streaming agent's re-encoding loop, greedy (every step kernel), beam and top-k sampling token ids against
the fp64 searches with the lag on the fp32 and the 16-bit wide paths, and `train` / `predict` of the WaitkTranslation task."""
import functools
import os

import numpy as np
import pytest
import torch
import yaml

from neurst_b200 import cli
from neurst_b200 import decode as D
from neurst_b200 import metrics as MT
from neurst_b200.runtime import GraphedTrainStep, Runtime, make_config
from neurst_b200 import lib as L
from oracle import restatement as R
from tests import parity_utils as U
from tests.test_mt_gpu import TINY, _corpus
from tests import beam_oracle as BO
from tests import sampling_oracle as SO
from tests.waitk_oracle import (given_memory_cache, lagged_decoder_fn, monotonic_padding, monotonic_text_cache, waitk_forward,
                                waitk_greedy)

pytestmark = pytest.mark.gpu

TOL = {"fp32": (1e-4, 1e-4, 1e-3), "fp16": (5e-3, 2e-3, 4e-2), "bf16": (6e-2, 3e-2, 1.5e-1)}   # test_mt_gpu.py's
MT_S = dict(model="text", d=256, heads=4, enc_layers=6, dec_layers=6, ffn=2048, vocab=8192, src_vocab=8190)
B, T, LQ = 4, 150, 136          # both lengths cross a 128-row query / key tile


def _runtime(cfg, precision, monotonic=True, disable_fused=False):
    # deterministic: the fused FFN reduces in a fixed order, so that forward passes repeat bit for bit
    c = make_config(L.MODEL_TEXT, cfg["d"], cfg["heads"], cfg["ffn"], cfg["enc_layers"], cfg["dec_layers"], cfg["vocab"],
                    src_vocab=cfg["src_vocab"], precision=precision, label_smoothing=0.1, encoder_monotonic=monotonic,
                    disable_fused_attention=disable_fused, deterministic=True)
    return Runtime(c)


def _batch(seed):
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, MT_S["src_vocab"], (B, T), generator=g)
    lens = torch.tensor([T, 97, 131, 12])
    padding = (torch.arange(T)[None, :] >= lens[:, None]).float()
    V = MT_S["vocab"]
    trg = torch.randint(0, V, (B, LQ), generator=g)
    trg_input = torch.cat([torch.full((B, 1), V - 2, dtype=torch.long), trg[:, :-1]], 1)
    trg_length = torch.tensor([LQ, 80, 121, 33])
    return dict(src=src, src_padding=padding, trg_input=trg_input, trg=trg, trg_length=trg_length)


@functools.lru_cache(maxsize=None)
def _params():
    return R.init_params(dict(MT_S), seed=31, random_bias=True)


@functools.lru_cache(maxsize=None)
def _oracle(k):
    P, batch = _params(), _batch(32)
    P64 = {n: v.double().requires_grad_(True) for n, v in P.items()}
    logits = waitk_forward(P64, MT_S, batch["src"], batch["src_padding"].double(), batch["trg_input"], k)
    loss = R.reduce_loss(logits, batch["trg"], batch["trg_length"], 0.1)
    grads = dict(zip(P64, torch.autograd.grad(loss, list(P64.values()))))
    return logits.detach(), float(loss.detach()), grads


def _run(rt, k, backward=True):
    rt.ensure_grads().zero_()
    out = rt.run(dict(U.to_cuda(_batch(32)), training=False, seed=0, want_logits=True, wait_k=k), backward=backward)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("k", [1, 3, T])
@pytest.mark.parametrize("precision", ["fp32", "fp16", "bf16"])
def test_waitk_parity_with_the_fp64_restatement(precision, k):
    logits, loss, grads = _oracle(k)
    rt = _runtime(MT_S, precision)
    rt.load_parameters(_params())
    out = _run(rt, k)
    S = float(rt.loss_scale_state[0]) if rt.fp16 else 1.0
    e_logits = float((out["logits"].cpu().double() - logits).abs().max())
    e_loss = abs(float(out["loss"]) - loss)
    errs = sorted(((U.rel_err(rt.grad_view(n) / S, g), n) for n, g in grads.items()), reverse=True)
    print("\n[waitk %s k=%d] logits %.3e loss %.3e worst grads %s" % (precision, k, e_logits, e_loss,
                                                                      ", ".join("%s %.2e" % (n, e) for e, n in errs[:3])))
    tl, tloss, tg = TOL[precision]
    if precision == "fp32" and k < T:
        # the line printed above read 1.6e-3 (k = 1) and 2.0e-3 (k = 3) on enc.4.ffn on an H100 (700 W), logits within
        # 5e-6.  fp32 summation order alone reaches that size on this model: the restatement itself evaluated in fp32 on
        # the CPU differs from its fp64 evaluation by 1.6e-3 (dec.1.ffn, k = T).  A mask error would show in the logits:
        # the fp32 path's backward reads the stored probabilities, already masked.
        tg = 3e-3
    assert e_logits < tl and e_loss < tloss * max(1.0, abs(loss)) and errs[0][0] < tg, (e_logits, e_loss, errs[:4])


def test_fused_attention_with_the_offset_equals_the_materialised_path():
    outs = []
    for disable in (False, True):
        rt = _runtime(MT_S, "fp16", disable_fused=disable)
        rt.load_parameters(_params())
        out = _run(rt, 3)
        outs.append((out["logits"].cpu(), float(out["loss"]), {n: rt.grad_view(n).cpu().clone() for n in rt.table}))
    (l0, s0, g0), (l1, s1, g1) = outs
    assert float((l0 - l1).abs().max()) < 5e-3 and abs(s0 - s1) < 2e-3 * max(1.0, abs(s0))
    worst = max(U.rel_err(g0[n], g1[n]) for n in g0)
    assert worst < 4e-2, worst


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_training_lag_at_least_the_source_length_is_a_no_op(precision):
    """k >= T masks nothing: the logits are bit-identical to wait_k = 0.  The loss and the gradients are reduced with fp32
    atomics in arrival order (the loss sum, attention dQ, split-K weight gradients), so two runs at the same k already differ
    in the last bits: a lag's loss and gradients must stay within that run-to-run spread."""
    rt = _runtime(MT_S, precision)
    rt.load_parameters(_params())
    res = []
    for k in (0, 0, T, T + 7):
        out = _run(rt, k)
        res.append((out["logits"].cpu(), out["loss"].cpu(), rt.grads.cpu().clone()))
    spread = U.rel_err(res[1][2], res[0][2])
    loss_spread = float((res[1][1] - res[0][1]).abs())
    for other in res[1:]:
        assert torch.equal(other[0], res[0][0])
        assert float((other[1] - res[0][1]).abs()) <= max(4 * loss_spread, 1e-6 * float(res[0][1].abs()))
        assert U.rel_err(other[2], res[0][2]) <= max(4 * spread, 1e-6)


def test_graphed_step_follows_a_fresh_lag():
    """GraphedTrainStep reads k from a device word: a replay with a new k equals the eager step with that k."""
    rt = _runtime(MT_S, "fp16")
    rt.load_parameters(_params())
    batch = U.to_cuda(_batch(32))
    step = GraphedTrainStep(rt, B, T, LQ, wait_k=True).capture()
    losses = []
    for k in (1, 5, T):
        rt.ensure_grads().zero_()
        got = step(batch, seed=0, wait_k=k)
        g_graph = rt.grads.clone()
        rt.ensure_grads().zero_()
        want = rt.run(dict(batch, training=True, seed=0, wait_k=k), backward=True)
        torch.cuda.synchronize()
        # the loss sum and the fp16 gradients are reduced with atomics in arrival order: last-bit differences between two
        # runs (gradients: measured 2.7e-4 relative)
        assert abs(float(got["loss"]) - float(want["loss"])) < 1e-5 * abs(float(want["loss"])), k
        assert U.rel_err(g_graph, rt.grads) < 2e-3, k
        losses.append(float(got["loss"]))
    assert len(set(losses)) == 3            # each replay follows its own lag


# ------------------------------------------------------------------------------------------------ decoding
SMALL = dict(model="text", d=64, heads=4, enc_layers=2, dec_layers=2, ffn=128, vocab=96, src_vocab=77)
BOS, EOS, UNK = 94, 95, 93
MIN_GAP = 1e-4


@functools.lru_cache(maxsize=None)
def _small(rows):
    P = U.chaotic_decode_params(R.init_params(SMALL, seed=5, random_bias=True), 4.0, 5)
    g = torch.Generator().manual_seed(6)
    src = torch.randint(0, 76, (rows, 13), generator=g)
    lens = torch.randint(3, 14, (rows,), generator=g)
    lens[0] = 13
    src[torch.arange(rows), lens - 1] = 76                     # an EOS-like last token per row
    padding = (torch.arange(13)[None, :] >= lens[:, None]).float()
    return P, src, padding


@functools.lru_cache(maxsize=None)
def _small_runtime(precision):
    rt = _runtime(SMALL, precision)
    rt.load_parameters(_small(1)[0])
    return rt


def _searches(rt, inputs, k, shadow):
    kw = dict(use_shadow=shadow, wait_k=k)
    out = {}
    for g in (0, 1, 2):
        out["greedy%d" % g] = D.greedy_search(rt, inputs, BOS, EOS, UNK, 20, 8, 0, use_graph=bool(g), persistent=g == 2, **kw)[:2]
    rows = inputs["src"].shape[0]
    sub = {n: v[:max(1, rows // 4)] for n, v in inputs.items()}
    out["beam"] = D.beam_search(rt, sub, BOS, EOS, UNK, beam_size=4, length_penalty=0.6, maximum_decode_length=20,
                                extra_decode_length=8, **kw)[:3]
    out["sample"] = D.sampling_search(rt, sub, BOS, EOS, UNK, 4, 10, 1.0, 20, 8, 1, 77, **kw)[:2]
    torch.cuda.synchronize()
    return out


def _same(a, b, exact):
    if a.dtype in (torch.int64, torch.int32) or exact:
        return torch.equal(a, b)
    return torch.allclose(a, b, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("rows, precision", [(8, "fp32"), (24, "fp16")])
def test_decoding_lag_at_least_the_memory_length_is_a_no_op(rows, precision):
    """k >= Tm: every search's token ids equal wait_k = 0's.  The wide 16-bit step (above 8 rows) uses no floating-point
    atomics, so there the scores and step logits are bit-identical too; the fp32 step of at most 8 rows sums the context
    and the projections with shared- and global-memory atomics, whose order varies from run to run."""
    _, src, padding = _small(rows)
    inputs = dict(src=src, src_padding=padding)
    rt = _small_runtime(precision)
    shadow = precision != "fp32"
    base = _searches(rt, inputs, 0, shadow)
    for k in (13, 40):
        got = _searches(rt, inputs, k, shadow)
        for name in base:
            assert all(_same(a, b, shadow) for a, b in zip(base[name], got[name])), (name, k)
    enc, bias = D.encode(rt, inputs)
    logits = []
    for k in (0, 13):
        cache = D.create_decoding_cache(rt, enc, bias, 20, use_shadow=shadow, wait_k=k)
        logits.append(torch.stack([D.decoder_step_logits(rt, torch.full((rows,), BOS), cache, t) for t in range(4)]))
    assert _same(logits[0], logits[1], shadow)


def _check_greedy(ids, ref_ids, ref_logits):
    """Token ids equal row by row up to the first fp64 near-tie (top-2 gap below MIN_GAP) of that row."""
    top2 = ref_logits.log_softmax(-1).topk(2, -1).values
    gap = top2[..., 0] - top2[..., 1]
    for r in range(ids.shape[0]):
        n = next((t for t in range(ref_ids.shape[1]) if gap[r, t] < MIN_GAP), ref_ids.shape[1])
        assert n > 2, "near-tie at the start of row %d" % r
        assert ids[r, :n].tolist() == ref_ids[r, :n].tolist(), (r, ids[r].tolist(), ref_ids[r].tolist())


def _fp64_search(search, k, P64, cache, B):
    """The fp64 search with lag k over the restated cached decoder (tests/waitk_oracle.py): tests/beam_oracle.py for greedy
    (beam 1, the reference's greedy) and beam 4, tests/sampling_oracle.py for top-k sampling (4 samples, top_k 10).  Returns
    the reference ids and the smallest margin of a rounding-sensitive decision met on the way."""
    fn = lagged_decoder_fn(P64, SMALL, k)
    bos = torch.full((B,), BOS, dtype=torch.long)
    with torch.no_grad():
        if search == "sample":
            r = SO.sampling_search(fn, bos, cache, EOS, UNK, sample_num=4, top_k=10, maximum_decode_length=20,
                                   extra_decode_length=8, minimum_decode_length=2, encoder_inputs_maxlen=13, seed=77)
            return r["ids"], min(r["draw_margin"], r["threshold_margin"])
        r = BO.beam_search(fn, bos, cache, EOS, UNK, 1 if search == "greedy" else 4, 0.6, 1, 20, 8, 0, encoder_inputs_maxlen=13)
        return r["hypotheses"], r["gap"]


def _device_search(rt, search, inputs, cache, shadow, use_graph=1):
    kw = dict(use_shadow=shadow, cache=cache)
    if search == "sample":
        return D.sampling_search(rt, inputs, BOS, EOS, UNK, 4, 10, 1.0, 20, 8, 2, 77, **kw)[0]
    if search == "beam":
        return D.beam_search(rt, inputs, BOS, EOS, UNK, beam_size=4, length_penalty=0.6, maximum_decode_length=20,
                             extra_decode_length=8, **kw)[0]
    return D.greedy_search(rt, inputs, BOS, EOS, UNK, 20, 8, 0, use_graph=use_graph > 0, persistent=use_graph == 2, **kw)[0]


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("search, use_graph", [("greedy", 0), ("greedy", 1), ("greedy", 2), ("beam", 1), ("sample", 1)])
def test_fp32_searches_with_a_lag_equal_the_fp64_searches(search, use_graph, k):
    """fp32 weights, at most 8 rows (attn_step_kernel, its beam variant, and the persistent kernel's attn_item): the whole
    model, monotonic encoder included, against the fp64 searches with the lag k + t at step t."""
    B = 6 if search == "greedy" else 2
    P, src, padding = _small(B)
    P64 = {n: v.double() for n, v in P.items()}
    ref, margin = _fp64_search(search, k, P64, monotonic_text_cache(P64, SMALL, src, padding.double()), B)
    assert margin > MIN_GAP, "near-tie in the oracle's search (%.2e)" % margin
    rt = _small_runtime("fp32")
    cache = D.create_decoding_cache(rt, *D.encode(rt, dict(src=src, src_padding=padding)), 20,
                                    beam=1 if search == "greedy" else 4, wait_k=k)
    ids = _device_search(rt, search, None, cache, False, use_graph)
    torch.cuda.synchronize()
    if search == "greedy":
        assert int(L.load().b200st_greedy_used_graph()) == use_graph
    assert torch.equal(ids.cpu(), ref), (ids.cpu().tolist(), ref.tolist())


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("search", ["greedy", "beam", "sample"])
def test_wide_searches_with_a_lag_equal_the_fp64_searches_on_rounded_weights(search, k):
    """More than 8 rows (rows_cross_attn_kernel with 1 or 4 rows per utterance) on a given ragged memory: the fp64 searches
    read the same 16-bit-rounded weights the shadow decoder reads (test_decode_shadow_gpu.py)."""
    from tests.test_decode_shadow_gpu import ragged_memory, shadow_rounded
    B = 16 if search == "greedy" else 4
    memory, bias = ragged_memory(SMALL, B, 13, seed=9)
    ref, margin = _fp64_search(search, k, shadow_rounded(_small(1)[0], torch.float16), given_memory_cache(SMALL, memory, bias), B)
    assert margin > MIN_GAP, "near-tie in the oracle's search (%.2e)" % margin
    rt = _small_runtime("fp16")
    cache = D.create_decoding_cache(rt, memory.cuda(), bias.cuda(), 20, use_shadow=True, beam=1 if search == "greedy" else 4,
                                    wait_k=k)
    ids = _device_search(rt, search, None, cache, True)
    torch.cuda.synchronize()
    assert torch.equal(ids.cpu(), ref), (ids.cpu().tolist(), ref.tolist())


def test_greedy_equals_the_streaming_agent():
    """The agent (simul_trans_text_agent.py) re-encodes the source read so far at every step: min(k + t, |x|) tokens of a
    source of |x| tokens with its EOS.  With a monotonic encoder this is the one-shot encoding with keys j >= k + t hidden."""
    P, src, padding = _small(6)
    P64 = {n: v.double() for n, v in P.items()}
    k, steps = 2, 20
    lens = (1 - padding).sum(-1).long()
    stream = torch.full((6, steps), EOS, dtype=torch.long)
    H, dh = SMALL["heads"], SMALL["d"] // SMALL["heads"]
    with torch.no_grad():
        for r in range(6):
            # the agent's decoder keeps its self-attention cache across steps (incremental decoding); only the source
            # encoding grows
            caches = [dict(keys=torch.zeros(1, 0, H, dh, dtype=torch.float64), values=torch.zeros(1, 0, H, dh, dtype=torch.float64))
                      for _ in range(SMALL["dec_layers"])]
            last = torch.full((1,), BOS, dtype=torch.long)
            for t in range(steps):
                n = min(k + t, int(lens[r]))
                s = src[r:r + 1, :n]
                pad = torch.zeros(1, n, dtype=torch.float64)
                enc = R.encoder(P64, R.add_position(P64["srcemb.emb"][s]), monotonic_padding(pad), SMALL["enc_layers"], H)
                x = R.target_embed(P64, last, time=t).unsqueeze(1)
                y = R.decoder(P64, x, enc, R.input_padding_to_bias(pad), SMALL["dec_layers"], H, caches=caches)
                lp = torch.log_softmax(R.logits_layer(P64, y)[0, -1], -1)
                lp[UNK] = R.FLOAT_MIN
                nxt = int(lp.argmax())
                stream[r, t] = nxt
                if nxt == EOS:
                    break
                last = torch.tensor([nxt])
        ref_ids, ref_logits = waitk_greedy(P64, SMALL, src, padding.double(), BOS, EOS, steps, k, UNK)
    _check_greedy(stream, ref_ids, ref_logits)
    ids, _ = D.greedy_search(_small_runtime("fp32"), dict(src=src, src_padding=padding), BOS, EOS, UNK, 20, 8, 0, wait_k=k)[:2]
    torch.cuda.synchronize()
    _check_greedy(ids.cpu()[:, :steps], stream, ref_logits)


# ------------------------------------------------------------------------------------------------ train / predict
@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    root = tmp_path_factory.mktemp("waitk")
    (root / "vocab.src").write_text("".join("s%d\t1\n" % i for i in range(85)))
    (root / "vocab.trg").write_text("".join("t%d\t1\n" % i for i in range(40)) + "x\n" + "".join("p%d\n" % i for i in range(4)))
    return root, _corpus(root, 600, 1, "train"), _corpus(root, 40, 2, "dev")


def _plan(corpus, model_dir, steps, entry="trainer", **extra):
    root, (ts, tt), (ds, dt) = corpus
    cfg = {"entry.class": entry, "task.class": "WaitkTranslation", "dtype": "float16", "model_dir": str(model_dir),
           "hparams_set": "waitk_transformer_s", "model.params": dict(TINY),
           "entry.params": {"train_steps": steps, "save_checkpoint_steps": 4, "summary_steps": 100},
           "task.params": {"batch_by_tokens": True, "batch_size": 2000, "max_src_len": 20, "max_trg_len": 30,
                           "src_data_pipeline.params": {"vocab_path": str(root / "vocab.src")},
                           "trg_data_pipeline.params": {"vocab_path": str(root / "vocab.trg")}},
           "dataset.class": "ParallelTextDataset",
           "dataset.params": {"src_file": ts, "trg_file": tt, "data_is_processed": True}}
    if entry == "trainer":
        cfg["task.params"]["wait_k"] = "[1, 3, 5]"
        cfg["validator.class"] = "SeqGenerationValidator"
        cfg["validator.params"] = {"eval_dataset": "ParallelTextDataset",
                                   "eval_dataset.params": {"src_file": ds, "trg_file": dt, "data_is_processed": True},
                                   "eval_batch_size": 16, "eval_steps": 4, "eval_criterion": "label_smoothed_cross_entropy",
                                   "eval_search_method": "beam_search",
                                   "eval_search_method.params": {"beam_size": 2, "maximum_decode_length": 30},
                                   "eval_metric": "tok_bleu", "eval_top_checkpoints_to_keep": 2}
    else:
        cfg["dataset.params"] = {"src_file": ds, "data_is_processed": True}
    cfg.update(extra)
    return cli.resolve(cfg)


@pytest.fixture(scope="module")
def trained(corpus, tmp_path_factory):
    model_dir = tmp_path_factory.mktemp("waitk_run") / "m"
    first = cli.train(_plan(corpus, model_dir, 8))
    second = cli.train(_plan(corpus, model_dir, 12))
    return model_dir, first, second


def test_waitk_train_validates_resumes_and_records_wait_k(trained):
    model_dir, first, second = trained
    assert first["global_step"] == 8 and second["global_step"] == 12
    assert np.isfinite(first["loss"]) and np.isfinite(second["loss"])
    assert [r["step"] for r in first["validations"]] == [4, 8] and [r["step"] for r in second["validations"]] == [12]
    assert all(r["metric"] and r["loss"] for r in first["validations"] + second["validations"])
    with open(os.path.join(model_dir, cli.MODEL_CONFIGS)) as f:
        configs = yaml.safe_load(f)
    assert configs["model.class"] == "WaitkTransformer" and configs["task.class"] == "WaitkTranslation"
    assert configs["task.params"]["wait_k"] == [1, 3, 5] and configs["model.params"]["encoder.attention_monotonic"] is True


def test_waitk_predict_batch_size_lag_override_and_latency(corpus, trained, tmp_path):
    """On a checkpoint whose decoder makes the hypotheses depend on the context (parity_utils.chaotic_decode_params: a model
    trained for a few steps emits the same tokens whatever the lag)."""
    from neurst_b200 import checkpoints as CK
    plan = _plan(corpus, trained[0], 0, entry="predict")
    model = cli._build_model(plan).init_parameters(7)
    model.load_parameters(U.chaotic_decode_params({n: v.cpu() for n, v in model.named_parameters().items()}, 4.0, 7))
    model_dir = tmp_path / "chaotic"
    cli.write_model_configs(dict(plan, model_dir=str(model_dir)))
    CK.save_npz(model.runtime, str(model_dir / "ckpt-1.npz"))
    outs, results = [], []
    for bs, k in ((16, None), (32, None), (16, 9)):
        extra = {"batch_size": bs, "output_file": str(tmp_path / ("hyp%d_%s.txt" % (bs, k)))}
        if k is not None:
            extra["wait_k"] = k
        plan = _plan(corpus, model_dir, 0, entry="predict", **extra)
        assert plan["wait_k"] == ([1, 3, 5] if k is None else k)
        results.append(cli.predict(plan))
        outs.append(open(extra["output_file"]).read().splitlines())
    assert outs[0] == outs[1] and any(outs[0])
    assert outs[2] != outs[0]
    # the logged latency is metrics' on the written hypotheses (model tokens: the vocabulary has no BPE marks here)
    srcs = open(corpus[2][0]).read().splitlines()
    for out, res, k in ((outs[0], results[0], 1), (outs[2], results[2], 9)):
        want = MT.corpus_waitk_latency(k, [(len(s.split()), len(h.split())) for s, h in zip(srcs, out)])
        assert res["latency"] == pytest.approx(want)
