"""Ensemble decoding on the device (b200st_ensemble_beam_search through decode.ensemble_beam_search, the ensemble model and
`predict`) against the restated reference search (tests/beam_oracle.py, unchanged) over an fp64 ensemble: its
symbols_to_logits_fn returns the mixture log(sum_m w_m softmax(z_m)) of the members' oracle decoders, and its cache is the
list of the members' caches (beam_oracle tiles and gathers lists like any other cache).  log_softmax of that normalised
log-probability vector is the identity, so the oracle search runs on the mixture exactly as the reference's
sequence_beam_search does (beam_search.py:97-115).  Every token-exact comparison first checks the oracle's gap guard."""
import ctypes as C
import functools
import math
import os

import pytest
import torch

from neurst_b200 import decode as D
from neurst_b200 import lib as L
from oracle import restatement as R
from tests import beam_oracle as BO
from tests import parity_utils as U
from tests.test_beam_search_gpu import BOS, EOS, MIN_GAP, SMALL, UNK, _check, _small
from tests.test_decode_shadow_gpu import DTYPES, ragged_memory, shadow_rounded

pytestmark = pytest.mark.gpu

# a second architecture on the same vocabulary: wider, more heads per model width and one more decoder layer
WIDE = dict(SMALL, d=128, heads=4, dec_layers=3, ffn=256)
MAX_LEN, EXTRA = 16, 8
# The members' mixture is smoother than either member, and the fp64 search meets near-ties sooner: with members 4 and 7 (the
# single-model tests' seeds) the 2 x 4 case at 1/len scores has a gap of 2e-5.  Seeds 6 and 10 keep every case of the
# two-member test above the 1e-4 guard at 16 steps (CPU: smallest gap 1.7e-4).
TWO = ((6, False), (10, False))


# ---- the fp64 oracle ---------------------------------------------------------------------------------------------------------
def _member_fn(P, cfg):
    def fn(ids, cache, time):
        x = R.target_embed(P, ids, time=time).unsqueeze(1)
        y = R.decoder(P, x, cache["memory"], cache["memory_bias"], cfg["dec_layers"], cfg["heads"], caches=cache["layers"])
        return R.logits_layer(P, y[:, 0])
    return fn


def _member_cache(cfg, memory, bias):
    B, H, d = memory.shape[0], cfg["heads"], cfg["d"]
    layers = [dict(keys=torch.zeros(B, 0, H, d // H, dtype=torch.float64), values=torch.zeros(B, 0, H, d // H, dtype=torch.float64))
              for _ in range(cfg["dec_layers"])]
    return dict(memory=memory.double(), memory_bias=bias.double(), layers=layers)


def _speech_memory(P, cfg, src, lens):
    """The oracle's encoder (fp64): memory [B, T', d] and its additive bias."""
    emb = R.add_position(R.conv_subsample(P, src.double()))
    padding = R.input_length_to_padding(R.length_after_conv(lens), emb.shape[1], emb.dtype)
    return R.encoder(P, emb, padding, cfg["enc_layers"], cfg["heads"]), R.input_padding_to_bias(padding)


def ensemble_oracle(members, weights, beam, alpha, bos=BOS, eos=EOS, unk=UNK, **kw):
    """members: [(P fp64, cfg, memory, bias)]; weights normalised.  tests/beam_oracle.beam_search on the fp64 mixture."""
    fns = [_member_fn(P, cfg) for P, cfg, _, _ in members]
    logw = torch.tensor(weights, dtype=torch.float64).log().view(-1, 1, 1)

    def mixture(ids, caches, time):
        lp = torch.stack([torch.log_softmax(fn(ids, c, time), -1) for fn, c in zip(fns, caches)])
        return torch.logsumexp(lp + logw, 0)

    caches = [_member_cache(cfg, m, b) for _, cfg, m, b in members]
    B, Tm = members[0][2].shape[0], members[0][2].shape[1]
    with torch.no_grad():
        return BO.beam_search(mixture, torch.full((B,), int(bos), dtype=torch.long), caches, eos, unk, beam, alpha,
                              encoder_inputs_maxlen=Tm, **kw)


@functools.lru_cache(maxsize=None)
def _params(seed, wide=False):
    cfg = WIDE if wide else SMALL
    return U.chaotic_decode_params(R.init_params(cfg, seed=seed, random_bias=True), 4.0, seed)


@functools.lru_cache(maxsize=None)
def _runtime(seed, wide=False, precision="fp32"):
    rt = U.speech_runtime(WIDE if wide else SMALL, precision)
    rt.load_parameters(_params(seed, wide))
    return rt


def _inputs(B):
    _, src, lens = _small(4)                      # every member decodes the same utterances
    return src[:B], lens[:B]


@functools.lru_cache(maxsize=None)
def _speech_oracle(specs, B, beam, alpha, weights):
    """specs: ((seed, wide), ...) members over the encoder path (fp32 weights)."""
    src, lens = _inputs(B)
    members = []
    for seed, wide in specs:
        P = {k: v.double() for k, v in _params(seed, wide).items()}
        memory, bias = _speech_memory(P, WIDE if wide else SMALL, src, lens)
        members.append((P, WIDE if wide else SMALL, memory, bias))
    return ensemble_oracle(members, list(weights), beam, alpha, maximum_decode_length=MAX_LEN, extra_decode_length=EXTRA)


def _device(specs, B, beam, alpha, weights, use_graph=True):
    src, lens = _inputs(B)
    out = D.ensemble_beam_search([_runtime(s, w) for s, w in specs], dict(src=src, src_length=lens), BOS, EOS, UNK, weights=weights,
                                 beam_size=beam, length_penalty=alpha, maximum_decode_length=MAX_LEN, extra_decode_length=EXTRA,
                                 use_graph=use_graph)
    torch.cuda.synchronize()
    return out


# ---- 1. one member is the plain search ------------------------------------------------------------------------------------
def test_one_member_is_the_plain_beam_search_fp32():
    """One member routes to b200st_beam_search itself.  The 8-row fp32 step reduces with fp32 atomics, so two runs agree to
    rounding rather than bit for bit (as test_beam_search_gpu's two searches); the deterministic wide step is compared bit
    for bit below."""
    src, lens = _inputs(2)
    rt = _runtime(4)
    kw = dict(beam_size=4, length_penalty=0.6, maximum_decode_length=MAX_LEN, extra_decode_length=EXTRA)
    ens = D.ensemble_beam_search([rt], dict(src=src, src_length=lens), BOS, EOS, UNK, weights="average", **kw)
    ref = D.beam_search(rt, dict(src=src, src_length=lens), BOS, EOS, UNK, **kw)
    torch.cuda.synchronize()
    assert torch.equal(ens[0], ref[0]) and torch.equal(ens[3], ref[3])
    assert torch.allclose(ens[1], ref[1], rtol=1e-5, atol=0.0) and torch.allclose(ens[2], ref[2], rtol=1e-5, atol=1e-6)


# 64 utterances x beam 4 on the wide step, fixed memory (as test_decode_rows_gpu's beam cases)
WIDE_B, WIDE_TM, WIDE_SEEDS = 64, 61, (2, 5)


@functools.lru_cache(maxsize=None)
def _wide_case():
    P0 = U.chaotic_decode_params(R.init_params(SMALL, seed=WIDE_SEEDS[0], random_bias=True), 4.0, WIDE_SEEDS[0])
    P1 = U.chaotic_decode_params(R.init_params(SMALL, seed=WIDE_SEEDS[1], random_bias=True), 4.0, WIDE_SEEDS[1])
    memory, bias = ragged_memory(SMALL, WIDE_B, WIDE_TM, 105)
    memory1 = torch.randn(memory.shape, generator=torch.Generator().manual_seed(7))     # same ragged lengths (bias)
    return (P0, memory), (P1, memory1), bias


@functools.lru_cache(maxsize=None)
def _wide_runtime(i, precision):
    rt = U.speech_runtime(SMALL, precision)
    rt.load_parameters(_wide_case()[i][0])
    return rt


def _wide_device(n, precision, steps, weights="average", B=WIDE_B, use_graph=True):
    case = _wide_case()
    rts = [_wide_runtime(i, precision) for i in range(n)]
    caches = [D.create_decoding_cache(rt, case[i][1][:B].cuda(), case[2][:B].cuda(), steps, use_shadow=True, beam=4)
              for i, rt in enumerate(rts)]
    out = D.ensemble_beam_search(rts, None, 94, 95, 93, weights=weights, beam_size=4, length_penalty=0.6, maximum_decode_length=steps,
                                 extra_decode_length=8, use_shadow=True, use_graph=use_graph, caches=caches)
    torch.cuda.synchronize()
    return out


def test_one_member_is_the_plain_beam_search_wide_fp16_bit_for_bit():
    steps = 8
    case = _wide_case()
    ens = _wide_device(1, "fp16", steps)
    rt = _wide_runtime(0, "fp16")
    ref = D.beam_search(rt, None, 94, 95, 93, beam_size=4, length_penalty=0.6, maximum_decode_length=steps, extra_decode_length=8,
                        use_shadow=True, cache=D.create_decoding_cache(rt, case[0][1].cuda(), case[2].cuda(), steps, use_shadow=True, beam=4))
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(ens, ref))


# ---- 2. token-exact against the fp64 ensemble oracle ---------------------------------------------------------------------
@pytest.mark.parametrize("B,beam", [(2, 4), (1, 8)])
@pytest.mark.parametrize("alpha", [-1.0, 0.6])
@pytest.mark.parametrize("use_graph", [True, False])
@pytest.mark.parametrize("weights", ["average", "0.7,0.3"])
def test_two_members_token_ids_exact(B, beam, alpha, use_graph, weights):
    specs = TWO
    ref = _speech_oracle(specs, B, beam, alpha, tuple(D.ensemble_weights(weights, 2)))
    ids, scores, logprob, length = _device(specs, B, beam, alpha, weights, use_graph)
    _check(ref, ids, scores, length)
    assert torch.allclose(logprob.cpu(), ref["logprob"], rtol=1e-4, atol=1e-5)


# ---- 3. members of different shapes --------------------------------------------------------------------------------------
def test_members_of_different_shapes():
    """d 64 / 4 heads / 2 decoder layers next to d 128 / 4 heads / 3 decoder layers: a member reading another's config,
    layout or scratch changes the mixture."""
    specs = ((6, False), (3, True))
    for alpha in (0.6, -1.0):
        ref = _speech_oracle(specs, 2, 4, alpha, (0.5, 0.5))
        ids, scores, logprob, length = _device(specs, 2, 4, alpha, "average")
        _check(ref, ids, scores, length)
        assert torch.allclose(logprob.cpu(), ref["logprob"], rtol=1e-4, atol=1e-5)


# wide step, beam 8, 1600 memory positions: the cross-attention step needs more than the 48 KB default of dynamic shared
# memory, and the member with the larger head (dh 64) comes first.  Setting the kernel's limit member after member would
# leave it at the second member's (dh 32) need, below the first member's launch.
SHAPES_TM, SHAPES_STEPS = 1600, 8
BIG_HEAD = dict(SMALL, d=64, heads=1)
SMALL_HEAD = dict(SMALL, d=128, heads=4, dec_layers=3, ffn=256)


@functools.lru_cache(maxsize=None)
def _shape_pitfall_case():
    cfgs = (BIG_HEAD, SMALL_HEAD)
    Ps = [U.chaotic_decode_params(R.init_params(c, seed=s, random_bias=True), 4.0, s) for c, s in zip(cfgs, (3, 8))]
    _, bias = ragged_memory(BIG_HEAD, 2, SHAPES_TM, 104)
    mems = [torch.randn(2, SHAPES_TM, c["d"], generator=torch.Generator().manual_seed(20 + i)) for i, c in enumerate(cfgs)]
    ref = ensemble_oracle([(shadow_rounded(P, torch.float16), c, m, bias) for P, c, m in zip(Ps, cfgs, mems)], [0.5, 0.5], 8, 0.6,
                          bos=94, eos=95, unk=93, maximum_decode_length=SHAPES_STEPS, extra_decode_length=8)
    return cfgs, Ps, mems, bias, ref


def test_members_of_different_head_sizes_share_the_shared_memory_limit():
    cfgs, Ps, mems, bias, ref = _shape_pitfall_case()
    rts = []
    for c, P in zip(cfgs, Ps):
        rt = U.speech_runtime(c, "fp16")
        rt.load_parameters(P)
        rts.append(rt)
    caches = [D.create_decoding_cache(rt, m.cuda(), bias.cuda(), SHAPES_STEPS, use_shadow=True, beam=8) for rt, m in zip(rts, mems)]
    ids, scores, logprob, length = D.ensemble_beam_search(rts, None, 94, 95, 93, beam_size=8, length_penalty=0.6,
                                                          maximum_decode_length=SHAPES_STEPS, extra_decode_length=8, use_shadow=True,
                                                          caches=caches)
    torch.cuda.synchronize()
    _check(ref, ids, scores, length)


# ---- 4. the wide step: 64 utterances x beam 4 on the 16-bit shadow --------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _wide_oracle(precision, steps, weights):
    case = _wide_case()
    dt = DTYPES[precision]
    members = [(shadow_rounded(case[i][0], dt), SMALL, case[i][1], case[2]) for i in range(2)]
    return ensemble_oracle(members, list(weights), 4, 0.6, bos=94, eos=95, unk=93, maximum_decode_length=steps, extra_decode_length=8)


WIDE_STEPS = 8


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
def test_wide_two_members_token_ids_exact(precision):
    ref = _wide_oracle(precision, WIDE_STEPS, (0.6, 0.4))
    ids, scores, logprob, length = _wide_device(2, precision, WIDE_STEPS, weights="0.6,0.4")
    print("\n[ensemble wide 64x4 %s] %d steps, gap %.2e" % (precision, ref["steps"], ref["gap"]))
    _check(ref, ids, scores, length)
    assert torch.allclose(logprob.cpu(), ref["logprob"], rtol=1e-4, atol=1e-5)


# ---- 5. beam_size 1: the ensemble's greedy search --------------------------------------------------------------------------
def test_beam_one_token_ids_exact():
    specs = TWO
    ref = _speech_oracle(specs, 2, 1, 0.6, (0.5, 0.5))
    ids, scores, logprob, length = _device(specs, 2, 1, 0.6, "average")
    _check(ref, ids, scores, length)
    assert torch.allclose(logprob.cpu(), ref["logprob"], rtol=1e-4, atol=1e-5)


# ---- 6. reproducibility ----------------------------------------------------------------------------------------------------
def test_bit_reproducible_and_rows_independent_of_their_batch():
    a, b = _wide_device(2, "fp16", WIDE_STEPS), _wide_device(2, "fp16", WIDE_STEPS)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    # the first 16 utterances as a batch of their own (64 rows) and inside the batch of 64 (256 rows): bit-equal
    part = _wide_device(2, "fp16", WIDE_STEPS, B=16)
    assert torch.equal(part[0], a[0][:16]) and torch.equal(part[1], a[1][:16]) and torch.equal(part[3], a[3][:16])


# ---- 7. limits ---------------------------------------------------------------------------------------------------------------
def _abi(rts, caches, weights, beam=4, steps=8, state_words=True):
    """b200st_ensemble_beam_search called directly -> (rc, message, kernels launched)."""
    lib = L.load()
    B = caches[0].B if caches else 1
    dev = torch.device("cuda")
    bos = torch.full((B,), 94, dtype=torch.int64, device=dev)
    out = torch.empty(B, steps, dtype=torch.int64, device=dev)
    f = [torch.zeros(B, dtype=torch.float32, device=dev) for _ in range(2)]
    ln = torch.zeros(B, dtype=torch.int32, device=dev)
    words = torch.zeros(1 << 20, dtype=torch.int64, device=dev)
    a = L.BeamArgs()
    a.bos_ids, a.eos_id, a.unk_id, a.min_len, a.max_steps = bos.data_ptr(), 95, 93, 0, steps
    a.beam_size, a.top_k, a.length_penalty = beam, 1, 0.6
    a.out_ids, a.out_scores, a.out_logprob, a.out_len = out.data_ptr(), f[0].data_ptr(), f[1].data_ptr(), ln.data_ptr()
    a.state_words, a.use_graph = (words.data_ptr() if state_words else None), 1
    n = len(weights)
    bufs = [D._bufs(rt) for rt in rts]
    members = (L.EnsembleMember * max(n, 1))()
    for i in range(min(n, len(rts))):
        members[i].h, members[i].buf, members[i].st = rts[i].handle, C.pointer(bufs[i]), C.pointer(caches[i].state)
    for i in range(n):
        members[i].weight = weights[i]
    torch.cuda.synchronize()
    before = L.launch_count()
    with torch.cuda.stream(torch.cuda.Stream()):          # the step is captured into a CUDA graph: not the legacy stream
        rc = lib.b200st_ensemble_beam_search(members, n, C.byref(a), L._stream())
    torch.cuda.synchronize()
    return rc, lib.b200st_last_error().decode(), L.launch_count() - before


def test_limits_fail_before_any_launch():
    P, memory, bias = _params(4), *ragged_memory(SMALL, 2, 61, 3)
    rt0, rt1 = _runtime(4), _runtime(7)
    other_vocab = dict(SMALL, vocab=104)
    rtv = U.speech_runtime(other_vocab, "fp32")
    rtv.load_parameters(R.init_params(other_vocab, seed=1, random_bias=True))

    def cache(rt, B=2, Tm=61, max_len=8, beam=4, shadow=False):
        return D.create_decoding_cache(rt, memory[:B, :Tm].cuda(), bias[:B, :Tm].cuda(), max_len, use_shadow=shadow, beam=beam)

    good = [cache(rt0), cache(rt1)]
    cases = [
        (([rt0, rtv], [good[0], cache(rtv)], [0.5, 0.5]), "vocabulary"),
        (([rt0, rt1], [good[0], cache(rt1, B=1)], [0.5, 0.5]), "decode state"),
        (([rt0, rt1], [good[0], cache(rt1, Tm=40)], [0.5, 0.5]), "decode state"),
        (([rt0, rt1], [good[0], cache(rt1, max_len=12)], [0.5, 0.5]), "decode state"),
        (([], [], []), "1..8 members"),
        (([rt0] * 9, [good[0]] * 9, [1.0] * 9), "1..8 members"),
        (([rt0, rt1], good, [-0.5, 1.5]), ">= 0"),
        (([rt0, rt1], good, [float("nan"), 1.0]), "finite"),
        (([rt0, rt1], good, [0.0, 0.0]), "positive sum"),
    ]
    for (rts, caches, weights), msg in cases:
        rc, err, launched = _abi(rts, caches, weights)
        assert rc != 0 and msg in err and launched == 0, (msg, rc, err, launched)
    rc, err, launched = _abi([rt0, rt1], good, [0.5, 0.5], state_words=False)
    assert rc != 0 and "null argument" in err and launched == 0, err
    # 16 x 4 rows: member 1's state is not on the shadow
    rt16 = [_wide_runtime(0, "fp16"), _wide_runtime(1, "fp16")]
    wide = [D.create_decoding_cache(rt, _wide_case()[i][1][:16].cuda(), _wide_case()[2][:16].cuda(), 8, use_shadow=True, beam=4)
            for i, rt in enumerate(rt16)]
    wide[1].state.use_shadow = 0
    rc, err, launched = _abi(rt16, wide, [0.5, 0.5])
    assert rc != 0 and "at most 8 rows" in err and launched == 0, err
    # the Python surface: the reference's count error, and the library's messages come through
    with pytest.raises(ValueError, match="equal to the models"):
        D.ensemble_beam_search([rt0, rt1], None, 94, 95, 93, weights="0.2,0.3,0.5", caches=good, maximum_decode_length=8)
    with pytest.raises(L.B200STError, match="positive sum"):
        D.ensemble_beam_search([rt0, rt1], None, 94, 95, 93, weights=[0, 0], caches=good, maximum_decode_length=8)
    # a valid call afterwards still works
    rc, err, launched = _abi([rt0, rt1], good, [0.5, 0.5])
    assert rc == 0 and launched > 0, err


# ---- 8. predict through the entry ------------------------------------------------------------------------------------------
def test_predict_with_an_ensemble_through_the_entry(tmp_path, monkeypatch):
    from neurst_b200 import cli
    from neurst_b200.models import EncoderDecoderEnsembleModel
    from tests import test_cli as T
    T._write_dataset(tmp_path, vocab=93)
    y = T._write_yaml(tmp_path, data=str(tmp_path / "train.tfrecords"), n_tokens=93)
    tiny = ["--model.params.encoder.num_layers", "2", "--model.params.decoder.num_layers", "2",
            "--model.params.encoder.hidden_size", "128", "--model.params.decoder.hidden_size", "128", "--model.params.modality.dim", "128",
            "--model.params.encoder.num_attention_heads", "2", "--model.params.decoder.num_attention_heads", "2",
            "--model.params.encoder.filter_size", "256", "--model.params.decoder.filter_size", "256",
            "--model.params.modality.source.channels", "64"]
    common = ["--config_paths", y, "--task.params.batch_size", "3000", "--task.params.max_src_len", "400",
              "--task.params.max_trg_len", "24", "--task.params.min_src_bucket_boundary", "128",
              "--task.params.experimental_frame_transcript_ratio", "20", "--save_checkpoint_steps", "3", "--summary_steps", "2"]
    dirs = [str(tmp_path / "model_a"), str(tmp_path / "model_b")]
    for d, seed in zip(dirs, (1, 2)):
        assert cli.main(common + tiny + ["--model_dir", d, "--train_steps", "4", "--random_seed", str(seed)])["global_step"] == 4
        assert os.path.exists(os.path.join(d, "model_configs.yml"))
    one = tmp_path / "one"
    one.mkdir()
    os.link(str(tmp_path / "train.tfrecords-00000-of-00003"), str(one / "train.tfrecords-00000-of-00001"))
    checked = []
    orig = EncoderDecoderEnsembleModel.beam_search

    def checked_search(self, inputs, **kw):
        ids, scores = orig(self, inputs, **kw)
        if len(checked) < 3:        # the same inputs straight through decode.ensemble_beam_search
            tm = self.models[0]._trg_meta
            ref = D.ensemble_beam_search([m.runtime for m in self.models], inputs, tm["bos_id"], tm["eos_id"], tm["unk_id"],
                                         weights=kw["ensemble_weights"], beam_size=kw["beam_size"], length_penalty=kw["length_penalty"],
                                         maximum_decode_length=kw["maximum_decode_length"],
                                         extra_decode_length=kw["extra_decode_length"])
            checked.append((torch.equal(ref[0], ids), kw["ensemble_weights"]))
        return ids, scores

    monkeypatch.setattr(EncoderDecoderEnsembleModel, "beam_search", checked_search)
    out = str(tmp_path / "hyp.txt")
    # the tiny architecture comes from each directory's model_configs.yml, not from the command line
    pred = common + ["--model_dir", ",".join(dirs), "--entry.class", "predict", "--output_file", out,
                     "--dataset.params.data_path", str(one / "train.tfrecords"), "--search_method", "beam_search",
                     "--search_method.params.beam_size", "4", "--search_method.params.length_penalty", "-1",
                     "--search_method.params.maximum_decode_length", "12"]
    res = cli.main(pred + ["--ensemble_weights", "0.6,0.4"])
    assert res["n_hypotheses"] == 70 and res["checkpoint_step"] == [4, 4]
    assert len(checked) == 3 and all(same for same, _ in checked), checked
    assert all(math.isclose(a, b) for a, b in zip(checked[0][1], [0.6, 0.4])), checked
    lines = open(out, encoding="utf-8").read().split("\n")
    assert len(lines) == 71 and all(all(t.startswith("tok") or t == "<UNK>" for t in l.split()) for l in lines[:-1])
    with pytest.raises(SystemExit, match="equal to the models"):
        cli.main(pred + ["--ensemble_weights", "0.5,0.3,0.2"])
    torch.cuda.synchronize()
