"""Streaming simultaneous translation on the device (b200st_stream_*, simultaneous.py): a source read in chunks of any size
equals the whole-prefix encoding and cross K/V, a WRITE equals the lagged decoder step, the agent with 1..3 members (with and
without force_segment; fp32 weights and 16-bit shadows) emits what an fp64 restatement of the reference agent emits, one
member with one-token words equals the wait-k greedy search, and the `simuleval` entry on a trained checkpoint."""
import json
import types

import pytest
import torch

from neurst_b200 import cli
from neurst_b200 import decode as D
from neurst_b200 import simultaneous as S
from neurst_b200.runtime import Runtime, make_config
from neurst_b200 import lib as L
from oracle import restatement as R
from tests import parity_utils as U
from tests.test_waitk_gpu import BOS, EOS, MIN_GAP, SMALL, _check_greedy, corpus, trained  # noqa: F401
from tests.waitk_oracle import monotonic_padding, waitk_greedy

pytestmark = pytest.mark.gpu

DT = {"fp16": torch.float16, "bf16": torch.bfloat16}
SRC_EOS = SMALL["src_vocab"] - 1
# tensors the streaming kernels read from the 16-bit shadow (use_shadow): the embeddings and the weight matrices of both
# stacks except the cross-attention K/V projection
SHADOW_SUFFIXES = (".qkv.kernel", ".out.kernel", ".q.kernel", ".w1", ".w2")


def _params(seed):
    return U.chaotic_decode_params(R.init_params(SMALL, seed=seed, random_bias=True), 4.0, seed)


def rounded(P, dtype):
    return {k: (v.to(dtype).float() if (k.endswith("emb") or k.endswith(SHADOW_SUFFIXES)) else v) for k, v in P.items()}


def _model(P, precision="fp32", k=3):
    c = make_config(L.MODEL_TEXT, SMALL["d"], SMALL["heads"], SMALL["ffn"], SMALL["enc_layers"], SMALL["dec_layers"], SMALL["vocab"],
                    src_vocab=SMALL["src_vocab"], precision=precision, encoder_monotonic=True)
    rt = Runtime(c)
    rt.load_parameters(P)
    meta = dict(vocab_size=SMALL["vocab"], unk_id=SMALL["vocab"] - 3, bos_id=BOS, eos_id=EOS, tokens=None)
    return types.SimpleNamespace(runtime=rt, wait_k=k, _trg_meta=meta)


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("precision", ["fp32", "fp16", "bf16"])
def test_chunked_reads_equal_the_whole_prefix_encoding(precision):
    P = _params(5)
    src = torch.randint(0, SMALL["src_vocab"] - 3, (30,), generator=torch.Generator().manual_seed(8))
    ref_m = _model(P if precision == "fp32" else rounded(P, DT[precision]))
    enc, bias = D.encode(ref_m.runtime, dict(src=src[None], src_padding=torch.zeros(1, 30)))
    ref_kv = D.create_decoding_cache(ref_m.runtime, enc, bias, 4).cross_kv[:, 0]
    m = _model(P, precision)
    s = S.StreamingSession([m], use_shadow=precision != "fp32", max_src=32, max_trg=8, keep_encoder_output=True)
    # fp32: summation order only; the shadow path reads the same rounded weights as the fp32 reference
    tol = 1e-5 if precision == "fp32" else 2e-5
    for chunks in ([1] * 30, [3] * 10, [8] * 3 + [6], [11, 11, 8], [1, 11, 3, 8, 1, 6], [8, 3, 11, 1, 1, 3, 3]):
        s.reset()
        o = 0
        for n in chunks:
            s.read(src[o:o + n])
            o += n
        torch.cuda.synchronize()
        assert s.lengths == (30, 0)
        st = s.states[0]
        assert _rel(st["enc_out"][:30], enc[0]) < tol, chunks
        assert _rel(st["cross_kv"][:, :30], ref_kv) < tol, chunks


def test_write_equals_the_lagged_decoder_step():
    """WRITE t after k + t source tokens gives b200st_decode_step's logits with wait_k = k on the whole source."""
    P, k, T = _params(5), 3, 13
    src = torch.randint(0, SMALL["src_vocab"] - 3, (T,), generator=torch.Generator().manual_seed(9))
    m = _model(P)
    rt = m.runtime
    enc, bias = D.encode(rt, dict(src=src[None], src_padding=torch.zeros(1, T)))
    cache = D.create_decoding_cache(rt, enc, bias, 16, wait_k=k)
    s = S.StreamingSession([m], max_src=16, max_trg=16)
    V = SMALL["vocab"]
    logits_view = s._keep[2][-64 - V:-64]          # the member's step logits: the last V floats before the scratch's pad
    s.read(src[:k])
    sym = BOS
    for t in range(8):
        if t:
            s.read(src[k + t - 1:k + t])
        nxt = s.write()
        got = logits_view.clone()
        want = D.decoder_step_logits(rt, torch.tensor([sym]), cache, t)[0]
        assert float((got - want).abs().max()) < 1e-4, t
        assert nxt == int(torch.log_softmax(got, -1).argmax())
        sym = nxt
    assert s.lengths == (k + 7, 8)


class Restated:
    """The reference agent's model side in fp64: every WRITE re-encodes the whole source read so far with the monotonic
    encoder (as test_greedy_equals_the_streaming_agent does) and runs each member's cached decoder step over all of it;
    the members' log-probabilities are mixed as logsumexp - log n and top_k(1) is taken.  `gaps` records the top-2 margin
    of every decision."""

    def __init__(self, Ps):
        self.Ps = [{n: v.double() for n, v in P.items()} for P in Ps]
        self.gaps, self.ids = [], []
        self.reset()

    def reset(self):
        H, dh = SMALL["heads"], SMALL["d"] // SMALL["heads"]
        self.src, self.t, self.last = [], 0, BOS
        self.caches = [[dict(keys=torch.zeros(1, 0, H, dh, dtype=torch.float64), values=torch.zeros(1, 0, H, dh, dtype=torch.float64))
                        for _ in range(SMALL["dec_layers"])] for _ in self.Ps]

    def read(self, ids):
        self.src += [int(i) for i in ids]

    def write(self):
        s = torch.tensor([self.src])
        pad = torch.zeros(1, len(self.src), dtype=torch.float64)
        lps = []
        for P, caches in zip(self.Ps, self.caches):
            enc = R.encoder(P, R.add_position(P["srcemb.emb"][s]), monotonic_padding(pad), SMALL["enc_layers"], SMALL["heads"])
            x = R.target_embed(P, torch.tensor([self.last]), time=self.t).unsqueeze(1)
            y = R.decoder(P, x, enc, R.input_padding_to_bias(pad), SMALL["dec_layers"], SMALL["heads"], caches=caches)
            lps.append(torch.log_softmax(R.logits_layer(P, y)[0, -1], -1))
        mix = torch.logsumexp(torch.stack(lps), 0) - torch.log(torch.tensor(float(len(lps)), dtype=torch.float64))
        top2 = mix.topk(2).values
        self.gaps.append(float(top2[0] - top2[1]))
        self.last = int(mix.argmax())
        self.ids.append(self.last)
        self.t += 1
        return self.last


class Recorded:
    def __init__(self, session):
        self.s, self.ids = session, []

    def reset(self):
        self.s.reset()

    def read(self, ids):
        self.s.read(ids)

    def write(self):
        self.ids.append(self.s.write())
        return self.ids[-1]


def _metas():
    src = ["s%d@@" % i if i % 7 == 3 else "s%d" % i for i in range(SMALL["src_vocab"] - 4)] + ["ok."]
    trg = ["t%d@@" % i if i % 5 == 2 else "t%d" % i for i in range(SMALL["vocab"] - 3)]
    src_meta = {"tokens": src, "vocab_size": len(src) + 3, "unk_id": len(src), "bos_id": len(src) + 1, "eos_id": len(src) + 2}
    return src_meta, {"tokens": trg, "vocab_size": len(trg) + 3, "unk_id": len(trg), "bos_id": BOS, "eos_id": EOS}


def _sentences(n, seed):
    g = torch.Generator().manual_seed(seed)
    src_meta, _ = _metas()
    out = []
    for _ in range(n):
        L_ = int(torch.randint(4, 12, (1,), generator=g))
        toks = [src_meta["tokens"][int(i)] for i in torch.randint(0, len(src_meta["tokens"]) - 1, (L_,), generator=g)]
        if L_ > 6:
            toks[L_ // 2] = "ok."                         # a forced segment end in the middle
        if toks[-1].endswith("@@"):
            toks[-1] = toks[-1][:-2]
        out.append(S.words_of(" ".join(toks)))
    return out


@pytest.mark.parametrize("precision", ["fp32", "fp16", "bf16"])
@pytest.mark.parametrize("n_members", [1, 2, 3])
@pytest.mark.parametrize("force_segment", [False, True])
def test_agent_emits_what_the_fp64_restated_agent_emits(precision, n_members, force_segment):
    Ps = [_params(5 + 11 * i) for i in range(n_members)]
    src_meta, trg_meta = _metas()
    ref_P = Ps if precision == "fp32" else [rounded(P, DT[precision]) for P in Ps]
    session = S.StreamingSession([_model(P, precision) for P in Ps], use_shadow=precision != "fp32", max_src=64, max_trg=64)
    compared = 0
    for i, words in enumerate(_sentences(4, 17 + n_members)):
        ref = Restated(ref_P)
        S.SimulTransTextAgent(ref, src_meta, trg_meta, 2, force_segment, max_len=30).translate(words)
        dev = Recorded(session)
        S.SimulTransTextAgent(dev, src_meta, trg_meta, 2, force_segment, max_len=30).translate(words)
        # the agents agree up to the first fp64 near-tie; the actions after it depend on which side of the tie each took
        n = next((t for t, g in enumerate(ref.gaps) if g < MIN_GAP), len(ref.gaps))
        assert dev.ids[:n] == ref.ids[:n], (i, dev.ids, ref.ids)
        compared += n
    assert compared >= 12, "too few decisions before a near-tie (%d)" % compared


def test_one_member_with_one_token_words_equals_the_waitk_greedy_search():
    P, k = _params(5), 2
    m = _model(P)
    src_meta = {"tokens": ["s%d" % i for i in range(SMALL["src_vocab"] - 3)], "unk_id": SMALL["src_vocab"] - 3, "eos_id": SRC_EOS}
    trg_meta = {"tokens": ["t%d" % i for i in range(SMALL["vocab"] - 3)], "eos_id": EOS, "bos_id": BOS}
    session = S.StreamingSession([m], max_src=32, max_trg=32)
    g = torch.Generator().manual_seed(21)
    P64 = {n: v.double() for n, v in P.items()}
    for n in (5, 9, 12):
        src = torch.randint(0, SMALL["src_vocab"] - 3, (n,), generator=g)
        r = S.SimulTransTextAgent(session, src_meta, trg_meta, k, max_len=24).translate([["s%d" % int(i)] for i in src])
        hyp = [int(w[1:]) for w in r["prediction"]][:20]
        full = torch.cat([src, torch.tensor([SRC_EOS])])[None]
        ids, _ = D.greedy_search(m.runtime, dict(src=full, src_padding=torch.zeros(1, n + 1)), BOS, EOS, None, 20, 20, 0,
                                 enable_unk=True, wait_k=k)[:2]
        ids = ids.cpu()[:, :20]
        ref_ids, ref_logits = waitk_greedy(P64, SMALL, full, torch.zeros(1, n + 1, dtype=torch.float64), BOS, EOS, 20, k, None)
        stream = torch.full((1, 20), EOS, dtype=torch.long)
        stream[0, :len(hyp)] = torch.tensor(hyp, dtype=torch.long)
        _check_greedy(stream, ref_ids, ref_logits)
        _check_greedy(ids, stream, ref_logits)


def test_simuleval_entry_on_a_trained_checkpoint(corpus, trained, tmp_path):  # noqa: F811
    from neurst_b200 import checkpoints as CK
    from tests.test_waitk_gpu import _plan
    plan = _plan(corpus, trained[0], 0, entry="predict", dtype="float32")
    model = cli._build_model(plan).init_parameters(7)
    model.load_parameters(U.chaotic_decode_params({n: v.cpu() for n, v in model.named_parameters().items()}, 4.0, 7))
    model_dir = tmp_path / "chaotic"
    cli.write_model_configs(dict(plan, model_dir=str(model_dir)))
    CK.save_npz(model.runtime, str(model_dir / "ckpt-1.npz"))
    (ds, dt) = corpus[2]
    out = tmp_path / "simul"
    res = cli.main(["--entry", "simuleval", "--model_dir", str(model_dir), "--wait_k", "3", "--source", ds, "--target", dt,
                    "--output", str(out), "--dtype", "float32"])
    lines = [json.loads(l) for l in open(out / "instances.log")]
    srcs = open(ds).read().splitlines()
    assert len(lines) == len(srcs) and all(len(l["delays"]) == len(l["prediction"].split()) for l in lines)
    assert all(a in ("R", "W") and t >= 0 for l in lines for a, t in l["action_seconds"])
    scores = json.load(open(out / "scores"))
    assert scores["n_sentences"] == len(srcs) and scores["BLEU"] is not None and scores["AL"] is not None
    assert res["AL"] == scores["AL"]
    # the same agent driven from Python
    p = cli.resolve({"entry": "simuleval", "model_dir": str(model_dir), "wait_k": 3, "source": ds, "output": str(out)})
    m, _ = cli._restore(p["members"][0], str(model_dir))
    agent = S.SimulTransTextAgent(S.StreamingSession([m], max_src=64, max_trg=p["max_len"] + 2), p["members"][0]["src_meta"],
                                  p["members"][0]["trg_meta"], 3)
    assert [" ".join(agent.translate(S.words_of(s))["prediction"]) for s in srcs] == [l["prediction"] for l in lines]
