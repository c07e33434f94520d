"""Streaming simultaneous translation without a GPU: the restated SimulTransTextAgent (policy, word recovery from `@@` and
`▁` units, force_segment and its state reset, max_len) against hand-worked cases with a scripted model side, the latency
of a replayed wait-k schedule, the `simuleval` entry's resolution and refusals, spill-free stream kernels, and the ABI."""
import os
import re

import pytest
import yaml

from neurst_b200 import cli
from neurst_b200 import lib as L
from neurst_b200 import metrics as MT
from neurst_b200 import simultaneous as S
from tests.test_mt_cpu import _mt_cfg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Scripted:
    """A model side that emits a fixed id sequence and records what the agent reads."""

    def __init__(self, emit):
        self.emit, self.reads, self.resets, self.t = list(emit), [], 0, 0

    def reset(self):
        self.resets += 1

    def read(self, ids):
        self.reads.append(list(ids))

    def write(self):
        x = self.emit[min(self.t, len(self.emit) - 1)]
        self.t += 1
        return x


def _meta(tokens):
    n = len(tokens) + 3
    return {"tokens": list(tokens), "vocab_size": n, "unk_id": n - 3, "bos_id": n - 2, "eos_id": n - 1}


SRC = _meta(["a", "b", "c", "d", "e", "ok.", "Dr.", 'end."', "wait...", "A.", "new@@", "york"])
TRG = _meta(["x1", "x2", "x3", "x4", "x5", "x6", "ne@@", "w"])
EOS = TRG["eos_id"]


def _run(agent, words):
    return agent.translate([[w] for w in words], clock=lambda: 0.0)


def test_policy_of_wait_2_over_five_words():
    model = Scripted([0, 1, 2, 3, 4, 5, EOS])
    agent = S.SimulTransTextAgent(model, SRC, TRG, wait_k=2)
    r = _run(agent, ["a", "b", "c", "d", "e"])
    assert "".join(a for a, _ in r["actions"]) == "RRWRWRWRWRWWW"
    assert r["prediction"] == ["x1", "x2", "x3", "x4", "x5", "x6"]
    assert r["delays"] == [2, 3, 4, 5, 5, 5]
    # each WRITE encodes what was read since the last one; the source EOS once reading has finished
    assert model.reads == [[0, 1], [2], [3], [4], [SRC["eos_id"]]]


@pytest.mark.parametrize("n_src, n_trg, k", [(5, 5, 2), (7, 3, 3), (3, 8, 1), (6, 6, 9)])
def test_latency_of_a_replayed_schedule_equals_waitk_latency(n_src, n_trg, k):
    model = Scripted(list(range(n_trg)) + [EOS])
    trg = _meta(["y%d" % i for i in range(n_trg)])
    model.emit[-1] = trg["eos_id"]
    agent = S.SimulTransTextAgent(model, SRC, trg, wait_k=k)
    r = _run(agent, ["a"] * n_src)
    assert len(r["prediction"]) == n_trg
    got, want = MT.simul_latency(r["delays"], n_src), MT.waitk_latency(k, n_src, n_trg)
    assert got == pytest.approx(want)


def test_word_recovery_from_bpe_and_bow_units():
    assert S.words_of("new@@ york is a@@ b@@ c .") == [["new@@", "york"], ["is"], ["a@@", "b@@", "c"], ["."]]
    assert S.words_of("▁new york ▁is ▁a b c", bow=True) == [["▁new", "york"], ["▁is"], ["▁a", "b", "c"]]
    # target side, subword-nmt: "ne@@ w" is one word, emitted when its last piece arrives
    model = Scripted([6, 7, 0, EOS])
    r = _run(S.SimulTransTextAgent(model, SRC, TRG, wait_k=1), ["a", "b", "c"])
    assert r["prediction"] == ["new", "x1"] and r["delays"] == [1, 2]
    # target side, BOW_PREFIX: a word is emitted when the next word's first piece arrives, the last one at EOS
    trg = _meta(["▁new", "york", "▁is", "▁big"])
    model = Scripted([0, 1, 2, 3, trg["eos_id"]])
    r = _run(S.SimulTransTextAgent(model, SRC, trg, wait_k=1), ["a", "b", "c", "d", "e"])
    assert r["prediction"] == ["newyork", "is", "big"] and r["delays"] == [1, 2, 3]
    # source units of a BPE'd word, unknown tokens as UNK
    agent = S.SimulTransTextAgent(Scripted([EOS]), SRC, TRG, wait_k=1)
    assert agent.segment_to_units(["new@@", "york"], S._States()) == [10, 11]
    assert agent.segment_to_units(["zzz"], S._States()) == [SRC["unk_id"]]


@pytest.mark.parametrize("word, ends", [('end."', True), ("wait...", True), ("Dr.", False), ("A.", False), ("ok.", True),
                                        ("a", False)])
def test_force_segment_rules(word, ends):
    agent = S.SimulTransTextAgent(Scripted([EOS]), SRC, TRG, wait_k=1, force_segment=True)
    st = S._States()
    units = agent.segment_to_units([word], st)
    assert st.segment is ends
    assert units[-1] == SRC["eos_id"] if ends else SRC["eos_id"] not in units
    plain = S.SimulTransTextAgent(Scripted([EOS]), SRC, TRG, wait_k=1)
    st = S._States()
    assert SRC["eos_id"] not in plain.segment_to_units([word], st) and not st.segment


def test_forced_segment_resets_the_states_and_the_stream():
    # "ok." ends a segment: EOS joins its units, the agent writes until EOS, then starts over with empty states (the
    # target EOS ends the segment, not the sentence) and reads the next word
    model = Scripted([0, EOS, 1, EOS])
    agent = S.SimulTransTextAgent(model, SRC, TRG, wait_k=1, force_segment=True)
    r = _run(agent, ["a", "ok.", "b"])
    assert r["prediction"] == ["x1", "x2"]
    assert model.resets == 2                      # the sentence's start and the forced segment's end
    assert model.reads[:2] == [[0], [5, SRC["eos_id"]]]
    assert model.reads[2] == [1]                  # after the reset, the stream restarts at the next word


def test_max_len_stops_the_translation():
    model = Scripted([0])                         # never emits EOS
    r = _run(S.SimulTransTextAgent(model, SRC, TRG, wait_k=1, max_len=3), ["a", "b"])
    assert r["prediction"] == ["x1"] * 4 and model.t == 4


def test_japanese_target_is_refused():
    with pytest.raises(ValueError, match="Japanese"):
        S.SimulTransTextAgent(Scripted([EOS]), SRC, dict(TRG, language="ja"), wait_k=1)


# ------------------------------------------------------------------------------------------------ the simuleval entry
def _waitk_dir(tmp_path, name, trg_tokens=("x", "y", "z"), model_class="WaitkTransformer", language="de"):
    sub = tmp_path / name
    sub.mkdir()
    cfg = _mt_cfg(sub, trg_tokens=trg_tokens, **{"task.class": "WaitkTranslation", "hparams_set": "waitk_transformer_s"})
    cfg["task.params"]["wait_k"] = 3
    cfg["task.params"]["trg_data_pipeline.params"]["language"] = language
    plan = cli.resolve(cfg)
    cli.write_model_configs(dict(plan, model_dir=str(sub / "m")))
    path = sub / "m" / cli.MODEL_CONFIGS
    if model_class != "WaitkTransformer":
        configs = yaml.safe_load(path.read_text())
        configs["model.class"] = model_class
        path.write_text(yaml.safe_dump(configs))
    return str(sub / "m")


def _entry(tmp_path, dirs, *extra):
    src = tmp_path / "src.bpe"
    src.write_text("a b\n")
    argv = ["--entry", "simuleval", "--model_dir", ",".join(dirs), "--source", str(src), "--target", str(src),
            "--output", str(tmp_path / "out")] + list(extra)
    paths, overrides = cli.parse_command_line(argv)
    return cli.resolve(cli.load_config(paths, overrides))


def test_simuleval_entry_resolves_members_and_overrides_wait_k(tmp_path):
    a, b = _waitk_dir(tmp_path, "a"), _waitk_dir(tmp_path, "b")
    plan = _entry(tmp_path, [a, b], "--wait_k", "4", "--force_segment", "true", "--max_len", "50")
    assert plan["entry"] == "simuleval" and plan["wait_k"] == 4
    assert plan["force_segment"] is True and plan["max_len"] == 50
    assert [m["model_dir"] for m in plan["members"]] == [a, b]
    assert all(m["wait_k"] == 4 and m["model_params"]["encoder.attention_monotonic"] is True for m in plan["members"])
    plan = _entry(tmp_path, [a], "--wait_k", "2")
    assert plan["force_segment"] is False and plan["max_len"] == 200 and len(plan["members"]) == 1


def test_simuleval_entry_refusals(tmp_path):
    a = _waitk_dir(tmp_path, "a")
    with pytest.raises(SystemExit, match="wait_k"):
        _entry(tmp_path, [a])
    with pytest.raises(SystemExit, match="wait_k"):
        _entry(tmp_path, [a], "--wait_k", "0")
    plain = _waitk_dir(tmp_path, "plain", model_class="Transformer")
    with pytest.raises(SystemExit, match="not a wait-k model"):
        _entry(tmp_path, [a, plain], "--wait_k", "3")
    other = _waitk_dir(tmp_path, "other", trg_tokens=("x", "y", "w"))
    with pytest.raises(SystemExit, match="target vocabulary"):
        _entry(tmp_path, [a, other], "--wait_k", "3")
    ja = _waitk_dir(tmp_path, "ja", language="ja")
    with pytest.raises(SystemExit, match="Japanese"):
        _entry(tmp_path, [ja], "--wait_k", "3")
    # the offline predict still refuses a wait-k ensemble
    with pytest.raises(SystemExit, match="ensemble"):
        cli.resolve({"entry.class": "predict", "task.class": "WaitkTranslation", "model_dir": [a, a], "wait_k": 3,
                     "task.params": yaml.safe_load(open(os.path.join(a, cli.MODEL_CONFIGS)))["task.params"],
                     "dataset.params": {"src_file": "-", "data_is_processed": True}})


# ------------------------------------------------------------------------------------------------ kernels and ABI
def test_stream_kernels_do_not_spill():
    from tests.test_waitk_cpu import _ptxas
    table = _ptxas("stream.cu")
    attn = {k: v for k, v in table.items() if "stream_attn_kernel" in k}
    assert len(attn) == 6, sorted(table)
    assert not any(re.search(r"attn_step_kernel|greedy_persistent_kernel|rows_cross_attn_kernel", k) for k in table)
    spilled = {k: v for k, v in table.items() if re.search(r"stream_|gemv_kernel|logits_step_kernel|embed_step", k) and (v[1] or v[2])}
    assert not spilled, spilled
    # the decode translation unit still holds exactly its attention-step instantiations
    assert len([k for k in _ptxas("decode.cu") if re.search(r"attn_step_kernel|greedy_persistent_kernel", k)]) == 15


def test_stream_abi_is_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "b200st.h")).read()
    declared = {s for s in re.findall(r"\b(b200st_stream_[a-z_]+)\s*\(", header)}
    assert declared == {"b200st_stream_scratch_floats", "b200st_stream_create", "b200st_stream_destroy", "b200st_stream_reset",
                        "b200st_stream_read", "b200st_stream_write", "b200st_stream_lengths"}
    assert declared <= set(L.EXPORTS)
    lib = L.load()
    assert all(hasattr(lib, s) for s in declared)
    fields = re.search(r"typedef struct \{\s*int32_t max_src, max_trg;(.*?)\} b200st_stream_state;", header, re.S).group(1)
    names = ["max_src", "max_trg"] + re.findall(r"[\*\s](\w+)[;,]", fields)
    assert names == [f for f, _ in L.StreamState._fields_]
