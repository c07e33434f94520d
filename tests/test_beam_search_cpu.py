"""Beam search without a GPU: the restated reference search (tests/beam_oracle.py) on a scripted model whose outcomes are
worked out by hand, beam 1 against the oracle's greedy search, the b200st_beam_args layout, the `predict` configuration
(entry alias, search_method) and the compiler's resource report of the beam-search kernels."""
import math
import os
import re
import subprocess
import tempfile

import pytest
import torch

from neurst_b200 import cli
from neurst_b200 import lib as L
from oracle import restatement as R
from tests import beam_oracle as BO
from tests import parity_utils as U

A, B_, C_, UNK, BOS, EOS = 0, 1, 2, 3, 4, 5
V = 6


def _p(**kw):
    """probability vector over (a, b, c, UNK, BOS, EOS)"""
    names = ("a", "b", "c", "unk", "bos", "eos")
    return [kw[n] for n in names]


# next-symbol distribution as a fixed function of the hypothesis prefix (BOS excluded), never of the row it sits in
TABLE = {
    (): _p(a=.5, b=.3, c=.06, unk=.02, bos=.02, eos=.1),
    (A,): _p(a=.2, b=.1, c=.06, unk=.02, bos=.02, eos=.6),
    (B_,): _p(a=.02, b=.02, c=.9, unk=.01, bos=.01, eos=.04),
    (B_, C_): _p(a=.04, b=.04, c=.04, unk=.04, bos=.04, eos=.8),
}
DEFAULT = _p(a=.1, b=.1, c=.1, unk=.1, bos=.1, eos=.5)
UNK_TABLE = {(): _p(a=.2, b=.1, c=.03, unk=.6, bos=.02, eos=.05)}


def _scripted(table):
    def fn(ids, cache, time):
        cache["prefix"] = torch.cat([cache["prefix"], ids.unsqueeze(1)], 1)          # follows the beam through the gathers
        rows = [table.get(tuple(r[1:]), DEFAULT) for r in cache["prefix"].tolist()]
        return torch.tensor(rows, dtype=torch.float64).log().to(torch.float32)
    return fn


def _search(table=TABLE, **kw):
    args = dict(eos_id=EOS, unk_id=UNK, beam_size=2, maximum_decode_length=6, extra_decode_length=50)
    args.update(kw)
    return BO.beam_search(_scripted(table), torch.full((1,), BOS, dtype=torch.long), {"prefix": torch.zeros(1, 0, dtype=torch.long)},
                          **args)


def _pen(n, alpha):
    return 1.0 / n if alpha < 0 else ((5.0 + n) / 6.0) ** (-alpha)


def test_scripted_search_alpha_minus_one():
    """t=0 only the first beam counts (a, b; not a twice).  t=1: [a EOS] and [b c].  t=2: the finished [a EOS] keeps its
    log-probability and length and only emits EOS; [b c EOS] scores -1.532/3 > -1.204/2 and wins under 1/len."""
    r = _search(length_penalty_alpha=-1.0, top_k=2)
    lp_aE = math.log(.5) + math.log(.6)
    lp_bcE = math.log(.3) + math.log(.9) + math.log(.8)
    assert r["hypotheses"].tolist() == [[B_, C_, EOS, EOS, EOS, EOS], [A, EOS, EOS, EOS, EOS, EOS]]      # EOS padded
    assert r["length"].tolist() == [3, 2] and r["steps"] == 3
    assert torch.allclose(r["logprob"], torch.tensor([lp_bcE, lp_aE]), atol=1e-5)
    assert torch.allclose(r["scores"], torch.tensor([lp_bcE / 3, lp_aE / 2]), atol=1e-5)
    assert r["scores"][0] > r["scores"][1]                                                 # top_k = beam: best first
    top1 = _search(length_penalty_alpha=-1.0, top_k=1)
    assert top1["hypotheses"].tolist() == [[B_, C_, EOS, EOS, EOS, EOS]]


def test_scripted_search_alpha_changes_the_winner():
    """alpha = 0.6: ((5+len)/6)^-0.6 penalises length less than 1/len, so the short [a EOS] wins."""
    r = _search(length_penalty_alpha=0.6, top_k=2)
    lp_aE = math.log(.5) + math.log(.6)
    lp_bcE = math.log(.3) + math.log(.9) + math.log(.8)
    assert r["hypotheses"].tolist() == [[A, EOS, EOS, EOS, EOS, EOS], [B_, C_, EOS, EOS, EOS, EOS]]
    assert torch.allclose(r["scores"], torch.tensor([lp_aE * _pen(2, .6), lp_bcE * _pen(3, .6)]), atol=1e-5)


def test_scripted_search_step_limit():
    """maximum_decode_length 2: the search stops after two steps with [b c] unfinished; 1/len picks the finished
    [a EOS] (-0.602 > -0.654)."""
    r = _search(length_penalty_alpha=-1.0, top_k=2, maximum_decode_length=2)
    assert r["steps"] == 2
    assert r["hypotheses"].tolist() == [[A, EOS], [B_, C_]] and r["length"].tolist() == [2, 2]


def test_scripted_search_minimum_length_and_unk():
    """minimum_decode_length 3 masks EOS at t = 0, 1: [a EOS] is not reachable, [a a] takes the second beam, then both
    beams end at t = 2.  UNK is the most likely first symbol of UNK_TABLE and is only chosen when enabled."""
    r = _search(length_penalty_alpha=-1.0, top_k=2, minimum_decode_length=3)
    assert r["hypotheses"].tolist() == [[B_, C_, EOS, EOS, EOS, EOS], [A, A, EOS, EOS, EOS, EOS]]
    lp_aaE = math.log(.5) + math.log(.2) + math.log(.5)
    assert abs(float(r["scores"][1]) - lp_aaE / 3) < 1e-5
    masked = _search(UNK_TABLE, length_penalty_alpha=-1.0, top_k=2)
    allowed = _search(UNK_TABLE, length_penalty_alpha=-1.0, top_k=2, unk_id=None)
    assert sorted(h[0] for h in masked["hypotheses"].tolist()) == [A, B_]
    assert sorted(h[0] for h in allowed["hypotheses"].tolist()) == [A, UNK]


SMALL = dict(model="speech", d=64, heads=4, enc_layers=2, dec_layers=2, ffn=128, channels=64, feat=80, in_channels=1, vocab=96)


@pytest.mark.parametrize("alpha", [-1.0, 0.6])
def test_oracle_beam_one_is_greedy(alpha):
    P = U.chaotic_decode_params(R.init_params(SMALL, seed=3, random_bias=True), 4.0, 3)
    g = torch.Generator().manual_seed(3)
    src = torch.randn(2, 61, 80, 1, generator=g)
    lens = torch.tensor([61, 40])
    src[1, 40:] = 0.0
    with torch.no_grad():
        hyp, lp, ln = R.greedy_search(P, SMALL, src, lens, 94, 95, 93, maximum_decode_length=24, extra_decode_length=8)
    r = BO.speech_beam_search(P, SMALL, src, lens, 94, 95, 93, beam_size=1, length_penalty_alpha=alpha,
                              maximum_decode_length=24, extra_decode_length=8)
    assert torch.equal(r["hypotheses"], hyp) and torch.equal(r["length"], ln)
    assert torch.allclose(r["scores"], lp * BO.length_penalty(ln, alpha), rtol=1e-6)


def test_beam_args_layout_matches_the_c_header_at_abi_version_203(tmp_path):
    names = [f for f, _ in L.BeamArgs._fields_]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200st.h"', 'int main(void) {',
             '  printf("sizeof %zu\\n", sizeof(b200st_beam_args));']
    lines += ['  printf("%s %%zu\\n", offsetof(b200st_beam_args, %s));' % (n, n) for n in names]
    lines += ['  return 0;', '}']
    src = tmp_path / "beam_layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "beam_layout"
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", inc, str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    import ctypes as C
    assert int(got["sizeof"]) == C.sizeof(L.BeamArgs)
    for n in names:
        assert int(got[n]) == getattr(L.BeamArgs, n).offset, n
    assert L.ABI_VERSION == 203 and "b200st_beam_search" in L.EXPORTS and "b200st_beam_state_bytes" in L.EXPORTS


TASK_YAML = """
dataset.class: AudioTFRecordDataset
dataset.params:
  data_path: DATA
  feature_key: audio
  transcript_key: translation
task.class: SpeechToText
task.params:
  audio_feature_dim: 80
  vocab_size: 96
  batch_size: 80000
  max_src_len: 3000
  max_trg_len: 150
"""
PREDICT_YAML = """
entry: predict
entry.params:
  output_file: hyp.txt
search_method: beam_search
search_method.params:
  beam_size: 4
  length_penalty: -1
  maximum_decode_length: 180
"""


def test_predict_config_entry_alias_and_search_method(tmp_path):
    task, pred = tmp_path / "task.yml", tmp_path / "predict.yml"
    task.write_text(TASK_YAML)
    pred.write_text(PREDICT_YAML)
    paths = [str(task), str(pred)]
    plan = cli.resolve(cli.load_config(paths))
    assert plan["entry"] == "predict" and plan["search_method"] == "beam_search"
    assert plan["search"] == {"maximum_decode_length": 180, "extra_decode_length": 50, "minimum_decode_length": 0, "beam_size": 4,
                              "length_penalty": -1.0, "top_k": 1, "enable_unk": False}
    both = cli.load_config(paths)
    both["entry.class"] = "trainer"                                                       # entry.class wins over entry
    assert cli.resolve(both)["entry"] == "trainer"
    _, ov = cli.parse_command_line(["--beam_size", "2"])
    assert cli.resolve(cli.load_config(paths, ov))["search"]["beam_size"] == 2          # flat flag -> search_method.params
    _, ov = cli.parse_command_line(["--search_method", "sampling"])
    with pytest.raises(SystemExit, match="sampling"):
        cli.resolve(cli.load_config(paths, ov))
    plain = cli.resolve(cli.load_config([str(task)]))                                    # no search_method: greedy as before
    assert plain["entry"] == "trainer" and "search_method" not in plain
    assert plain["search"] == {"maximum_decode_length": 150, "extra_decode_length": 50, "minimum_decode_length": 0}


def _ptxas_table():
    from neurst_b200.csrc import build as B
    if not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available (%s)" % B.NVCC)
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, "decode.cu"), "-o",
                                                 os.path.join(tmp, "decode.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    from tests.test_kernel_resources_cpu import spill_table
    return spill_table(r.stdout + r.stderr)


def test_beam_kernels_do_not_spill():
    """The beam-search kernels and the beam variants of the attention step keep everything in registers.  The greedy
    instantiations are not listed: they compile to the same code as before this search was added (the greedy
    cross-attention step has carried a 20-byte spill since then)."""
    table = _ptxas_table()
    beam = {k: v for k, v in table.items() if re.search(r"beam_(select|init|extract)_kernel|beam1_score_kernel", k)}
    assert len(beam) == 4, sorted(beam)
    attn = {k: v for k, v in table.items() if "attn_step_kernel" in k}
    assert len(attn) == 12, sorted(attn)                                # {fp32, fp16, bf16} x {self, cross} x {greedy, beam}
    beam_attn = {k: v for k, v in attn.items() if re.search(r"Lb[01]ELb1E", k)}
    greedy_self = {k: v for k, v in attn.items() if "Lb1ELb0E" in k}
    assert len(beam_attn) == 6 and len(greedy_self) == 3
    spilled = {k: v for k, v in {**beam, **beam_attn, **greedy_self}.items() if v[1] or v[2]}
    assert not spilled, spilled
