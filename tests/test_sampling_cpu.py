"""Top-k / nucleus sampling without a GPU: the b200st_sampling_args layout against the C header and the exported symbols,
the numpy Philox4x32-7 of the test oracle against common.cuh's host function, the `predict` plans of search_method
top_sampling (names, defaults, the reference's two errors, the ensemble and validator refusals, the row limits), and the
compiler's resource report of the selection kernel."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from neurst_b200 import cli
from neurst_b200 import lib as L
from tests import sampling_oracle as SO
from tests.test_beam_search_cpu import TASK_YAML

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sampling_args_layout_matches_the_c_header(tmp_path):
    names = [f for f, _ in L.SamplingArgs._fields_]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200st.h"', 'int main(void) {',
             '  printf("sizeof %zu\\n", sizeof(b200st_sampling_args));']
    lines += ['  printf("%s %%zu\\n", offsetof(b200st_sampling_args, %s));' % (n, n) for n in names]
    lines += ['  return 0;', '}']
    src = tmp_path / "sampling_layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "sampling_layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["sizeof"]) == C.sizeof(L.SamplingArgs)
    for n in names:
        assert int(got[n]) == getattr(L.SamplingArgs, n).offset, n
    assert names == ["bos_ids", "eos_id", "unk_id", "min_len", "max_steps", "sample_num", "top_k", "top_p", "seed", "row_offset",
                     "out_ids", "out_logprob", "out_len", "state_words", "use_graph"]


def test_symbols_exported_at_abi_version_203():
    header = open(os.path.join(ROOT, "include", "b200st.h")).read()
    for sym in ("b200st_sampling_search", "b200st_sample_logits"):
        assert sym in L.EXPORTS and re.search(r"\b%s\s*\(" % sym, header), sym
        assert hasattr(L.load(), sym), sym
    assert L.ABI_VERSION == 203


def test_numpy_philox_matches_the_library_generator(tmp_path):
    """The oracle's Philox4x32-7 gives the words of common.cuh's philox4x32 (a host-only program built with nvcc)."""
    from neurst_b200.csrc import build as B
    if not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available (%s)" % B.NVCC)
    cases = [(0, 0, 0), (1234, 0, 0), (1234, 7, 3), (0xFFFFFFFFFFFFFFFF, 0xFFFFFFFF, 255), (0x9E3779B97F4A7C15, 1 << 40, 1 << 33),
             (42, 199, 123456789)]
    body = "\n".join('  p(%duLL, %duLL, %duLL);' % c for c in cases)
    src = tmp_path / "philox.cu"
    src.write_text('#include "common.cuh"\n'
                   'static void p(uint64_t s, uint64_t c, uint64_t k) {\n'
                   '  const b200st::Philox4 r = b200st::philox4x32(s, c, k);\n'
                   '  printf("%u %u %u %u\\n", r.x, r.y, r.z, r.w);\n}\n'
                   'int main() {\n' + body + '\n  return 0;\n}\n')
    exe = tmp_path / "philox"
    r = subprocess.run([B.NVCC, "-std=c++17", "-I", B.HERE, str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    for (s, c, k), line in zip(cases, out):
        want = [int(x) for x in line.split()]
        got = [int(w) for w in SO.philox4x32(np.uint64(s), np.uint64(c), np.uint64(k))]
        assert got == want, (s, c, k, got, want)
    u = SO.uniforms(1234, 5, np.arange(4, dtype=np.uint64))
    assert u.shape == (4,) and bool(((u >= 0) & (u < 1)).all())


def test_filter_restatement():
    z = np.array([[3.0, 1.0, 2.0, 2.0, 0.0, -1.0]])
    keep, margin = SO.filter_keep(z, top_k=3)
    assert keep.tolist() == [[True, False, True, True, False, False]] and margin == 1.0
    keep, margin = SO.filter_keep(z, top_k=2)                                                 # k-th value 2: its tie is kept too
    assert keep.tolist() == [[True, False, True, True, False, False]] and margin == 0.0
    keep, _ = SO.filter_keep(z, top_p=1e-9)
    assert keep.tolist() == [[True, False, False, False, False, False]]
    keep, _ = SO.filter_keep(z, top_p=0.5)                                                    # p(3) = 0.516
    assert keep.tolist() == [[True, False, False, False, False, False]]
    keep, _ = SO.filter_keep(z, top_p=0.8)                                                    # 0.516 + 2 x 0.190 = 0.895
    assert keep.tolist() == [[True, False, True, True, False, False]]
    keep, _ = SO.filter_keep(z, top_p=0.9)                                                    # + 0.070 = 0.965
    assert keep.tolist() == [[True, True, True, True, False, False]]
    keep = SO.filter_keep(z)[0]
    assert SO.draw(z, keep, np.array([0.0]))[0].tolist() == [0]
    assert SO.draw(z, keep, np.array([0.6]))[0].tolist() == [2]                               # running sums 0.516, 0.586, 0.775


PREDICT = """
entry: predict
search_method: SEARCH
search_method.params:
  maximum_decode_length: 120
"""


def _plan(tmp_path, method="top_sampling", overrides=(), extra=None):
    task, pred = tmp_path / "task.yml", tmp_path / "predict.yml"
    task.write_text(TASK_YAML)
    pred.write_text(PREDICT.replace("SEARCH", method))
    paths = [str(task), str(pred)]
    if extra:
        (tmp_path / "extra.yml").write_text(extra)
        paths.append(str(tmp_path / "extra.yml"))
    _, ov = cli.parse_command_line(list(overrides))
    return cli.resolve(cli.load_config(paths, ov))


@pytest.mark.parametrize("name", ["top_sampling", "TopSampling", "topsampling"])
def test_top_sampling_plan_and_defaults(tmp_path, name):
    plan = _plan(tmp_path, name)
    assert plan["search_method"] == "top_sampling"
    assert plan["search"] == {"maximum_decode_length": 120, "extra_decode_length": 50, "minimum_decode_length": 0, "sample_num": 1,
                              "top_k": 0, "top_p": 1.0}
    plan = _plan(tmp_path, name, ["--sample_num", "4", "--top_p", "0.9", "--random_seed", "7"])      # flat flags
    assert (plan["search"]["sample_num"], plan["search"]["top_p"], plan["seed"]) == (4, 0.9, 7)
    plan = _plan(tmp_path, name, ["--search_method.params.top_k", "10", "--minimum_decode_length", "5"])
    assert (plan["search"]["top_k"], plan["search"]["minimum_decode_length"]) == (10, 5)


def test_reference_errors_and_refusals(tmp_path):
    with pytest.raises(SystemExit, match="Not implemented search logic when top_k > 0 and top_p < 1."):
        _plan(tmp_path, overrides=["--search_method.params.top_k", "5", "--search_method.params.top_p", "0.9"])
    with pytest.raises(SystemExit, match="minimum_decode_length` must be less than maximum decode length"):
        _plan(tmp_path, overrides=["--search_method.params.minimum_decode_length", "120"])
    with pytest.raises(SystemExit, match="sample_num"):
        _plan(tmp_path, overrides=["--search_method.params.sample_num", "9"])
    with pytest.raises(SystemExit, match="'sampling'"):
        _plan(tmp_path, "sampling")
    with pytest.raises(SystemExit, match="top_sampling.*ensemble"):
        _plan(tmp_path, overrides=["--model_dir", "/m/a,/m/b"])
    assert _plan(tmp_path, "beam_search", ["--model_dir", "/m/a,/m/b"])["ensemble_weights"] == [0.5, 0.5]     # as before
    validator = ("validator: SeqGenerationValidator\nvalidator.params:\n  eval_dataset: AudioTFRecordDataset\n"
                 "  eval_dataset.params: {data_path: DEV}\n  eval_search_method: top_sampling\n")
    with pytest.raises(SystemExit, match="eval_search_method 'top_sampling' is outside this path"):
        _plan(tmp_path, "beam_search", extra=validator)


def test_rows_per_call(tmp_path):
    # fp32 weights: 8 rows per step
    per_call, kw = cli.decode_settings(_plan(tmp_path, overrides=["--sample_num", "4", "--dtype", "float32"]))
    assert per_call == 2 and "use_shadow" not in kw and kw["sample_num"] == 4
    assert cli.decode_settings(_plan(tmp_path, overrides=["--sample_num", "8", "--dtype", "float32"]))[0] == 1
    plan = _plan(tmp_path, overrides=["--sample_num", "4", "--dtype", "float32"], extra="batch_size: 64\n")
    assert cli.decode_settings(plan)[0] == 2                                       # batch_size is capped by the 8 rows
    # 16-bit weights: batch_size x sample_num up to 256 rows, one call per batch
    per_call, kw = cli.decode_settings(_plan(tmp_path, overrides=["--sample_num", "4"], extra="batch_size: 64\n"))
    assert per_call == 64 and kw["use_shadow"]
    with pytest.raises(SystemExit, match="batch_size 65 x sample_num 4 exceeds the 256 rows"):
        cli.decode_settings(_plan(tmp_path, overrides=["--sample_num", "4"], extra="batch_size: 65\n"))


def test_sampling_seed_folds_the_rank_in():
    assert cli.sampling_seed(1234, 0) == 1234
    seeds = {cli.sampling_seed(1234, r) for r in range(8)}
    assert len(seeds) == 8 and all(0 <= s < 2 ** 64 for s in seeds)


def test_selection_kernel_does_not_spill():
    from neurst_b200.csrc import build as B
    from tests.test_kernel_resources_cpu import spill_table
    if not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available (%s)" % B.NVCC)
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, "sampling.cu"), "-o",
                                                 os.path.join(tmp, "sampling.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    table = {k: v for k, v in spill_table(r.stdout + r.stderr).items() if "sample_" in k}
    select = {k: v for k, v in table.items() if "sample_select_kernel" in k}
    assert len(select) == 2 and len(table) == 3, sorted(table)               # search / caller logits, and the init kernel
    assert not any(v[0] or v[1] or v[2] for v in table.values()), table
