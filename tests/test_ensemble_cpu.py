"""Ensemble decoding without a GPU: the b200st_ensemble_member layout against the C header, the exported symbol, the
`predict` plan for several model_dirs (ensemble_weights: default, normalisation, the reference's count error; `train`
refuses several directories), and the compiler's resource report of the mixing kernel and of beam_select_kernel on
log-probabilities."""
import ctypes as C
import os
import subprocess
import tempfile

import pytest

from neurst_b200 import cli
from neurst_b200 import decode as D
from neurst_b200 import lib as L
from tests.test_beam_search_cpu import PREDICT_YAML, TASK_YAML

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ensemble_member_layout_matches_the_c_header(tmp_path):
    names = [f for f, _ in L.EnsembleMember._fields_]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200st.h"', 'int main(void) {',
             '  printf("sizeof %zu\\n", sizeof(b200st_ensemble_member));',
             '  printf("max %d\\n", B200ST_ENSEMBLE_MAX_MODELS);']
    lines += ['  printf("%s %%zu\\n", offsetof(b200st_ensemble_member, %s));' % (n, n) for n in names]
    lines += ['  return 0;', '}']
    src = tmp_path / "ensemble_layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "ensemble_layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["sizeof"]) == C.sizeof(L.EnsembleMember)
    for n in names:
        assert int(got[n]) == getattr(L.EnsembleMember, n).offset, n
    assert int(got["max"]) == L.ENSEMBLE_MAX_MODELS == 8


def test_symbol_exported_at_abi_version_203():
    assert "b200st_ensemble_beam_search" in L.EXPORTS and L.ABI_VERSION == 203


def test_ensemble_weights():
    assert D.ensemble_weights("average", 4) == [0.25] * 4
    assert D.ensemble_weights("0.6,0.2", 2) == pytest.approx([0.75, 0.25])
    assert D.ensemble_weights([3, 1], 2) == pytest.approx([0.75, 0.25])
    assert D.ensemble_weights(2.0, 1) == [1.0]
    with pytest.raises(ValueError, match="The number of manual weights must have equal to the models."):
        D.ensemble_weights("0.5,0.3,0.2", 2)


def _plan(tmp_path, overrides=(), predict=True):
    task, pred = tmp_path / "task.yml", tmp_path / "predict.yml"
    task.write_text(TASK_YAML)
    pred.write_text(PREDICT_YAML)
    paths = [str(task)] + ([str(pred)] if predict else [])
    _, ov = cli.parse_command_line(list(overrides))
    return cli.resolve(cli.load_config(paths, ov))


def test_predict_plan_for_several_model_dirs(tmp_path):
    single = _plan(tmp_path, ["--model_dir", "/m/a"])
    assert single["model_dir"] == "/m/a" and "ensemble_weights" not in single           # as before
    plan = _plan(tmp_path, ["--model_dir", "/m/a, /m/b,"])
    assert plan["model_dir"] == ["/m/a", "/m/b"] and plan["ensemble_weights"] == [0.5, 0.5]
    listed = tmp_path / "dirs.yml"
    listed.write_text("model_dir:\n  - /m/a\n  - /m/b,/m/c\n")
    plan = cli.resolve(cli.load_config([str(tmp_path / "task.yml"), str(tmp_path / "predict.yml"), str(listed)]))
    assert plan["model_dir"] == ["/m/a", "/m/b", "/m/c"] and plan["ensemble_weights"] == pytest.approx([1 / 3] * 3)
    plan = _plan(tmp_path, ["--model_dir", "/m/a,/m/b", "--ensemble_weights", "0.6,0.2"])          # flat flag -> entry.params
    assert plan["ensemble_weights"] == pytest.approx([0.75, 0.25])
    plan = _plan(tmp_path, ["--model_dir", "/m/a,/m/b", "--ensemble_weights", "0.6,0.2",
                            "--search_method.params.ensemble_weights", "1,3"])                     # search_method.params first
    assert plan["ensemble_weights"] == pytest.approx([0.25, 0.75])
    with pytest.raises(SystemExit, match="equal to the models"):
        _plan(tmp_path, ["--model_dir", "/m/a,/m/b", "--ensemble_weights", "0.5,0.3,0.2"])
    with pytest.raises(SystemExit, match="one model_dir"):
        _plan(tmp_path, ["--model_dir", "/m/a,/m/b"], predict=False)                               # train


def test_member_architecture_from_model_configs(tmp_path):
    import yaml
    plan = _plan(tmp_path, ["--model_dir", str(tmp_path / "a") + "," + str(tmp_path / "b")])
    a = dict(plan, model_dir=str(tmp_path / "a"), model_params=dict(plan["model_params"], **{"decoder.num_layers": 3}))
    cli.write_model_configs(a)
    written = yaml.safe_load(open(tmp_path / "a" / "model_configs.yml"))
    assert written["model.class"] == "SpeechTransformer" and written["model.params"]["decoder.num_layers"] == 3
    assert cli.member_model_params(plan, str(tmp_path / "a"))["decoder.num_layers"] == 3
    assert cli.member_model_params(plan, str(tmp_path / "b")) == plan["model_params"]              # no file: the run's


def test_mixing_and_log_probability_selection_kernels_do_not_spill():
    from neurst_b200.csrc import build as B
    from tests.test_kernel_resources_cpu import spill_table
    if not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available (%s)" % B.NVCC)
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, "ensemble.cu"), "-o",
                                                 os.path.join(tmp, "ensemble.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    table = spill_table(r.stdout + r.stderr)
    mix = {k: v for k, v in table.items() if "ensemble_logprob_kernel" in k}
    select = {k: v for k, v in table.items() if "beam_select_kernelILb1E" in k}
    assert len(mix) == 1 and len(select) == 1, sorted(table)
    assert not any(v[0] or v[1] or v[2] for v in {**mix, **select}.values()), {**mix, **select}
