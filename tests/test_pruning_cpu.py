"""Weight pruning, host side: the two schedules against a float32 restatement of the reference's pruning_schedule.py, the
k of a turn, the choice of the pruned variables by pattern, the trainer's flags and the C struct's layout."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from neurst_b200 import cli
from neurst_b200 import lib as L
from neurst_b200 import pruning as PR
from neurst_b200.checkpoints import tf_variable_names
from oracle import restatement as R

RECIPE = "(ln/gamma)|(ln/beta)|(modalit)"


def _ref_should(step, begin, end, freq):
    return step >= begin and (step <= end or end < 0) and (step - begin) % freq == 0


def _ref_poly(step, begin, end, initial, target, power):
    f = np.float32
    p = np.clip(f(step - begin) / f(end - begin), f(0), f(1)).astype(np.float32)
    # pruning_schedule.py:173-174: `(self._initial_sparsity - self._target_sparsity)` subtracts Python floats; the float32
    # cast happens where the result meets the float32 tensor
    return f(initial - target) * f(np.power(f(1) - p, f(power))) + f(target)


@pytest.mark.parametrize("begin,end,freq", [(0, 40, 4), (3, 17, 5), (10, 10, 1), (0, -1, 7)])
def test_constant_sparsity_turns_and_sparsity(begin, end, freq):
    s = PR.ConstantSparsity(target_sparsity=0.3, begin_pruning_step=begin, end_pruning_step=end, pruning_frequency=freq)
    for step in range(0, 60):
        assert s.should_prune_in_step(step) == _ref_should(step, begin, end, freq), step
        assert s.sparsity_in_step(step) == np.float32(0.3) and s.sparsity_in_step(step).dtype == np.float32


@pytest.mark.parametrize("begin,end,freq,initial,target,power", [(0, 500, 100, 0.0, 0.1, 3), (2, 9, 1, 0.1, 0.5, 2.5),
                                                                  (0, 4, 2, 0.0, 0.5, 3), (5, 30, 3, 0.6, 0.2, 1)])
def test_polynomial_decay_turns_and_sparsity(begin, end, freq, initial, target, power):
    s = PR.PolynomialDecay(initial_sparsity=initial, polynomial_power=power, target_sparsity=target, begin_pruning_step=begin,
                           end_pruning_step=end, pruning_frequency=freq)
    for step in list(range(0, 40)) + [end - 1, end, end + 1, 10 * end + 3]:
        assert s.should_prune_in_step(step) == _ref_should(step, begin, end, freq), step
        got = s.sparsity_in_step(step)
        assert got.dtype == np.float32 and got == _ref_poly(step, begin, end, initial, target, power), step
    assert s.sparsity_in_step(end) == np.float32(target) and abs(s.sparsity_in_step(begin) - np.float32(initial)) < 1e-7
    assert s.max_sparsity() == np.float32(max(initial, target))


def test_polynomial_difference_is_taken_in_double():
    # 0.01 - 0.3 in double then float32 is not float32(0.01) - float32(0.3): one ulp apart
    f = np.float32
    assert f(0.01 - 0.3) != f(0.01) - f(0.3)
    s = PR.PolynomialDecay(initial_sparsity=0.01, target_sparsity=0.3, end_pruning_step=10, polynomial_power=1)
    assert s.sparsity_in_step(0) == f(0.01 - 0.3) * f(1) + f(0.3)


def test_k_rounds_half_to_even_in_float32():
    # size * (1 - s) exactly on .5: banker's rounding as tf.math.round
    assert PR.k_of(5, 0.5) == 2 and PR.k_of(7, 0.5) == 4 and PR.k_of(3, 0.5) == 2 and PR.k_of(1, 0.5) == 0
    assert PR.k_of(8, 0.0) == 8 and PR.k_of(9 * 256, 0.25) == 1728
    for size in (8, 9, 100, 1023, 4096, 2 ** 21 + 3):
        for sp in (0.0, 0.1, 0.3, 0.4375, 0.5, 0.9, 0.99):
            f = np.float32
            assert PR.k_of(size, sp) == int(np.rint(f(size) * (f(1) - f(sp)))), (size, sp)
    # 0.1 in float32 is not 0.1: the product is rounded in float32, as the reference casts the size to float32
    assert PR.k_of(10, 0.3) == int(np.rint(np.float32(10) * (np.float32(1) - np.float32(0.3))))


@pytest.mark.parametrize("cls,kw,msg", [
    (PR.ConstantSparsity, dict(target_sparsity=0.1, begin_pruning_step=-1), "begin_pruning_step should be >= 0"),
    (PR.ConstantSparsity, dict(target_sparsity=0.1, begin_pruning_step=5, end_pruning_step=4), "<= end_pruning_step"),
    (PR.ConstantSparsity, dict(target_sparsity=0.1, pruning_frequency=0), "pruning_frequency should be > 0"),
    (PR.ConstantSparsity, dict(target_sparsity=1.0), "target_sparsity must be in range"),
    (PR.ConstantSparsity, dict(target_sparsity=-0.1), "target_sparsity must be in range"),
    (PR.PolynomialDecay, dict(target_sparsity=0.1, initial_sparsity=1.0, end_pruning_step=5), "initial_sparsity must be in range"),
    (PR.PolynomialDecay, dict(target_sparsity=0.1), "end_pruning_step must > 0"),
    (PR.PolynomialDecay, dict(target_sparsity=0.1, begin_pruning_step=3, end_pruning_step=3), "end_pruning_step > begin"),
])
def test_constructor_errors(cls, kw, msg):
    with pytest.raises(ValueError, match=msg.replace("(", r"\(")):
        cls(**kw)


def test_new_returns_none_at_zero_target():
    assert PR.PolynomialDecay.new(dict(target_sparsity=0)) is None          # even with end_pruning_step -1
    assert PR.build_schedule("constant_sparsity", dict(target_sparsity=0.0)) is None
    s = PR.build_schedule("polynomial_decay", dict(target_sparsity=0.3, end_pruning_step=10))
    assert isinstance(s, PR.PolynomialDecay) and s.polynomial_power == 3 and s.pruning_frequency == 100
    for name in ("ConstantSparsity", "constant_sparsity", "constantsparsity"):
        assert PR.schedule_class(name) is PR.ConstantSparsity
    for name in ("PolynomialDecay", "polynomial_decay"):
        assert PR.schedule_class(name) is PR.PolynomialDecay
    with pytest.raises(ValueError):
        PR.schedule_class("cosine")


def _names(cfg):
    table = R.param_shapes(cfg)
    return table, tf_variable_names(table)


TABLES = {"speech_transformer_s": R.CONFIGS["speech_transformer_s"],
          "transformer_big": dict(model="text", d=1024, heads=16, enc_layers=6, dec_layers=6, ffn=4096, vocab=32768,
                                  src_vocab=32768)}


@pytest.mark.parametrize("name", sorted(TABLES))
def test_recipe_pattern_excludes_exactly_layer_norms_and_modalities(name):
    table, tf = _names(TABLES[name])
    pruned = PR.pruned_parameters(table, None, RECIPE)
    excluded = [k for k in table if k not in pruned]
    is_ln = lambda k: k.endswith(".gamma") or k.endswith(".beta")                   # noqa: E731
    is_modality = lambda k: k.startswith(("src.", "srcemb.", "trg."))                # noqa: E731
    assert excluded == [k for k in table if is_ln(k) or is_modality(k)]
    assert pruned and all(k.endswith(("kernel", "bias", ".w1", ".w2", ".b1", ".b2")) for k in pruned)
    assert all("modalit" not in tf[k] and "/ln/" not in tf[k] and "output_ln" not in tf[k] for k in pruned)
    # no pattern: everything; pruning_variable_pattern wins over nopruning_variable_pattern
    assert PR.pruned_parameters(table) == list(table)
    only = PR.pruned_parameters(table, "ffn/dense1/kernel", RECIPE)
    assert only == [k for k in table if k.endswith(".ffn.w1")]


def _plan(tmp_path, overrides):
    from tests.test_cli import _write_yaml
    y = _write_yaml(tmp_path)
    return cli.resolve(cli.load_config([y], overrides))


def test_plan_parses_schedule_params_flat_flags_and_initial_global_step(tmp_path):
    plan = _plan(tmp_path, [])
    assert plan["pruning"] is None and plan["initial_global_step"] is None
    # the recipe's flat flags (examples/weight_pruning/README.md)
    ov = cli.parse_command_line(["--initial_global_step", "250000", "--pruning_schedule", "polynomial_decay", "--initial_sparsity", "0",
                                 "--target_sparsity", "0.1", "--begin_pruning_step", "0", "--end_pruning_step", "500",
                                 "--pruning_frequency", "100", "--nopruning_variable_pattern", RECIPE])[1]
    plan = _plan(tmp_path, ov)
    s = plan["pruning"]["schedule"]
    assert isinstance(s, PR.PolynomialDecay) and (s.target_sparsity, s.end_pruning_step, s.pruning_frequency) == (0.1, 500, 100)
    assert plan["pruning"]["nopruning_variable_pattern"] == RECIPE and plan["pruning"]["pruning_variable_pattern"] is None
    assert plan["initial_global_step"] == 250000
    # pruning_schedule.params (dotted), class alias, and a flat flag overriding one of its keys
    ov = cli.parse_command_line(["--pruning_schedule", "ConstantSparsity", "--pruning_schedule.params.target_sparsity", "0.2",
                                 "--pruning_schedule.params.pruning_frequency", "7", "--pruning_variable_pattern", "kernel"])[1]
    s = _plan(tmp_path, ov)["pruning"]["schedule"]
    assert isinstance(s, PR.ConstantSparsity) and s.target_sparsity == 0.2 and s.pruning_frequency == 7
    s = _plan(tmp_path, ov + [("target_sparsity", 0.4)])["pruning"]["schedule"]
    assert s.target_sparsity == 0.4
    # the default class is PolynomialDecay; target_sparsity 0 turns pruning off (no schedule: the plain optimizer step)
    s = _plan(tmp_path, [("target_sparsity", 0.5), ("end_pruning_step", 4)])["pruning"]["schedule"]
    assert isinstance(s, PR.PolynomialDecay)
    assert _plan(tmp_path, [("pruning_schedule", "polynomial_decay"), ("target_sparsity", 0)])["pruning"] is None
    for bad in ([("target_sparsity", 0.5)], [("target_sparsity", 1.5), ("end_pruning_step", 4)],
                [("pruning_schedule", "cosine"), ("target_sparsity", 0.5)],
                [("target_sparsity", 0.5), ("end_pruning_step", 4), ("nopruning_variable_pattern", "(")]):
        with pytest.raises(SystemExit):
            _plan(tmp_path, bad)


class _RecordingRuntime:
    """The surface of Runtime that DataParallelTrainer uses, recording the optimizer calls instead of running them."""

    def __init__(self):
        import torch
        self.config = type("Cfg", (), {"d": 8})()
        self.table = {"a": (0, (8,)), "b": (8, (4,))}
        self.grads = torch.zeros(16)
        self.setups, self.steps = [], []

    def ensure_grads(self):
        return self.grads

    def prune_setup(self, schedule, names):
        self.setups.append((schedule, list(names)))

    def adam_step(self, lr, step_t, *args, **kw):
        self.steps.append((step_t, kw.get("prune")))


def _recording_trainer(**kw):
    import torch
    from neurst_b200.trainer import DataParallelTrainer
    rt = _RecordingRuntime()
    model = type("Model", (), {"runtime": rt, "forward_backward": lambda self, b, **k: {"loss": torch.zeros(1)}})()
    return rt, DataParallelTrainer(model, **kw)


def test_zero_sparsity_trainer_keeps_the_plain_optimizer_step():
    """A schedule with target_sparsity 0 is no pruning: the trainer keeps no schedule, sets nothing up and calls the plain
    optimizer step (no `prune`); a schedule with a target sets up the pruned tensors once and passes itself to every step."""
    batch = {"src": np.zeros((1, 2)), "trg_input": np.zeros((1, 2))}
    for zero in (PR.ConstantSparsity(target_sparsity=0.0), PR.PolynomialDecay(initial_sparsity=0.5, end_pruning_step=4)):
        rt, tr = _recording_trainer(pruning_schedule=zero)
        assert tr.pruning_schedule is None
        for _ in range(3):
            tr.train_step(batch)
        assert rt.setups == [] and rt.steps == [(1, None), (2, None), (3, None)]
    sched = PR.ConstantSparsity(target_sparsity=0.3)
    rt, tr = _recording_trainer(pruning_schedule=sched, update_cycle=2)
    for _ in range(4):
        tr.train_step(batch)
    assert rt.setups == [(sched, ["a", "b"])] and rt.steps == [(1, sched), (2, sched)]
    # initial_global_step: the noam position moves, Adam's t counts this run's updates
    rt, tr = _recording_trainer(lr_schedule_params=dict(dmodel=8, warmup_steps=4000))
    tr.global_step = tr.adam_step_base = 1000
    tr.train_step(batch)
    assert tr.global_step == 1001 and rt.steps == [(1, None)]


def test_prune_args_layout_matches_the_c_header(tmp_path):
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200st.h"', 'int main(void) {',
             '  printf("sizeof %zu\\n", sizeof(b200st_prune_args));']
    for fname, _ in L.PruneArgs._fields_:
        lines.append('  printf("%s %%zu\\n", offsetof(b200st_prune_args, %s));' % (fname, fname))
    lines += ['  printf("max %d %d %d\\n", B200ST_PRUNE_MAX_TENSORS, B200ST_PRUNE_CONSTANT, B200ST_PRUNE_POLYNOMIAL);',
              '  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", inc, str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    got = {l.split()[0]: l.split()[1:] for l in out}
    assert int(got["sizeof"][0]) == C.sizeof(L.PruneArgs) == 96
    for fname, _ in L.PruneArgs._fields_:
        assert int(got[fname][0]) == getattr(L.PruneArgs, fname).offset, fname
    assert [int(x) for x in got["max"]] == [L.PRUNE_MAX_TENSORS, L.PRUNE_CONSTANT, L.PRUNE_POLYNOMIAL]
    lib = L.load()
    assert lib.b200st_prune_scratch_bytes(3) == 4 * (1152 + 3 * 2048) and lib.b200st_prune_scratch_bytes(0) == -1
