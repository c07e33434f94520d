"""Prune-Tune without a GPU: the entries' plans and flags, their refusals, the mask file (round trip, refusals, packing into the
device bitmap against a hand-built one), the trainer's partial-tuning wiring and the ctypes signatures of the new symbols."""
import ctypes as C
import os
import pickle
import subprocess
import types

import numpy as np
import pytest

from neurst_b200 import cli
from neurst_b200 import lib as L
from neurst_b200 import prune_tune as PT
from neurst_b200 import pruning as PR
from neurst_b200.checkpoints import tf_variable_names
from oracle import restatement as R

RECIPE = "(ln/gamma)|(ln/beta)|(modalit)"


def _plan(tmp_path, argv):
    from tests.test_cli import _write_yaml
    y = _write_yaml(tmp_path)
    paths, ov = cli.parse_command_line(["--config_paths", y] + argv)
    return cli.resolve(cli.load_config(paths, ov))


def _mask_file(tmp_path, name="mask.pkl"):
    path = tmp_path / name
    path.write_bytes(b"PK\x03\x04")
    return str(path)


def test_bare_partial_tuning_include_and_the_entries(tmp_path):
    mask = _mask_file(tmp_path)
    # the README's command line: --include, then --partial_tuning bare in the middle and at the end
    for argv in (["--include", "examples/prune_tune/src/", "--entry", "prune_tune_train", "--partial_tuning", "--mask_pkl", mask],
                 ["--include", "examples/prune_tune/src/", "--entry", "prune_tune_train", "--mask_pkl", mask, "--partial_tuning"]):
        paths, ov = cli.parse_command_line(argv)
        assert ("partial_tuning", True) in ov and all(k != "include" for k, _ in ov)
        plan = _plan(tmp_path, argv)
        assert plan["entry"] == "prune_tune_train" and plan["entry"] in cli.TRAIN_ENTRIES
        assert plan["prune_tune"] == {"partial_tuning": True, "mask_pkl": mask}
    # the flags around it still take their values
    paths, ov = cli.parse_command_line(["--partial_tuning", "--train_steps", "10", "--summary_steps=3"])
    assert ov == [("partial_tuning", True), ("train_steps", 10), ("summary_steps", 3)]
    assert cli.parse_command_line(["--partial_tuning=false"])[1] == [("partial_tuning", False)]
    # prune_tune_train without the flags: the pruning half of the recipe
    ov = ["--entry", "prune_tune_train", "--pruning_schedule", "ConstantSparsity", "--target_sparsity", "0.1",
          "--nopruning_variable_pattern", RECIPE]
    plan = _plan(tmp_path, ov)
    assert plan["prune_tune"] == {"partial_tuning": False, "mask_pkl": None} and plan["pruning"]["schedule"].target_sparsity == 0.1
    # the other entries carry no Prune-Tune flags; mask_predict / mask_generation carry mask_pkl
    assert _plan(tmp_path, [])["prune_tune"] is None and _plan(tmp_path, ["--entry", "predict"])["prune_tune"] is None
    for entry in ("mask_predict", "mask_generation"):
        plan = _plan(tmp_path, ["--entry", entry, "--mask_pkl", mask])
        assert plan["entry"] in cli.PREDICT_ENTRIES and plan["prune_tune"] == {"mask_pkl": mask}
        assert _plan(tmp_path, ["--entry", entry])["prune_tune"] == {"mask_pkl": None}
        # without mask_pkl an ensemble is a plain ensemble predict
        plan = _plan(tmp_path, ["--entry", entry, "--model_dir", "a,b"])
        assert plan["model_dir"] == ["a", "b"] and plan["ensemble_weights"] == [0.5, 0.5]


def test_entry_refusals(tmp_path):
    mask = _mask_file(tmp_path)
    prune = ["--pruning_schedule", "ConstantSparsity", "--target_sparsity", "0.1"]
    with pytest.raises(SystemExit, match="partial_tuning together with a pruning schedule"):
        _plan(tmp_path, ["--entry", "prune_tune_train", "--partial_tuning"] + prune)
    with pytest.raises(SystemExit, match="takes one model_dir"):
        _plan(tmp_path, ["--entry", "mask_predict", "--model_dir", "a,b", "--mask_pkl", mask])
    for entry in ("mask_predict", "prune_tune_train"):
        with pytest.raises(SystemExit, match="no such file"):
            _plan(tmp_path, ["--entry", entry, "--mask_pkl", str(tmp_path / "missing.pkl"), "--partial_tuning"])
    from neurst_b200.trainer import DataParallelTrainer
    rt = _RecordingRuntime()
    model = types.SimpleNamespace(runtime=rt)
    with pytest.raises(ValueError, match="pruning schedule"):
        DataParallelTrainer(model, pruning_schedule=PR.ConstantSparsity(target_sparsity=0.2), partial_tuning_mask="weights")


# ---- the mask file and the device bitmap ---------------------------------------------------------------------------------
class _HostRuntime:
    """A Runtime's table, arena and bitmap builders on the host (the layout of the device arena: every tensor at a multiple
    of 8 elements)."""
    from neurst_b200.runtime import Runtime as _R
    derive_prune_mask = _R.derive_prune_mask
    mask_counts = _R.mask_counts
    _numel_of = _R._numel_of

    def __init__(self, cfg):
        import torch
        self.table, off = {}, 0
        for k, shape in R.param_shapes(cfg).items():
            self.table[k] = (off, tuple(shape))
            off += (int(np.prod(shape)) + 7) // 8 * 8
        self.numel = off + 16                        # an arena tail outside every tensor
        self.device = torch.device("cpu")
        self.params = torch.zeros(self.numel)


# odd sizes everywhere: the tables and biases of these vocabularies are no multiples of 8 elements
TEXT = dict(model="text", d=12, heads=2, enc_layers=1, dec_layers=1, ffn=20, vocab=13, src_vocab=11)
SPEECH = dict(model="speech", d=12, heads=2, enc_layers=1, dec_layers=1, ffn=20, vocab=13, channels=3, feat=9, in_channels=1)


def _random_masks(rt, seed):
    rng = np.random.default_rng(seed)
    return {k: (rng.random(shape) < 0.7).astype(np.uint8) for k, (_, shape) in rt.table.items()}


def _hand_bitmap(rt, masks):
    bits = np.ones(rt.numel, dtype=np.uint8)
    for k, (off, shape) in rt.table.items():
        bits[off:off + int(np.prod(shape))] = masks[k].reshape(-1)
    out = np.zeros(rt.numel // 8, dtype=np.uint8)
    for j in range(8):
        out |= (bits[j::8] << j).astype(np.uint8)
    return out


@pytest.mark.parametrize("cfg", [TEXT, SPEECH], ids=["text", "speech"])
def test_mask_file_round_trip_and_packing(tmp_path, cfg):
    rt = _HostRuntime(cfg)
    assert any(int(np.prod(s)) % 8 for _, s in rt.table.values())
    masks = _random_masks(rt, 1)
    bitmap = PT.mask_bitmap(rt, masks)
    assert np.array_equal(bitmap.numpy(), _hand_bitmap(rt, masks))
    frozen = sum(int(m.sum()) for m in masks.values())
    total = sum(m.size for m in masks.values())
    assert rt.mask_counts(bitmap) == (total - frozen, frozen)
    path = str(tmp_path / "mask.pkl")
    names = PT.save_masks(rt, path, bitmap)
    assert os.path.isfile(path) and not os.path.exists(path + ".npz")
    assert names == sorted(tf_variable_names(rt.table).values())
    z = np.load(path, allow_pickle=False)
    for k, v in tf_variable_names(rt.table).items():
        assert z[v].dtype == np.uint8 and np.array_equal(z[v], masks[k]), k
    back = PT.load_masks(rt, path)
    assert sorted(back) == sorted(masks) and all(np.array_equal(back[k], masks[k]) for k in masks)
    # the weight != 0 case goes through the same builder
    import torch
    for k, (off, shape) in rt.table.items():
        n = int(np.prod(shape))
        rt.params[off:off + n] = torch.from_numpy(masks[k].reshape(-1).astype(np.float32)) * 0.5
    assert np.array_equal(rt.derive_prune_mask(list(rt.table)).numpy(), bitmap.numpy())
    # an archive under another top-level scope (a model saved under its own name) is read as load_npz reads it
    other = {v.replace(v.split("/")[0], "Renamed", 1): z[v] for v in z.files}
    np.savez(str(tmp_path / "other.npz"), **other)
    back = PT.load_masks(rt, str(tmp_path / "other.npz"))
    assert all(np.array_equal(back[k], masks[k]) for k in masks)


def test_mask_file_refusals(tmp_path):
    rt = _HostRuntime(TEXT)
    masks = _random_masks(rt, 2)
    tf = tf_variable_names(rt.table)
    good = {tf[k]: v for k, v in masks.items()}

    def write(arrays, name):
        path = str(tmp_path / name)
        with open(path, "wb") as f:
            np.savez(f, **arrays)
        return path

    with pytest.raises(PT.MaskFileError, match="no such file"):
        PT.load_masks(rt, str(tmp_path / "none.pkl"))
    real = tmp_path / "real.pkl"
    with open(real, "wb") as f:
        pickle.dump([np.ones(3)], f)
    with pytest.raises(PT.MaskFileError, match="TensorFlow variables"):
        PT.load_masks(rt, str(real))
    name = sorted(good)[0]
    with pytest.raises(PT.MaskFileError, match="misses the masks of 1 variables"):
        PT.load_masks(rt, write({k: v for k, v in good.items() if k != name}, "missing.pkl"))
    with pytest.raises(PT.MaskFileError, match="does not have"):
        PT.load_masks(rt, write(dict(good, **{name.split("/")[0] + "/extra/kernel": np.ones(3, np.uint8)}), "extra.pkl"))
    with pytest.raises(PT.MaskFileError, match="shape"):
        PT.load_masks(rt, write(dict(good, **{name: good[name].reshape(-1)[:-1]}), "shape.pkl"))
    two = good[name].copy()
    two.flat[3] = 2
    with pytest.raises(PT.MaskFileError, match="other than 0 and 1"):
        PT.load_masks(rt, write(dict(good, **{name: two}), "two.pkl"))
    # bool and float 0/1 arrays are masks too
    back = PT.load_masks(rt, write({k: v.astype(bool) if i % 2 else v.astype(np.float32) for i, (k, v) in enumerate(good.items())},
                                   "kinds.pkl"))
    assert all(np.array_equal(back[k], masks[k]) and back[k].dtype == np.uint8 for k in masks)


# ---- the trainer's wiring ------------------------------------------------------------------------------------------------
class _RecordingRuntime:
    """The surface of Runtime that DataParallelTrainer uses, recording the optimizer calls instead of running them."""

    def __init__(self):
        import torch
        self.config = types.SimpleNamespace(d=8)
        self.table = {"a": (0, (8,)), "b": (8, (4,))}
        self.grads = torch.zeros(16)
        self.derived, self.setups, self.steps = [], [], []

    def ensure_grads(self):
        return self.grads

    def derive_prune_mask(self, names=None, source=None):
        self.derived.append((list(names), source))
        return "bitmap%d" % len(self.derived)

    def partial_setup(self, bitmap):
        self.setups.append(bitmap)
        self.partial_frozen = bitmap
        return (3, 9)

    def adam_step(self, lr, step_t, *args, **kw):
        self.steps.append((step_t, kw.get("frozen"), kw.get("prune")))


def test_trainer_sets_up_the_frozen_bitmap_once_and_passes_it_to_every_step():
    import torch
    from neurst_b200.trainer import DataParallelTrainer
    batch = {"src": np.zeros((1, 2)), "trg_input": np.zeros((1, 2))}
    for source in ("weights", {"a": np.ones(8), "b": np.zeros(4)}):
        rt = _RecordingRuntime()
        model = types.SimpleNamespace(runtime=rt, forward_backward=lambda b, **k: {"loss": torch.zeros(1)})
        tr = DataParallelTrainer(model, update_cycle=2, partial_tuning_mask=source)
        assert rt.setups == []                                   # nothing before the broadcast
        assert tr.setup_partial_tuning() == (3, 9) and tr.setup_partial_tuning() == (3, 9)
        for _ in range(4):
            tr.train_step(batch)
        assert rt.derived == [(["a", "b"], None if source == "weights" else source)] and rt.setups == ["bitmap1"]
        assert rt.steps == [(1, "bitmap1", None), (2, "bitmap1", None)]
    rt = _RecordingRuntime()
    tr = DataParallelTrainer(types.SimpleNamespace(runtime=rt, forward_backward=lambda b, **k: {"loss": torch.zeros(1)}))
    tr.train_step(batch)
    assert tr.setup_partial_tuning() is None and rt.steps == [(1, None, None)]
    with pytest.raises(ValueError):
        DataParallelTrainer(types.SimpleNamespace(runtime=rt), partial_tuning_mask="zeros")


# ---- the C interface -----------------------------------------------------------------------------------------------------
def test_step_and_mask_ctypes_signatures_match_the_header(tmp_path):
    """The header's prototypes, assigned to pointers of the types the ctypes declarations spell out (gcc -Werror refuses any
    difference), and the declarations themselves."""
    src = tmp_path / "sig.c"
    src.write_text("\n".join([
        '#include <stdint.h>', '#include "b200st.h"',
        'int (*step)(b200st_handle, const b200st_optim_args*, void*) = b200st_optimizer_step;',
        'int (*masking)(float*, void*, int, const uint8_t*, int64_t, void*) = b200st_apply_mask;',
        'int main(void) { return step == 0 || masking == 0; }']))
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-c", "-I", inc, str(src), "-o", str(tmp_path / "sig.o")], check=True)
    lib = L.load()
    assert {"b200st_optimizer_step", "b200st_apply_mask"} <= set(L.EXPORTS)
    assert lib.b200st_optimizer_step.argtypes == [C.c_void_p, C.POINTER(L.OptimArgs), C.c_void_p]
    assert lib.b200st_apply_mask.argtypes == [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p]
    assert lib.b200st_optimizer_step.restype is C.c_int and lib.b200st_apply_mask.restype is C.c_int
