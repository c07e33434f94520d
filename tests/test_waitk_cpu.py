"""Wait-k simultaneous translation without a GPU: WaitkTranslation plans (wait_k as an int, a list, a YAML string), the
waitk_transformer_* presets, predict's override order and the refusals; the fp64 restatement of the monotonic encoder and
the wait-k cross-attention mask (the masks against a direct construction, the encoder's prefix property); the offline
latency metrics; and spill-free kernels."""
import os
import re
import subprocess
import tempfile

import pytest
import torch
import yaml

from neurst_b200 import cli
from neurst_b200 import metrics as MT
from neurst_b200.models import parse_wait_k, transformer_hparams, waitk_transformer_hparams
from oracle import restatement as R
from tests.test_mt_cpu import _mt_cfg
from tests.waitk_oracle import lagged_bias, monotonic_padding, waitk_memory_bias


# ------------------------------------------------------------------------------------------------ restated masks
@pytest.mark.parametrize("k", [1, 3, 9, 40])
def test_restated_waitk_mask_is_band_part_with_padding(k):
    Lq, Tm = 7, 9
    padding = torch.zeros(3, Tm, dtype=torch.float64)
    padding[1, 6:] = 1.0
    padding[2, 2:] = 1.0
    got = waitk_memory_bias(padding, Lq, k)
    band = torch.ones(Lq, Tm, dtype=torch.float64).tril(k - 1)        # band_part(ones, -1, k-1): j <= i + k - 1
    for b in range(3):
        for i in range(Lq):
            for j in range(Tm):
                visible = band[i, j] == 1 and padding[b, j] == 0
                assert float(got[b, i, j]) == (0.0 if visible else R.FLOAT_MIN)
    if k >= Tm:
        assert torch.equal(got, waitk_memory_bias(padding, Lq, 0))


@pytest.mark.parametrize("k", [0, 1, 3, 40])
def test_search_step_bias_is_the_teacher_forced_row(k):
    """The searches' step-t bias (lagged_bias) is row t of the teacher-forced wait-k bias."""
    padding = torch.zeros(2, 9, dtype=torch.float64)
    padding[1, 5:] = 1.0
    full = waitk_memory_bias(padding, 12, k)
    for t in range(12):
        assert torch.equal(lagged_bias(R.input_padding_to_bias(padding), k, t)[:, 0], full[:, t])


def test_monotonic_bias_is_min_of_padding_and_lower_triangle():
    padding = torch.tensor([[0., 0., 0., 1.], [0., 0., 0., 0.]], dtype=torch.float64)
    bias = R.input_padding_to_bias(monotonic_padding(padding))
    want = torch.minimum(R.input_padding_to_bias(padding)[:, None, :], R.lower_triangle_attention_bias(4, torch.float64)[0])
    assert torch.equal(bias, want)


def test_monotonic_encoder_prefix_does_not_depend_on_later_tokens():
    cfg = dict(model="text", d=32, heads=4, enc_layers=2, dec_layers=1, ffn=64, vocab=40, src_vocab=37)
    P = {k: v.double() for k, v in R.init_params(cfg, seed=3, random_bias=True).items()}
    g = torch.Generator().manual_seed(4)
    src = torch.randint(0, 37, (2, 11), generator=g)
    padding = torch.zeros(2, 11, dtype=torch.float64)
    padding[1, 8:] = 1.0

    def enc(s):
        return R.encoder(P, R.add_position(P["srcemb.emb"][s]), monotonic_padding(padding), cfg["enc_layers"], cfg["heads"])
    base = enc(src)
    for n in (1, 4, 7):
        changed = src.clone()
        changed[:, n:] = torch.randint(0, 37, changed[:, n:].shape, generator=g)
        other = enc(changed)
        assert torch.equal(other[:, :n], base[:, :n])
        assert not torch.equal(other[:, n:], base[:, n:])


# ------------------------------------------------------------------------------------------------ plans
def _waitk_cfg(tmp_path, wait_k=3, **extra):
    cfg = _mt_cfg(tmp_path, **{"task.class": "WaitkTranslation", "hparams_set": "waitk_transformer_s"})
    if wait_k is not None:
        cfg["task.params"]["wait_k"] = wait_k
    cfg.update(extra)
    return cfg


@pytest.mark.parametrize("value, want", [(3, 3), ([3, 5, 7], [3, 5, 7]), ("[1, 3]", [1, 3]), ("4", 4)])
def test_waitk_translation_plan_parses_wait_k(tmp_path, value, want):
    plan = cli.resolve(_waitk_cfg(tmp_path, value))
    assert plan["wait_k"] == want and plan["model_class"] == "Transformer"
    assert plan["model_params"]["encoder.attention_monotonic"] is True
    assert plan["task_config"] == {"task.class": "WaitkTranslation", "task.params": dict(plan["task_config"]["task.params"], wait_k=want)}
    cli.write_model_configs(dict(plan, model_dir=str(tmp_path / "m")))
    with open(tmp_path / "m" / cli.MODEL_CONFIGS) as f:
        configs = yaml.safe_load(f)
    assert configs["model.class"] == "WaitkTransformer" and configs["task.params"]["wait_k"] == want
    assert configs["model.params"]["encoder.attention_monotonic"] is True


@pytest.mark.parametrize("name", ["waitk_translation", "WaitkTranslation"])
def test_waitk_task_aliases(tmp_path, name):
    assert cli.resolve(_waitk_cfg(tmp_path, 2, **{"task.class": name}))["wait_k"] == 2


@pytest.mark.parametrize("base", ["transformer_s", "transformer_base", "transformer_toy", "transformer_512_3e_2d_4h"])
def test_waitk_presets_are_monotonic_transformer_presets(base):
    want = transformer_hparams(base)
    for name in ("waitk_transformer_" + base[len("transformer_"):], "waitktransformer_" + base[len("transformer_"):]):
        hp = waitk_transformer_hparams(name)
        assert hp["model.class"] == "WaitkTransformer"
        assert hp["model.params"] == dict(want["model.params"], **{"encoder.attention_monotonic": True})
        assert hp["optimizer.params"] == want["optimizer.params"] and hp["lr_schedule.params"] == want["lr_schedule.params"]
    assert waitk_transformer_hparams(base) is None and waitk_transformer_hparams("waitk_transformer_nope") is None
    assert "encoder.attention_monotonic" not in want["model.params"]


def test_plain_transformer_honours_attention_monotonic(tmp_path):
    plan = cli.resolve(_mt_cfg(tmp_path, **{"model.params": {"encoder.attention_monotonic": True}}))
    assert plan["model_params"]["encoder.attention_monotonic"] is True and plan.get("wait_k") is None
    from neurst_b200.models import _model_flags
    assert any(f[:3] == ("encoder.attention_monotonic", bool, False) for f in _model_flags(False))
    assert not any(f[0] == "encoder.attention_monotonic" for f in _model_flags(True))


def test_predict_wait_k_override_order(tmp_path):
    train = cli.resolve(_waitk_cfg(tmp_path, [5, 7]))
    model_dir = str(tmp_path / "m")
    cli.write_model_configs(dict(train, model_dir=model_dir))
    pred = _waitk_cfg(tmp_path, None, **{"entry.class": "predict", "model_dir": model_dir})
    assert cli.resolve(pred)["wait_k"] == [5, 7]                                   # model_configs.yml
    pred["task.params"]["wait_k"] = 4
    assert cli.resolve(pred)["wait_k"] == 4                                        # task.params
    path = tmp_path / "predict.yml"
    path.write_text(yaml.safe_dump(pred))
    paths, overrides = cli.parse_command_line(["--config_paths", str(path), "--wait_k", "2"])
    assert cli.resolve(cli.load_config(paths, overrides))["wait_k"] == 2           # --wait_k (lands in task.params)
    del pred["task.params"]["wait_k"]
    path.write_text(yaml.safe_dump(pred))
    cfg = cli.load_config(paths, overrides)
    assert cfg["entry.params"]["wait_k"] == 2 and cli.resolve(cfg)["wait_k"] == 2   # --wait_k beats model_configs.yml
    flat = dict(pred, **{"entry.params": {"wait_k": 6}, "task.params": dict(pred["task.params"], wait_k=4)})
    assert cli.resolve(flat)["wait_k"] == 6                                        # a flat --wait_k beats task.params


def test_waitk_refusals(tmp_path):
    with pytest.raises(SystemExit, match="wait_k"):
        cli.resolve(_waitk_cfg(tmp_path, None))
    for bad in (0, -2, [3, 0], "[]", "abc", True):
        with pytest.raises(SystemExit, match="wait_k"):
            cli.resolve(_waitk_cfg(tmp_path, bad))
    with pytest.raises(SystemExit, match="SpeechToText"):
        cli.resolve({"task.class": "SpeechToText", "task.params": {"wait_k": 3, "batch_size": 100}})
    with pytest.raises(SystemExit, match="WaitkTransformer only"):
        cli.resolve(_waitk_cfg(tmp_path, 3, **{"model.class": "Transformer"}))
    with pytest.raises(SystemExit, match="WaitkTranslation"):
        cli.resolve(_mt_cfg(tmp_path, **{"model.class": "WaitkTransformer"}))
    with pytest.raises(SystemExit, match="ensemble"):
        cli.resolve(_waitk_cfg(tmp_path, 3, **{"entry.class": "predict", "model_dir": ["a", "b"]}))
    # an ensemble member or a cascade MT model that is a wait-k model
    train = cli.resolve(_waitk_cfg(tmp_path, 3))
    wk = str(tmp_path / "wk")
    cli.write_model_configs(dict(train, model_dir=wk))
    plain = cli.resolve(_mt_cfg(tmp_path, **{"entry.class": "predict", "model_dir": [wk, wk]}))
    with pytest.raises(SystemExit, match="ensemble"):
        cli.member_model_params(plain, wk)
    with pytest.raises(SystemExit, match="wait-k"):
        cli.resolve({"entry.class": "cascade_st", "asr_model_dir": wk, "mt_model_dir": wk,
                     "dataset.params": {"data_path": "x"}})
    with pytest.raises(ValueError):
        parse_wait_k([])


# ------------------------------------------------------------------------------------------------ latency
@pytest.mark.parametrize("n", [1, 5, 12])
def test_latency_equals_k_when_lengths_match(n):
    for k in range(1, n + 1):
        r = MT.waitk_latency(k, n, n)
        assert r["AL"] == pytest.approx(k, abs=1e-12) and r["DAL"] == pytest.approx(k, abs=1e-12)


def test_latency_hand_computed_values():
    # |x| = |y| = 4, k = 2: g = 2, 3, 4, 4 -> AP = 13 / 16
    assert MT.waitk_latency(2, 4, 4)["AP"] == pytest.approx(13 / 16)
    # |x| = 6, |y| = 3, k = 2: g = 2, 3, 4 (never reaches |x|: tau = 3); step |x|/|y| = 2
    r = MT.waitk_latency(2, 6, 3)
    assert r["AL"] == pytest.approx(((2 - 0) + (3 - 2) + (4 - 4)) / 3)
    assert r["AP"] == pytest.approx(9 / 18)
    # g' = 2, max(3, 4) = 4, max(4, 6) = 6 -> (2 + 2 + 2) / 3
    assert r["DAL"] == pytest.approx(2.0)
    # |x| = 2, |y| = 4, k = 3: g = 2, 2, 2, 2 (tau = 1); step 1/2
    r = MT.waitk_latency(3, 2, 4)
    assert r["AL"] == pytest.approx(2.0) and r["AP"] == pytest.approx(8 / 8)
    # g' = 2, 2.5, 3, 3.5 -> sum(g' - (i-1)/2) / 4 = 2
    assert r["DAL"] == pytest.approx(2.0)
    assert MT.waitk_latency(3, 0, 4) is None and MT.waitk_latency(3, 4, 0) is None
    assert MT.corpus_waitk_latency(2, [(4, 4), (6, 3), (0, 2)]) == pytest.approx(
        {m: (MT.waitk_latency(2, 4, 4)[m] + MT.waitk_latency(2, 6, 3)[m]) / 2 for m in ("AL", "AP", "DAL")})


# ------------------------------------------------------------------------------------------------ kernels
def _ptxas(src):
    from neurst_b200.csrc import build as B
    if not os.path.exists(B.NVCC):
        pytest.skip("nvcc not available (%s)" % B.NVCC)
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, src), "-o", os.path.join(tmp, "x.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    from tests.test_kernel_resources_cpu import spill_table
    return spill_table(r.stdout + r.stderr)


@pytest.mark.parametrize("src, pattern, count", [
    ("decode.cu", r"attn_step_kernel|greedy_persistent_kernel", 15),
    ("decode_rows.cu", r"rows_cross_attn_kernel", 1),
    ("elem_kernels.cu", r"softmax_fwd_kernel", 12),
    ("attention.cu", r"attn_fwd_kernel|attn_bwd_kernel", 8),
])
def test_changed_kernels_do_not_spill(src, pattern, count):
    table = {k: v for k, v in _ptxas(src).items() if re.search(pattern, k)}
    assert len(table) == count, sorted(table)
    spilled = {k: v for k, v in table.items() if v[1] or v[2]}
    assert not spilled, spilled
