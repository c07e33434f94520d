"""Prune-Tune on the device: the partial-tuning optimizer step against the plain step on a clone of the same arena, the
refusals of the step's two masks, the trainer with the captured step and update_cycle 2, its launches, and the whole recipe
through the entries (prune and write mask.pkl, tune the pruned positions, resume, derive the masks without mask_pkl,
mask_predict) for the text and speech models."""
import ctypes as C
import os
import shutil

import numpy as np
import pytest
import torch
import yaml

from neurst_b200 import cli
from neurst_b200 import lib as L
from neurst_b200 import pruning as PR
from oracle import restatement as R
from tests import parity_utils as U

pytestmark = pytest.mark.gpu

RECIPE = "(ln/gamma)|(ln/beta)|(modalit)"
SMALL = dict(model="speech", d=64, heads=4, enc_layers=1, dec_layers=1, ffn=64, channels=64, feat=80, in_channels=1, vocab=96)


def _bits(bitmap):
    return ((bitmap.to(torch.int32)[:, None] >> torch.arange(8, device=bitmap.device)) & 1).flatten().bool()


def _pair(precision):
    P = R.init_params(SMALL, seed=1, random_bias=True)
    rts = []
    for _ in range(2):
        rt = U.speech_runtime(SMALL, precision)
        rt.load_parameters(P)
        rt.refresh_shadow()
        rts.append(rt)
    return rts


def _valid(rt):
    v = torch.zeros(rt.numel, dtype=torch.bool, device="cuda")
    for k, (off, shape) in rt.table.items():
        v[off:off + int(np.prod(shape))] = True
    return v


@pytest.mark.parametrize("precision,kw", [("fp32", {}), ("bf16", {}), ("fp16", {}), ("bf16", {"clip_norm": 0.05}),
                                          ("fp32", {"clip_value": 1e-3}), ("fp16", {"clip_norm": 0.05, "clip_value": 2e-3})],
                         ids=["fp32", "bf16", "fp16", "bf16-clip_norm", "fp32-clip_value", "fp16-clip_both"])
def test_partial_step_against_the_plain_step(precision, kw):
    a, b = _pair(precision)
    g = torch.Generator().manual_seed(4)
    masks = {k: (torch.rand(shape, generator=g) < 0.6).to(torch.uint8) for k, (_, shape) in a.table.items()}
    tuned, frozen_n = a.partial_setup(a.derive_prune_mask(list(a.table), masks))
    assert frozen_n == sum(int(m.sum()) for m in masks.values()) and tuned + frozen_n == sum(m.numel() for m in masks.values())
    frozen = _bits(a.partial_frozen)
    assert frozen[~_valid(a)].all()                                     # padding bits are 1
    p_start = a.params.clone()
    sh_start = a.shadow.clone() if a.shadow is not None else None
    scale = 2.0 ** 12 if precision == "fp16" else 1.0
    valid = _valid(a)
    for step in range(1, 6):
        # multiples of 1/4: every per-tensor sum of squares is exact, so the statistics pass (float atomics in arrival order)
        # gives both arms the same clip_norm scales and loss-scale state bit for bit
        grad = torch.randint(-2, 3, (a.numel,), generator=g).float().cuda() * 0.25 * valid * scale
        if precision == "fp16" and step == 2:
            grad[11] = float("inf")                                     # skipped by the dynamic loss scale on both arms
        b_before = b.params.clone()
        for rt in (a, b):
            rt.ensure_grads().copy_(grad)
        a.adam_step(1e-2, step, frozen=a.partial_frozen, **kw)
        b.adam_step(1e-2, step, **kw)
        torch.cuda.synchronize()
        assert torch.equal(a.adam_m, b.adam_m) and torch.equal(a.adam_v, b.adam_v), step
        assert torch.equal(a.grads, b.grads)
        if precision == "fp16":
            assert torch.equal(a.loss_scale_state, b.loss_scale_state), step
            assert float(a.loss_scale_state[2]) == (1.0 if step == 2 else 0.0)
        if "clip_norm" in kw or precision == "fp16":
            assert torch.equal(a.tensor_sumsq, b.tensor_sumsq)
        assert torch.equal(a.params[~frozen], b.params[~frozen]), step
        assert torch.equal(a.params[frozen], p_start[frozen]), step
        if a.shadow is not None:
            assert torch.equal(a.shadow[~frozen], b.shadow[~frozen]) and torch.equal(a.shadow[frozen], sh_start[frozen]), step
        skipped = precision == "fp16" and step == 2
        assert bool((b.params[frozen & valid] != b_before[frozen & valid]).any()) != skipped     # the plain step moved them
    assert bool((a.params[~frozen] != p_start[~frozen]).any())


def test_partial_step_launches_what_the_plain_step_launches():
    for precision, kw in (("bf16", {}), ("fp16", {}), ("fp32", {"clip_norm": 1.0})):
        a, _ = _pair(precision)
        a.partial_setup(a.derive_prune_mask(list(a.table)))
        a.ensure_grads().normal_()
        counts = []
        for frozen in (None, a.partial_frozen, None, a.partial_frozen):
            before = L.launch_count()
            a.adam_step(1e-3, 1, frozen=frozen, zero_grad=False, **kw)
            torch.cuda.synchronize()
            counts.append(L.launch_count() - before)
        assert counts[0] == counts[1] == counts[2] == counts[3] > 0, (precision, counts)
        keep = a.partial_frozen.clone()
        keep[::3] = 0x5A
        before = L.launch_count()
        a.apply_mask(keep)
        torch.cuda.synchronize()
        assert L.launch_count() - before == 1
        zero = ~_bits(keep)
        assert not bool(a.params[zero].any())
        if a.shadow is not None:
            assert not bool(a.shadow[zero].float().any())


def test_optimizer_step_refuses_two_masks_and_a_mask_without_a_handle():
    """b200st_optimizer_step with a pruning schedule and a frozen-element bitmap together, or with either and no handle, is
    refused with the reason before any launch and writes no byte of the arenas, the masks or the pruning state; the same
    arguments with the pruning schedule alone and the handle are accepted."""
    rt, _ = _pair("bf16")
    sched = PR.ConstantSparsity(target_sparsity=0.3, begin_pruning_step=0, pruning_frequency=1)
    rt.prune_setup(sched, PR.pruned_parameters(rt.table, None, RECIPE))
    rt.partial_setup(rt.derive_prune_mask(list(rt.table)))
    rt.ensure_grads().normal_()
    rt.adam_m, rt.adam_v = torch.randn_like(rt.params) * 0.1, torch.rand_like(rt.params)
    a = L.OptimArgs()
    a.params, a.grads, a.m, a.v = rt.params.data_ptr(), rt.grads.data_ptr(), rt.adam_m.data_ptr(), rt.adam_v.data_ptr()
    a.shadow, a.shadow_dtype, a.numel = rt.shadow.data_ptr(), rt.prec, rt.numel
    a.lr, a.beta1, a.beta2, a.eps, a.step_t, a.grad_scale, a.zero_grad = 1e-3, 0.9, 0.98, 1e-9, 1, 1.0, 1
    prune = C.pointer(rt._prune_args(sched))
    written = (rt.params, rt.grads, rt.adam_m, rt.adam_v, rt.shadow, rt.prune_mask, rt.prune_state, rt.prune_thresholds,
               rt.prune_scratch, rt.partial_frozen)
    before = [x.clone() for x in written]
    torch.cuda.synchronize()
    launches = L.launch_count()
    for handle, p, frozen, reason in ((rt.handle, prune, rt.partial_frozen, "not both"), (None, prune, None, "handle"),
                                      (None, None, rt.partial_frozen, "handle")):
        a.prune, a.frozen = p, None if frozen is None else frozen.data_ptr()
        rc = rt.lib.b200st_optimizer_step(handle, C.byref(a), L._stream())
        assert rc != 0 and reason in rt.lib.b200st_last_error().decode(), (reason, rt.lib.b200st_last_error())
    torch.cuda.synchronize()
    assert L.launch_count() == launches
    for x, y in zip(written, before):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))
    a.prune, a.frozen = prune, None
    L.check(rt.lib.b200st_optimizer_step(rt.handle, C.byref(a), L._stream()))
    torch.cuda.synchronize()
    assert L.launch_count() > launches and int(rt.prune_state[0]) == 1 and not torch.equal(rt.params, before[0])


def test_trainer_with_the_captured_step_and_update_cycle_keeps_frozen_weights():
    from neurst_b200.models import SpeechTransformer, speech_transformer_hparams
    from neurst_b200.runtime import Runtime, make_config
    from neurst_b200.trainer import DataParallelTrainer, synthetic_batch
    args = dict(speech_transformer_hparams("speech_transformer_s")["model.params"])
    args.update({"encoder.num_layers": 2, "decoder.num_layers": 2, "encoder.hidden_size": 128, "decoder.hidden_size": 128,
                 "modality.dim": 128, "encoder.filter_size": 256, "decoder.filter_size": 256, "modality.source.channels": 64})
    tm = {"vocab_size": 96, "eos_id": 95, "bos_id": 94, "unk_id": 93, "pad_id": 95}
    cfg = make_config(L.MODEL_SPEECH, 128, args["encoder.num_attention_heads"], 256, 2, 2, 96, feat=80, in_channels=1, channels=64,
                      conv_layer_norm=args.get("modality.source.layer_norm", False), precision="bf16", label_smoothing=0.1)
    m = SpeechTransformer(args, {"audio_feature_dim": 80, "audio_feature_channels": 1}, tm, Runtime(cfg, "cuda"))
    m.init_parameters(7)
    rt = m.runtime
    g = torch.Generator(device="cuda").manual_seed(2)
    for k in PR.pruned_parameters(rt.table, None, RECIPE):             # a pruned model: 30 % zeros in the pruned tensors
        v = rt.view(k)
        v.mul_((torch.rand(v.shape, generator=g, device="cuda") >= 0.3).float())
    rt._shadow_stale = True
    tr = DataParallelTrainer(m, update_cycle=2, use_cuda_graph=True, partial_tuning_mask="weights",
                             lr_schedule_params=dict(dmodel=128, warmup_steps=10, initial_factor=1.0))
    tr.broadcast_parameters()
    tuned, frozen_n = tr.setup_partial_tuning()
    p0 = rt.params.clone()
    frozen = _bits(rt.partial_frozen)
    assert frozen_n == int((p0[_valid(rt)] != 0).sum()) and tuned == int((p0[_valid(rt)] == 0).sum()) > 0
    batch = synthetic_batch(4, 120, 9, 96, seed=3, device="cuda")
    for i in range(8):
        tr.train_step(batch, seed=i)
    torch.cuda.synchronize()
    assert tr.global_step == 4 and len(tr._graphs) >= 1
    assert torch.equal(rt.params[frozen], p0[frozen])
    assert torch.equal(rt.shadow[frozen], p0.to(torch.bfloat16)[frozen])
    moved = (rt.params != p0) & ~frozen
    assert int(moved.sum()) > 0.5 * tuned


# ---- the whole recipe through the entries ----------------------------------------------------------------------------------
def _f32_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def _weights(path):
    z = np.load(path)
    return {k: z[k] for k in z.files if "/.OPTIMIZER_SLOT/" not in k}


def _masks(path):
    z = np.load(path, allow_pickle=False)
    return {k: z[k] for k in z.files}


def _ckpts(model_dir):
    return sorted(os.path.join(model_dir, f) for f in os.listdir(model_dir) if f.startswith("ckpt-") and f.endswith(".npz"))


def _text_recipe(root):
    from tests.test_mt_gpu import TINY, _corpus
    (root / "vocab.src").write_text("".join("s%d\t1\n" % i for i in range(85)))
    (root / "vocab.trg").write_text("".join("t%d\t1\n" % i for i in range(40)) + "x\n" + "".join("p%d\n" % i for i in range(4)))
    ts, tt = _corpus(root, 300, 1, "train")
    ds, dt = _corpus(root, 24, 2, "dev")
    cfg = {"entry.class": "trainer", "task.class": "seq_to_seq", "dtype": "bfloat16", "hparams_set": "transformer_s",
           "model.params": dict(TINY), "entry.params": {"summary_steps": 100},
           "task.params": {"batch_by_tokens": True, "batch_size": 2000, "max_src_len": 20, "max_trg_len": 30,
                           "src_data_pipeline.params": {"vocab_path": str(root / "vocab.src")},
                           "trg_data_pipeline.params": {"vocab_path": str(root / "vocab.trg")}},
           "dataset.class": "ParallelTextDataset", "dataset.params": {"src_file": ts, "trg_file": tt, "data_is_processed": True}}
    val = {"validator.class": "CriterionValidator",
           "validator.params": {"eval_dataset": "ParallelTextDataset",
                                "eval_dataset.params": {"src_file": ds, "trg_file": dt, "data_is_processed": True},
                                "eval_batch_size": 8, "eval_steps": 2, "eval_criterion": "label_smoothed_cross_entropy"}}
    for name, c in (("train.yml", cfg), ("validation.yml", val)):
        (root / name).write_text(yaml.safe_dump(c))
    (root / "batch.yml").write_text("batch_size: 8\n")          # the prediction recipes' top-level batch_size: 16-bit weights
    train = ["--config_paths", str(root / "train.yml")]
    predict = ["--config_paths", str(root / "train.yml"), "--dataset.params.src_file", ds, "--dataset.params.trg_file", dt]
    searches = [["--config_paths", str(root / "batch.yml"), "--search_method", "beam_search", "--search_method.params.beam_size", "2",
                 "--maximum_decode_length", "30"],
                ["--search_method", "top_sampling", "--search_method.params.top_k", "5", "--maximum_decode_length", "30",
                 "--dtype", "float32"]]
    return train, predict, str(root / "validation.yml"), searches


def _speech_recipe(root):
    from tests.test_cli import _write_dataset, _write_yaml
    _write_dataset(root, vocab=93)
    y = _write_yaml(root, data=str(root / "train.tfrecords"), n_tokens=93)
    one = root / "one"
    one.mkdir()
    os.link(str(root / "train.tfrecords-00000-of-00003"), str(one / "train.tfrecords-00000-of-00001"))
    tiny = ["--model.params.encoder.num_layers", "2", "--model.params.decoder.num_layers", "2",
            "--model.params.encoder.hidden_size", "128", "--model.params.decoder.hidden_size", "128", "--model.params.modality.dim", "128",
            "--model.params.encoder.num_attention_heads", "2", "--model.params.decoder.num_attention_heads", "2",
            "--model.params.encoder.filter_size", "256", "--model.params.decoder.filter_size", "256",
            "--model.params.modality.source.channels", "64"]
    common = ["--config_paths", y, "--task.params.batch_size", "3000", "--task.params.max_src_len", "400",
              "--task.params.max_trg_len", "24", "--task.params.min_src_bucket_boundary", "128", "--dtype", "bfloat16",
              "--task.params.experimental_frame_transcript_ratio", "20", "--summary_steps", "100"] + tiny
    val = {"validator.class": "CriterionValidator",
           "validator.params": {"eval_dataset": "AudioTFRecordDataset", "eval_batch_size": 8, "eval_steps": 2,
                                "eval_dataset.params": {"data_path": str(one / "train.tfrecords"), "feature_key": "audio",
                                                        "transcript_key": "translation"},
                                "eval_criterion": "label_smoothed_cross_entropy"}}
    (root / "validation.yml").write_text(yaml.safe_dump(val))
    (root / "batch.yml").write_text("batch_size: 16\n")
    predict = common + ["--dataset.params.data_path", str(one / "train.tfrecords")]
    searches = [["--maximum_decode_length", "12", "--dtype", "float32"],
                ["--config_paths", str(root / "batch.yml"), "--search_method", "beam_search", "--search_method.params.beam_size", "2",
                 "--maximum_decode_length", "12"]]
    return common, predict, str(root / "validation.yml"), searches


@pytest.mark.parametrize("model", ["text", "speech"])
def test_prune_tune_recipe_through_the_entries(tmp_path, model):
    train, predict, validation, searches = (_text_recipe if model == "text" else _speech_recipe)(tmp_path)
    pruned_dir, tuned_dir, resumed_dir, derived_dir = (str(tmp_path / d) for d in ("pruned", "tuned", "tuned", "derived"))
    # 1. prune: mask.pkl = weight != 0 of the final checkpoint, over every variable
    res = cli.main(train + ["--entry", "prune_tune_train", "--include", "examples/prune_tune/src/", "--model_dir", pruned_dir,
                            "--train_steps", "4", "--save_checkpoint_steps", "4", "--pruning_schedule", "ConstantSparsity",
                            "--target_sparsity", "0.3", "--begin_pruning_step", "0", "--pruning_frequency", "2",
                            "--nopruning_variable_pattern", RECIPE])
    assert res["global_step"] == 4 and res["pruning"]["turns"] == 2
    pre = _weights(os.path.join(pruned_dir, "ckpt-4.npz"))
    mask_file = os.path.join(pruned_dir, "mask.pkl")
    masks = _masks(mask_file)
    assert sorted(masks) == sorted(pre)
    for k, w in pre.items():
        assert masks[k].dtype == np.uint8 and np.array_equal(masks[k], (w != 0).astype(np.uint8)), k
    pruned = PR.select_variables(sorted(pre), None, RECIPE)
    assert all(masks[k].min() == 0 for k in pruned)
    frozen_n = sum(int(m.sum()) for m in masks.values())

    # 2. tune the pruned positions from that model, with a validator: every checkpoint keeps the mask-1 weights bit for bit
    tune = train + ["--config_paths", validation, "--entry", "prune_tune_train", "--include", "examples/prune_tune/src/",
                    "--pretrain_model", pruned_dir, "--model_dir", tuned_dir, "--partial_tuning", "--save_checkpoint_steps", "2"]
    res = cli.main(tune + ["--initial_global_step", "0", "--train_steps", "4", "--mask_pkl", mask_file])
    assert res["global_step"] == 4 and res["partial_tuning"] == {"tuned": sum(m.size for m in masks.values()) - frozen_n,
                                                                 "frozen": frozen_n}
    assert [v["step"] for v in res["validations"]] == [2, 4]

    def check(ckpts):
        assert ckpts
        for path in ckpts:
            w = _weights(path)
            for k in pre:
                keep = masks[k] == 1
                assert _f32_equal(w[k][keep], pre[k][keep]), (path, k)
            assert all(np.any(w[k][masks[k] == 0] != 0) for k in pruned), path

    check(_ckpts(tuned_dir))
    assert all(np.array_equal(v, masks[k]) for k, v in _masks(os.path.join(tuned_dir, "mask.pkl")).items())
    # 3. resume without mask_pkl: the model_dir's mask.pkl, not the tuned weights, says what stays frozen
    res = cli.main(tune + ["--train_steps", "6"])
    assert res["global_step"] == 6 and res["partial_tuning"]["frozen"] == frozen_n
    check([os.path.join(resumed_dir, "ckpt-6.npz")])
    # 4. without mask_pkl the masks are weight != 0 of the pretrained model: the same frozen set
    res = cli.main(tune[:-2] + ["--save_checkpoint_steps", "100", "--model_dir", derived_dir, "--train_steps", "2"])
    derived = _masks(os.path.join(derived_dir, "mask.pkl"))
    assert res["partial_tuning"]["frozen"] == frozen_n and all(np.array_equal(derived[k], masks[k]) for k in masks)
    check([os.path.join(derived_dir, "ckpt-2.npz")])

    # 5. mask_predict --mask_pkl == predict on a copy of the tuned checkpoint with the mask-0 weights zeroed in NumPy
    last = _ckpts(tuned_dir)[-1]
    zeroed_dir = tmp_path / "zeroed"
    zeroed_dir.mkdir()
    shutil.copy(os.path.join(tuned_dir, "model_configs.yml"), str(zeroed_dir))
    w = _weights(last)
    np.savez(str(zeroed_dir / os.path.basename(last)), **{k: np.where(masks[k] == 1, v, np.float32(0)) for k, v in w.items()})

    def hyps(entry, model_dir, search, extra=()):
        out = str(tmp_path / "hyp.txt")
        cli.main(predict + ["--entry", entry, "--model_dir", model_dir, "--output_file", out] + search + list(extra))
        with open(out) as f:
            return f.read()

    for search in searches:
        masked = hyps("mask_predict", tuned_dir, search, ["--mask_pkl", mask_file])
        assert masked.strip() and masked == hyps("predict", str(zeroed_dir), search), search
        assert hyps("mask_generation", tuned_dir, search) == hyps("predict", tuned_dir, search), search
