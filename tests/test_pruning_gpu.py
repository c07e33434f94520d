"""Weight pruning on the device (b200st_optimizer_step with a prune schedule, b200st_prune_select) against torch
restatements of the reference's pruning optimizer (neurst/sparsity/pruning_optimizer.py, keep_prune_property=True): the
exact segmented selection, the step semantics over a dozen updates, the fp16 skip, the 16-bit shadow, and `train` /
`predict` through the entry for the speech and the text model."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from neurst_b200 import cli
from neurst_b200 import lib as L
from neurst_b200 import pruning as PR
from oracle import restatement as R
from tests import parity_utils as U

pytestmark = pytest.mark.gpu

RECIPE = "(ln/gamma)|(ln/beta)|(modalit)"


def _bits(mask):
    return ((mask.cpu().to(torch.int32)[:, None] >> torch.arange(8)) & 1).flatten().bool()


def _arena(sizes, fill, seed):
    g = torch.Generator().manual_seed(seed)
    offs, o = [], 0
    for n in sizes:
        offs.append(o)
        o += (n + 7) // 8 * 8
    w = torch.zeros(o)
    for off, n, f in zip(offs, sizes, fill):
        w[off:off + n] = f(n, g)
    return w, offs


def _select(w, offs, sizes, ks, shadow=None):
    lib = L.load()
    n = len(offs)
    mask = torch.full((w.numel() // 8,), 0xAB, dtype=torch.uint8, device="cuda")
    thr = torch.zeros(n, device="cuda")
    scratch = torch.zeros(int(lib.b200st_prune_scratch_bytes(n)), dtype=torch.uint8, device="cuda")
    k = torch.tensor(ks, dtype=torch.int64, device="cuda")
    L.check(lib.b200st_prune_select(w.data_ptr(), None if shadow is None else shadow.data_ptr(), (C.c_int64 * n)(*offs),
                                    (C.c_int64 * n)(*sizes), k.data_ptr(), n, mask.data_ptr(), thr.data_ptr(), scratch.data_ptr(),
                                    L._stream()))
    torch.cuda.synchronize()
    return mask, thr, scratch


def test_segmented_selection_is_exact_top_k():
    randn = lambda n, g: torch.randn(n, generator=g)                                               # noqa: E731
    ties = lambda n, g: torch.randint(-2, 3, (n,), generator=g).float() * 0.25                     # noqa: E731
    zeros = lambda n, g: torch.zeros(n)                                                            # noqa: E731
    tiny = lambda n, g: torch.randn(n, generator=g) * 1e-30                                        # noqa: E731 (denormals)
    cases = [(8, randn, 3), (9 * 256, randn, 1000), (2 * 1024 * 1024 + 5, randn, 700001), (4096, ties, 1500), (5000, zeros, 17),
             (777, randn, 1), (1000, randn, 1000), (1, randn, 1), (13, ties, 13), (300, tiny, 150), (16384, randn, 8192),
             (16385, ties, 16385)]
    g = torch.Generator().manual_seed(5)
    for _ in range(60):                          # many small tensors of random sizes
        n = int(torch.randint(1, 40000, (1,), generator=g))
        cases.append((n, randn, int(torch.randint(1, n + 1, (1,), generator=g))))
    sizes = [c[0] for c in cases]
    ks = [c[2] for c in cases]
    w0, offs = _arena(sizes, [c[1] for c in cases], seed=1)
    w = w0.cuda()
    shadow = w.to(torch.bfloat16)
    mask, thr, _ = _select(w, offs, sizes, ks, shadow)
    bits = _bits(mask)
    wc = w.cpu()
    for i, (off, n, k) in enumerate(zip(offs, sizes, ks)):
        t = w0[off:off + n].abs()
        ref = torch.topk(t, k).values[-1]
        assert float(thr[i]) == float(ref), (i, n, k)
        keep = t >= ref
        assert torch.equal(bits[off:off + n], keep), (i, n, k)
        assert bits[off + n:(off + n + 7) // 8 * 8].all()               # padding bits stay 1
        assert torch.equal(wc[off:off + n], torch.where(keep, w0[off:off + n], torch.zeros(())))
    assert torch.equal(shadow.cpu(), (w0 * bits.float()).to(torch.bfloat16))
    # a second run on the same data is bitwise identical
    w2 = w0.cuda()
    mask2, thr2, _ = _select(w2, offs, sizes, ks)
    assert torch.equal(mask2, mask) and torch.equal(thr2, thr) and torch.equal(w2, w)


def _toy(precision="fp32", scale=1.0):
    cfg = dict(R.CONFIGS["speech_transformer_toy"])
    if precision != "fp32":
        cfg = dict(model="speech", d=64, heads=4, enc_layers=1, dec_layers=1, ffn=64, channels=64, feat=80, in_channels=1, vocab=96)
    rt = U.speech_runtime(cfg, precision)
    P = R.init_params(cfg, seed=1, random_bias=True)
    rt.load_parameters({k: v * scale for k, v in P.items()})
    return rt


def _numel(rt, k):
    return int(np.prod(rt.table[k][1]))


def test_pruned_steps_follow_the_reference_rules():
    """A dozen updates with given gradients: mask from zeros at the start, Adam then w *= mask off-turn, on a turn the new
    mask from the Adam-updated weights without the old one (pruned weights can come back), exact masks, Adam moments kept."""
    rt = _toy(scale=0.05)
    names = [k for k in rt.table if not k.endswith(("gamma", "beta"))]
    k0 = names[2]
    off0 = rt.table[k0][0]
    rt.params[off0:off0 + 5] = 0.0                       # weights already zero at the start stay masked until a turn
    sched = PR.PolynomialDecay(initial_sparsity=0.2, target_sparsity=0.6, begin_pruning_step=2, end_pruning_step=10,
                               pruning_frequency=3, polynomial_power=2)
    rt.prune_setup(sched, names)
    valid = torch.zeros(rt.numel, dtype=torch.bool)
    for k in rt.table:
        valid[rt.table[k][0]:rt.table[k][0] + _numel(rt, k)] = True
    p, m, v = rt.params.cpu().clone(), torch.zeros(rt.numel), torch.zeros(rt.numel)
    keep = torch.ones(rt.numel, dtype=torch.bool)
    for k in names:
        off = rt.table[k][0]
        keep[off:off + _numel(rt, k)] = p[off:off + _numel(rt, k)] != 0
    assert torch.equal(_bits(rt.prune_mask), keep)
    g = torch.Generator().manual_seed(3)
    regrown = 0
    lr = 1e-2
    for step in range(1, 13):
        grad = torch.randn(rt.numel, generator=g) * valid
        rt.ensure_grads().copy_(grad.cuda())
        rt.adam_step(lr, step, prune=sched)
        torch.cuda.synchronize()
        p, m, v = R.adam_update(p, grad, m, v, lr, step)
        state = rt.prune_state.cpu().tolist()
        turn = sched.should_prune_in_step(step)
        assert state[0] == step and state[1] == int(turn)
        if turn:
            sp = np.float32(sched.sparsity_in_step(step))
            assert np.frombuffer(np.int32(state[3]).tobytes(), np.float32)[0] == sp
            before = keep.clone()
            for i, k in enumerate(names):
                off, n = rt.table[k][0], _numel(rt, k)
                t = p[off:off + n].abs()
                thr = torch.topk(t, PR.k_of(n, sp)).values[-1]
                keep[off:off + n] = t >= thr
                assert abs(float(rt.prune_thresholds[i]) - float(thr)) <= 1e-6 * max(float(thr), 1e-30) + 1e-9, k
            regrown += int((keep & ~before).sum())
        p = p * keep
        assert torch.equal(_bits(rt.prune_mask), keep), step
        assert float((rt.params.cpu() - p).abs().max()) < 1e-5, step
    assert regrown > 0
    assert torch.equal(rt.params.cpu() == 0, ~keep | (p == 0))
    # the moments of pruned weights kept moving
    assert float(rt.adam_m.cpu()[~keep].abs().min()) > 0 and float((rt.adam_m.cpu() - m).abs().max()) < 1e-5


def test_fp16_skipped_update_shifts_the_next_turn_and_the_shadow_follows():
    rt = _toy("fp16")
    names = [k for k in rt.table if k.endswith(("kernel", ".w1", ".w2"))]
    sched = PR.ConstantSparsity(target_sparsity=0.5, begin_pruning_step=0, pruning_frequency=2)
    rt.prune_setup(sched, names)
    g = torch.randn(rt.numel, device="cuda") * 2.0 ** 12
    mask0 = rt.prune_mask.clone()
    rt.ensure_grads().copy_(g)
    rt.adam_step(1e-3, 1, prune=sched)                     # applied: step 1, no turn
    torch.cuda.synchronize()
    assert rt.prune_state.cpu().tolist()[:3] == [1, 0, 0] and torch.equal(rt.prune_mask, mask0)
    p1, sh1 = rt.params.clone(), rt.shadow.clone()
    rt.grads.copy_(g)
    rt.grads[7] = float("nan")
    rt.adam_step(1e-3, 2, prune=sched)                     # skipped: nothing applied, the step does not advance
    torch.cuda.synchronize()
    assert float(rt.loss_scale_state[2]) == 1.0
    assert rt.prune_state.cpu().tolist()[:3] == [1, 0, 0]
    assert torch.equal(rt.params, p1) and torch.equal(rt.shadow, sh1) and torch.equal(rt.prune_mask, mask0)
    rt.grads.copy_(g)
    rt.adam_step(1e-3, 3, prune=sched)                     # applied: step 2, the turn (one update later than without the skip)
    torch.cuda.synchronize()
    assert rt.prune_state.cpu().tolist()[:3] == [2, 1, 1]
    for k in names:
        n = _numel(rt, k)
        assert int((rt.view(k) != 0).sum()) == PR.k_of(n, 0.5), k
    # the 16-bit shadow is the cast of the masked master weights
    assert torch.equal(rt.shadow, rt.params.to(torch.float16))


def test_zero_sparsity_schedule_leaves_parameters_bitwise_identical():
    from neurst_b200.models import SpeechTransformer
    from neurst_b200.trainer import DataParallelTrainer, synthetic_batch
    from neurst_b200.models import speech_transformer_hparams
    from neurst_b200.runtime import Runtime, make_config
    args = dict(speech_transformer_hparams("speech_transformer_s")["model.params"])
    args.update({"encoder.num_layers": 2, "decoder.num_layers": 2, "encoder.hidden_size": 128, "decoder.hidden_size": 128,
                 "modality.dim": 128, "encoder.filter_size": 256, "decoder.filter_size": 256, "modality.source.channels": 64})
    for side in ("encoder", "decoder"):
        for k in ("attention_dropout_rate", "ffn_dropout_rate", "layer_postprocess_dropout_rate"):
            args["%s.%s" % (side, k)] = 0.0
    tm = {"vocab_size": 96, "eos_id": 95, "bos_id": 94, "unk_id": 93, "pad_id": 95}
    batches = [synthetic_batch(4, 120, 9, 96, seed=i, device="cuda") for i in range(4)]

    def model():
        cfg = make_config(L.MODEL_SPEECH, 128, args["encoder.num_attention_heads"], 256, 2, 2, 96, feat=80, in_channels=1,
                          channels=64, conv_layer_norm=args.get("modality.source.layer_norm", False), precision="bf16",
                          label_smoothing=0.1, deterministic=True)
        m = SpeechTransformer(args, {"audio_feature_dim": 80, "audio_feature_channels": 1}, tm, Runtime(cfg, "cuda"))
        m.init_parameters(7)
        return m

    # the gradients of real backward passes, replayed into every arm: the split-K weight gradients sum in arrival order, so
    # two backward passes are not bit-identical even in the deterministic mode, and the optimizer step is what is compared
    ref = model()
    grads = []
    for i, b in enumerate(batches):
        ref.runtime.ensure_grads().zero_()
        ref.forward_backward(dict(b, seed=i))
        grads.append(ref.runtime.grads.clone())
    outs = []
    # no schedule; a zero-sparsity one (no pruning, as PruningSchedule.new); a schedule whose first turn never comes, over
    # tensors with no zero at the start: the masked Adam pass with an all-ones mask
    later = PR.ConstantSparsity(target_sparsity=0.5, begin_pruning_step=10 ** 6)
    for sched in (None, PR.ConstantSparsity(target_sparsity=0.0, begin_pruning_step=0, pruning_frequency=2), later):
        m = model()
        kernels = [k for k in m.runtime.table if k.endswith(("kernel", ".w1", ".w2"))]
        tr = DataParallelTrainer(m, pruning_schedule=sched, pruning_variables=kernels)
        assert (tr.pruning_schedule is None) == (sched is not later)
        it = iter(grads)
        m.forward_backward = lambda inputs, is_training=True, loss_scale=1.0, m=m, it=it: (
            m.runtime.grads.add_(next(it)), {"loss": torch.zeros(1, device="cuda")})[1]
        for i, b in enumerate(batches):
            tr.train_step(b, seed=i)
        torch.cuda.synchronize()
        outs.append((m.runtime.params.clone(), m.runtime.shadow.clone()))
        if sched is later:
            assert int(m.runtime.prune_state[0]) == 4 and bool((m.runtime.prune_mask == 255).all())
    assert not torch.equal(outs[0][0], ref.runtime.params)          # the steps did update the weights
    for params, shadow in outs[1:]:
        assert torch.equal(outs[0][0], params) and torch.equal(outs[0][1], shadow)


def _check_pruned_checkpoint(path, res, scope):
    z = np.load(path)
    names = [k for k in z.files if "/.OPTIMIZER_SLOT/" not in k]
    assert all(k.startswith(scope + "/") for k in names)
    pruned = PR.select_variables(names, None, RECIPE)
    assert len(pruned) == res["pruning"]["tensors"] and 0 < len(pruned) < len(names)
    sp = res["pruning"]["turn_sparsity"]
    for k in pruned:
        assert int(np.count_nonzero(z[k])) == PR.k_of(z[k].size, sp), k
    for k in set(names) - set(pruned):
        assert np.count_nonzero(z[k]) == z[k].size, k              # no zeros in the LayerNorms and modalities
    return z


def test_speech_train_prunes_resumes_and_predicts_through_the_entry(tmp_path):
    from tests.test_cli import _write_dataset, _write_yaml
    _write_dataset(tmp_path, vocab=93)
    y = _write_yaml(tmp_path, data=str(tmp_path / "train.tfrecords"), n_tokens=93)
    model_dir = str(tmp_path / "model")
    tiny = ["--model.params.encoder.num_layers", "2", "--model.params.decoder.num_layers", "2",
            "--model.params.encoder.hidden_size", "128", "--model.params.decoder.hidden_size", "128", "--model.params.modality.dim", "128",
            "--model.params.encoder.num_attention_heads", "2", "--model.params.decoder.num_attention_heads", "2",
            "--model.params.encoder.filter_size", "256", "--model.params.decoder.filter_size", "256",
            "--model.params.modality.source.channels", "64"]
    common = ["--config_paths", y, "--model_dir", model_dir, "--task.params.batch_size", "3000", "--task.params.max_src_len", "400",
              "--task.params.max_trg_len", "24", "--task.params.min_src_bucket_boundary", "128", "--dtype", "bfloat16",
              "--task.params.experimental_frame_transcript_ratio", "20", "--save_checkpoint_steps", "3", "--summary_steps", "2"] + tiny
    prune = ["--pruning_schedule", "polynomial_decay", "--target_sparsity", "0.5", "--end_pruning_step", "4",
             "--pruning_frequency", "2", "--nopruning_variable_pattern", RECIPE]
    res = cli.main(common + prune + ["--train_steps", "6"])
    assert res["global_step"] == 6 and res["pruning"]["updates"] == 6 and res["pruning"]["turns"] == 2
    assert res["pruning"]["turn_sparsity"] == 0.5
    z = _check_pruned_checkpoint(os.path.join(model_dir, "ckpt-6.npz"), res, "SpeechTransformer")
    # resume: the mask is re-derived from the zeros; one more update is no turn of the restarted schedule
    res = cli.main(common + prune + ["--train_steps", "7"])
    assert res["global_step"] == 7 and res["pruning"]["updates"] == 1 and res["pruning"]["turns"] == 0
    z7 = np.load(os.path.join(model_dir, "ckpt-7.npz"))
    for k in PR.select_variables([k for k in z.files if "/.OPTIMIZER_SLOT/" not in k], None, RECIPE):
        assert np.array_equal(z7[k] == 0, z[k] == 0), k
    one = tmp_path / "one"
    one.mkdir()
    os.link(str(tmp_path / "train.tfrecords-00000-of-00003"), str(one / "train.tfrecords-00000-of-00001"))
    res = cli.main(common + ["--entry.class", "predict", "--dataset.params.data_path", str(one / "train.tfrecords"),
                             "--maximum_decode_length", "12"])
    assert res["checkpoint_step"] == 7 and res["n_hypotheses"] == 70


def test_text_train_prunes_and_initial_global_step(tmp_path):
    from tests.test_mt_gpu import _corpus, _mt_plan
    root = tmp_path
    (root / "vocab.src").write_text("".join("s%d\t1\n" % i for i in range(85)))
    (root / "vocab.trg").write_text("".join("t%d\t1\n" % i for i in range(40)) + "x\n" + "".join("p%d\n" % i for i in range(4)))
    mt = (root, _corpus(root, 300, 1, "train"), _corpus(root, 20, 2, "dev"))
    model_dir = root / "m"
    prune = {"validator.class": None, "dtype": "bfloat16", "pruning_schedule": "polynomial_decay", "target_sparsity": 0.5,
             "end_pruning_step": 4, "pruning_frequency": 2, "nopruning_variable_pattern": RECIPE}
    res = cli.train(_mt_plan(mt, model_dir, 6, **prune))
    assert res["global_step"] == 6 and res["pruning"]["turns"] == 2 and res["pruning"]["turn_sparsity"] == 0.5
    _check_pruned_checkpoint(os.path.join(model_dir, "ckpt-6.npz"), res, "Transformer")
    out = cli.predict(_mt_plan(mt, model_dir, 6, entry="predict", **{"dtype": "bfloat16"}))
    assert out["checkpoint_step"] == 6 and len(out["hypotheses"]) == 20
    # initial_global_step: train_steps updates from that step, checkpoints numbered from it, noam position from it; Adam's
    # t counts this run's updates from 1 (the reference's optimizer iterations start at 0 whatever the initial step)
    from neurst_b200 import trainer as T
    from neurst_b200.runtime import Runtime
    lrs, calls, first = [], [], {}
    orig_lr, orig_adam = T.noam_learning_rate, Runtime.adam_step

    def adam_step(rt, lr, step_t, beta1=0.9, beta2=0.98, eps=1e-9, grad_scale=1.0, **kw):
        calls.append(step_t)
        if not first:
            first.update(p=rt.params.cpu().clone(), g=rt.grads.cpu().clone(), lr=lr, b=(beta1, beta2, eps), s=grad_scale,
                         fresh=rt.adam_m is None)
        orig_adam(rt, lr, step_t, beta1, beta2, eps, grad_scale=grad_scale, **kw)
        if "after" not in first:
            first["after"] = rt.params.cpu().clone()

    T.noam_learning_rate = lambda step, **kw: (lrs.append(step), orig_lr(step, **kw))[1]
    Runtime.adam_step = adam_step
    try:
        model_dir2 = root / "m2"
        res = cli.train(_mt_plan(mt, model_dir2, 5, initial_global_step=1000, **{"validator.class": None, "dtype": "bfloat16"}))
    finally:
        T.noam_learning_rate, Runtime.adam_step = orig_lr, orig_adam
    assert res["global_step"] == 1005 and lrs == [1000, 1001, 1002, 1003, 1004] and calls == [1, 2, 3, 4, 5]
    assert sorted(os.listdir(model_dir2)) == sorted(["checkpoint", "ckpt-1004.npz", "ckpt-1005.npz", "model_configs.yml"])
    # the first update of the bf16 run is Adam with t = 1 from zero moments (and not t = 1001)
    assert first["fresh"]
    b1, b2, eps = first["b"]
    zero = torch.zeros_like(first["p"])
    want, _, _ = R.adam_update(first["p"], first["g"] * first["s"], zero, zero, first["lr"], 1, b1, b2, eps)
    late, _, _ = R.adam_update(first["p"], first["g"] * first["s"], zero, zero, first["lr"], 1001, b1, b2, eps)
    step = (want - first["p"]).abs().max()
    assert float((first["after"] - want).abs().max()) < 1e-3 * float(step)
    assert float((first["after"] - late).abs().max()) > 0.1 * float(step)
