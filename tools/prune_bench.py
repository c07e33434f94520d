"""Cost of weight pruning during training (b200st_optimizer_step with a prune schedule) on the parameter arenas of
speech_transformer_s and transformer_big, bf16 shadow, random weights and gradients.

Arms per arena, timed with CUDA events over ITERS back-to-back steps, alternated, REPEATS times after a warm-up of each:
  plain      b200st_optimizer_step (Keras Adam + shadow refresh + gradient zeroing)
  off_turn   the pruned step off a pruning turn: the mask in the Adam pass, the control kernel, the selection kernels
             launched and exiting at once (the recipe's pattern: LayerNorms and modalities are not pruned)
  turn       the pruned step on a pruning turn (every update a turn): Adam, three radix-digit passes and the mask update
and the cfg-2 training step (speech_transformer_s, [32,1000,80], L 88, bf16, one captured forward + backward and the optimizer
step) without pruning and with a schedule whose turn comes every 100 updates.  The bytes Adam moves per parameter (34) and
what the mask adds (1 bit) are computed from the arena sizes.  Prints the GPU name and power limit read in the same run and
writes the numbers to a temporary directory.

    python tools/prune_bench.py
"""
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ITERS, REPEATS = 20, 5
RECIPE = "(ln/gamma)|(ln/beta)|(modalit)"


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # noqa
        return {"error": str(e)}


def _time(fn, iters=ITERS):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def _arms(arms):
    """{name: [ms per call] * REPEATS}, the arms alternated inside each repeat."""
    for fn in arms.values():
        _time(fn, 3)
    out = {k: [] for k in arms}
    for _ in range(REPEATS):
        for k, fn in arms.items():
            out[k].append(_time(fn))
    return out


def optimizer_arms(name, cfg):
    import torch
    from neurst_b200 import lib as L
    from neurst_b200 import pruning as PR
    from neurst_b200.runtime import Runtime, make_config
    text = cfg["model"] == "text"
    c = make_config(L.MODEL_TEXT if text else L.MODEL_SPEECH, cfg["d"], cfg["heads"], cfg["ffn"], cfg["enc_layers"], cfg["dec_layers"],
                    cfg["vocab"], src_vocab=cfg.get("src_vocab", 0), channels=cfg.get("channels", 0), precision="bf16")
    rt = Runtime(c)
    g = torch.Generator(device="cuda").manual_seed(1)
    rt.params.copy_(torch.randn(rt.numel, generator=g, device="cuda") * 0.02)
    rt.refresh_shadow()
    grads = torch.randn(rt.numel, generator=g, device="cuda")
    names = PR.pruned_parameters(rt.table, None, RECIPE)
    never = PR.ConstantSparsity(target_sparsity=0.3, begin_pruning_step=10 ** 9)
    every = PR.ConstantSparsity(target_sparsity=0.3, begin_pruning_step=0, pruning_frequency=1)
    state = {"t": 0}

    def step(prune):
        def run():
            state["t"] += 1
            rt.ensure_grads().copy_(grads)
            if prune is not None and getattr(rt, "prune_schedule", None) is not prune:
                rt.prune_setup(prune, names)
            rt.adam_step(1e-6, state["t"], zero_grad=True, prune=prune)
        return run

    copy_ms = _arms({"grad_copy": lambda: rt.ensure_grads().copy_(grads)})["grad_copy"]
    res = _arms({"plain": step(None), "off_turn": step(never)})
    res.update(_arms({"turn": step(every)}))
    pruned = sum(rt._numel_of(k) for k in names)
    return {"arena": name, "parameters": rt.numel, "tensors": len(rt.table), "pruned_tensors": len(names), "pruned_parameters": pruned,
            "adam_bytes": 34 * rt.numel, "mask_bytes": rt.numel // 8, "grad_copy_ms": copy_ms,
            "ms": res, "note": "each arm includes one device copy of the gradient arena (grad_copy_ms)"}


def training_arms():
    import torch
    from neurst_b200 import pruning as PR
    from neurst_b200.trainer import build_speech_transformer_trainer, synthetic_batch
    out = {}
    batch = synthetic_batch(32, 1000, 88, 8192, device="cuda")
    trainers = {}
    for arm in ("dense", "pruned"):
        tr, _ = build_speech_transformer_trainer("speech_transformer_s", precision="bf16", use_cuda_graph=True)
        if arm == "pruned":
            tr.pruning_schedule = PR.ConstantSparsity(target_sparsity=0.3, begin_pruning_step=0, pruning_frequency=100)
            tr.pruning_variables = PR.pruned_parameters(tr.rt.table, None, RECIPE)
        trainers[arm] = tr
    arms = {k: (lambda tr=tr: tr.train_step(batch, seed=1)) for k, tr in trainers.items()}
    out["ms"] = _arms(arms)
    out["workload"] = "speech_transformer_s [32,1000,80] L 88 bf16, one captured fwd+bwd + optimizer step; pruned: turn every 100"
    torch.cuda.synchronize()
    return out


def main():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("prune_bench needs a CUDA device")
    from oracle import restatement as R
    info = gpu_info()
    res = {"gpu": info, "optimizer": [], "iters": ITERS, "repeats": REPEATS}
    big = dict(model="text", d=1024, heads=16, enc_layers=6, dec_layers=6, ffn=4096, vocab=32768, src_vocab=32768)
    for name, cfg in (("speech_transformer_s", R.CONFIGS["speech_transformer_s"]), ("transformer_big", big)):
        r = optimizer_arms(name, cfg)
        res["optimizer"].append(r)
        ms = {k: min(v) for k, v in r["ms"].items()}
        print("%s: %.1f M parameters (%.1f M pruned, %d tensors): plain %.3f ms, off-turn %.3f ms (+%.3f), turn %.3f ms (+%.3f); "
              "spread plain %.3f..%.3f off-turn %.3f..%.3f; gradient copy %.3f ms included" % (
                  name, r["parameters"] / 1e6, r["pruned_parameters"] / 1e6, r["pruned_tensors"], ms["plain"], ms["off_turn"],
                  ms["off_turn"] - ms["plain"], ms["turn"], ms["turn"] - ms["off_turn"], min(r["ms"]["plain"]), max(r["ms"]["plain"]),
                  min(r["ms"]["off_turn"]), max(r["ms"]["off_turn"]), min(r["grad_copy_ms"])))
    tr = training_arms()
    res["training"] = tr
    print("cfg-2 training step bf16: dense %.2f ms, pruned %.2f ms (min of %d x %d steps; dense %s, pruned %s)" % (
        min(tr["ms"]["dense"]), min(tr["ms"]["pruned"]), REPEATS, ITERS, ["%.2f" % x for x in tr["ms"]["dense"]],
        ["%.2f" % x for x in tr["ms"]["pruned"]]))
    print("GPU %s, power limit %s, SM clock %s (max %s)" % (info.get("name"), info.get("power.limit"), info.get("clocks.sm"),
                                                          info.get("clocks.max.sm")))
    out = os.path.join(tempfile.mkdtemp(prefix="prune_bench_"), "prune_bench.json")
    with open(out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))
    print("wrote", out)


if __name__ == "__main__":
    main()
