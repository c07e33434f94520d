"""Cost of the partial-tuning optimizer step (b200st_optimizer_step with a frozen bitmap) against the plain step on the
parameter arenas of speech_transformer_s and transformer_big, bf16 shadow, random weights and gradients, a tenth of the
weights of the recipe's pruned tensors (all but LayerNorms and modalities) zero and tuned, everything else frozen.

The two arms are timed with CUDA events over ITERS back-to-back steps, alternated, REPEATS times after a warm-up of each.
Each arm includes one device copy of the gradient arena (timed alone as grad_copy).  The partial step reads numel / 8 bytes
more than the plain step's 34 bytes per parameter.  Prints the GPU name, power limit and clocks read in the same run and writes
the numbers to a temporary directory.

    python tools/prune_tune_bench.py
"""
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ITERS, REPEATS = 20, 7
RECIPE = "(ln/gamma)|(ln/beta)|(modalit)"


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
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
    for k in PR.pruned_parameters(rt.table, None, RECIPE):        # a pruned model: 10 % zeros in the pruned tensors
        v = rt.view(k)
        v.mul_((torch.rand(v.shape, generator=g, device="cuda") >= 0.1).float())
    rt.refresh_shadow()
    grads = torch.randn(rt.numel, generator=g, device="cuda")
    tuned, frozen = rt.partial_setup(rt.derive_prune_mask(list(rt.table)))
    state = {"t": 0}

    def step(partial):
        def run():
            state["t"] += 1
            rt.ensure_grads().copy_(grads)
            rt.adam_step(1e-6, state["t"], zero_grad=True, frozen=rt.partial_frozen if partial else None)
        return run

    copy_ms = _arms({"grad_copy": lambda: rt.ensure_grads().copy_(grads)})["grad_copy"]
    res = _arms({"plain": step(False), "partial": step(True)})
    return {"arena": name, "parameters": rt.numel, "tuned": tuned, "frozen": frozen, "adam_bytes": 34 * rt.numel,
            "bitmap_bytes": rt.numel // 8, "grad_copy_ms": copy_ms, "ms": res}


def main():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("prune_tune_bench needs a CUDA device")
    from oracle import restatement as R
    info = gpu_info()
    res = {"gpu": info, "optimizer": [], "iters": ITERS, "repeats": REPEATS}
    big = dict(model="text", d=1024, heads=16, enc_layers=6, dec_layers=6, ffn=4096, vocab=32768, src_vocab=32768)
    for name, cfg in (("speech_transformer_s", R.CONFIGS["speech_transformer_s"]), ("transformer_big", big)):
        r = optimizer_arms(name, cfg)
        res["optimizer"].append(r)
        p, q = r["ms"]["plain"], r["ms"]["partial"]
        print("%s: %.1f M parameters (%.2f M tuned), bitmap %.1f MB: plain %.4f ms (%.4f..%.4f), partial %.4f ms (%.4f..%.4f), "
              "partial - plain %+.1f us (min), per repeat %s us; gradient copy %.4f ms included" % (
                  name, r["parameters"] / 1e6, r["tuned"] / 1e6, r["bitmap_bytes"] / 1e6, min(p), min(p), max(p), min(q), min(q),
                  max(q), (min(q) - min(p)) * 1e3, ["%+.1f" % ((b - a) * 1e3) for a, b in zip(p, q)], min(r["grad_copy_ms"])))
    print("GPU %s, power limit %s, SM clock %s (max %s), memory clock %s" % (
        info.get("name"), info.get("power.limit"), info.get("clocks.sm"), info.get("clocks.max.sm"), info.get("clocks.mem")))
    out = os.path.join(tempfile.mkdtemp(prefix="prune_tune_bench_"), "prune_tune_bench.json")
    with open(out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))
    print("wrote", out)


if __name__ == "__main__":
    main()
