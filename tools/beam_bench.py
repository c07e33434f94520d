"""Beam search vs greedy decoding at the cfg-5 size: speech_transformer_s, one utterance [1,2000,80], never-EOS decoding
(EOS masked until the 200th position), random-init weights.

Arms, alternated, 3 repeats each after a warm-up of every arm:
  greedy graph       the per-token CUDA graph of the greedy search (fp32 master weights)
  greedy persistent  the single cooperative kernel of the greedy search (fp32 master weights)
  beam4 fp32 / fp16  beam search, beam 4, length_penalty -1 (4 rows per step), fp32 master or fp16 shadow weights

Times the search only (the encoder pass and the cache set-up are outside the CUDA events) and divides by the positions
decoded.  Prints the GPU name, power limit and SM clock next to the numbers and writes bench_out/beam_bench.json.

    python tools/beam_bench.py
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STEPS, T, V, REPEATS = 200, 2000, 8192, 3


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # noqa
        return {"error": str(e)}


def main():
    import torch
    from neurst_b200 import decode as D
    from neurst_b200 import lib
    from neurst_b200.models import SpeechTransformer, speech_transformer_hparams
    if not torch.cuda.is_available():
        raise SystemExit("beam_bench.py needs a CUDA device")
    lib.load()
    hp = dict(speech_transformer_hparams("speech_transformer_s")["model.params"])
    tm = {"vocab_size": V, "eos_id": V - 1, "bos_id": V - 2, "unk_id": V - 3}
    g = torch.Generator().manual_seed(5)
    inputs = dict(src=torch.randn(1, T, 80, 1, generator=g), src_length=torch.tensor([T]))
    runtimes = {}
    for dtype in ("fp32", "fp16"):
        model = SpeechTransformer.new(hp, {"audio_feature_dim": 80, "audio_feature_channels": 1}, tm, precision=dtype)
        model.init_parameters(1234)
        rt = model.runtime
        enc, bias = D.encode(rt, inputs)
        runtimes[dtype] = (model, rt, enc, bias)
    bos, eos, unk = tm["bos_id"], tm["eos_id"], tm["unk_id"]

    def greedy(persistent):
        _, rt, enc, bias = runtimes["fp32"]
        cache = D.create_decoding_cache(rt, enc, bias, STEPS)
        def run():
            _, _, ln = D.greedy_search(rt, None, bos, eos, unk, maximum_decode_length=STEPS, extra_decode_length=STEPS,
                                       minimum_decode_length=STEPS, cache=cache, persistent=persistent)
            return ln
        return run, lambda ln: int(ln.max())

    def beam(dtype):
        _, rt, enc, bias = runtimes[dtype]
        # the reference requires minimum < maximum decode length: EOS is masked for the first 199 positions, the search
        # runs until every beam has emitted it (200 positions) or 201 positions
        cache = D.create_decoding_cache(rt, enc, bias, STEPS + 1, use_shadow=dtype == "fp16", beam=4)
        def run():
            _, _, _, ln = D.beam_search(rt, None, bos, eos, unk, beam_size=4, top_k=4, length_penalty=-1.0,
                                        maximum_decode_length=STEPS + 1, extra_decode_length=STEPS,
                                        minimum_decode_length=STEPS, cache=cache)
            return ln
        return run, lambda ln: int(ln.max())

    arms = {"greedy_graph_fp32": greedy(False), "greedy_persistent_fp32": greedy(True), "beam4_fp32": beam("fp32"),
            "beam4_fp16_shadow": beam("fp16")}
    for run, _ in arms.values():       # warm-up: module loading, graph capture paths, shared-memory attributes
        run()
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    positions = {}
    for _ in range(REPEATS):
        for name, (run, count) in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ln = run()
            e1.record()
            torch.cuda.synchronize()
            positions[name] = count(ln)
            res[name].append(e0.elapsed_time(e1) * 1e3 / positions[name])
    info = gpu_info()
    out = {"gpu": info, "workload": "speech_transformer_s, one utterance [1,2000,80], never-EOS decoding, search only",
           "us_per_token": {k: {"median": sorted(v)[len(v) // 2], "min": min(v), "max": max(v), "runs": v} for k, v in res.items()},
           "positions": positions}
    print("GPU %s, power limit %s, SM clock %s (max %s)" % (info.get("name"), info.get("power.limit"), info.get("clocks.sm"),
                                                            info.get("clocks.max.sm")))
    for k, v in out["us_per_token"].items():
        print("%-24s %8.1f us/token (min %.1f, max %.1f, %d positions)" % (k, v["median"], v["min"], v["max"], positions[k]))
    os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
    with open(os.path.join(ROOT, "bench_out", "beam_bench.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
