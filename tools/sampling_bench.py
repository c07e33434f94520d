"""Top-k / nucleus sampling at the prediction recipes' width: speech_transformer_s, fp16 shadow weights, 64 utterances
[64,1000,80] x sample_num 4 = 256 rows per step, 150 positions forced by masking EOS (minimum_decode_length 150), random-init
weights.

Arms, alternated, 3 repeats each after a warm-up of every arm:
  sample_topk0   top_k 0, top_p 1.0 (no filter)
  sample_topk10  top_k 10
  sample_topp09  top_p 0.9
  beam4          beam search, beam 4, length_penalty -1, on the same 64 x 4 rows

Times the search only (the encoder pass and the cache set-up are outside the CUDA events) and divides by the positions
decoded.  A second process (B200ST_NO_PDL=1, so kernel times do not include the wait for the previous kernel) runs each arm
once under torch.profiler and reports the per-token time of the selection kernel (sample_select_kernel / beam_select_kernel).
Prints the GPU name, power limit and SM clock next to the numbers and writes them to a temporary directory.

    python tools/sampling_bench.py
"""
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

UTT, SAMPLES, T, V, STEPS, REPEATS = 64, 4, 1000, 8192, 150, 3


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # noqa
        return {"error": str(e)}


def arms():
    import torch
    from neurst_b200 import decode as D
    from neurst_b200 import lib
    from neurst_b200.models import SpeechTransformer, speech_transformer_hparams
    if not torch.cuda.is_available():
        raise SystemExit("sampling_bench.py needs a CUDA device")
    lib.load()
    hp = dict(speech_transformer_hparams("speech_transformer_s")["model.params"])
    tm = {"vocab_size": V, "eos_id": V - 1, "bos_id": V - 2, "unk_id": V - 3}
    model = SpeechTransformer.new(hp, {"audio_feature_dim": 80, "audio_feature_channels": 1}, tm, precision="fp16")
    model.init_parameters(1234)
    rt = model.runtime
    g = torch.Generator().manual_seed(5)
    enc, bias = D.encode(rt, dict(src=torch.randn(UTT, T, 80, 1, generator=g), src_length=torch.full((UTT,), T)))
    bos, eos, unk = tm["bos_id"], tm["eos_id"], tm["unk_id"]
    # the reference requires minimum < maximum decode length: EOS is masked for the first 149 positions
    cache = D.create_decoding_cache(rt, enc, bias, STEPS + 1, use_shadow=True, beam=SAMPLES)
    kw = dict(maximum_decode_length=STEPS + 1, extra_decode_length=STEPS, minimum_decode_length=STEPS, use_shadow=True, cache=cache)

    def sample(top_k, top_p):
        return lambda: D.sampling_search(rt, None, bos, eos, unk, sample_num=SAMPLES, top_k=top_k, top_p=top_p, **kw)[2]

    def beam():
        return D.beam_search(rt, None, bos, eos, unk, beam_size=SAMPLES, top_k=SAMPLES, length_penalty=-1.0, **kw)[3]

    return {"sample_topk0": sample(0, 1.0), "sample_topk10": sample(10, 1.0), "sample_topp09": sample(0, 0.9), "beam4": beam}


def profile():
    """One run of each arm under torch.profiler: per-token CUDA time of the selection kernels."""
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    runs = arms()
    for run in runs.values():
        run()
    torch.cuda.synchronize()
    out = {}
    for name, run in runs.items():
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            ln = run()
            torch.cuda.synchronize()
        tokens = int(ln.max())
        us = {"sample_select_kernel": 0.0, "beam_select_kernel": 0.0}
        for e in p.events():
            for k in us:
                if k in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
                    us[k] += e.device_time
        out[name] = {k: v / tokens for k, v in us.items() if v > 0}
    print(json.dumps(out))


def main():
    import torch
    runs = arms()
    for run in runs.values():           # warm-up: module loading, graph capture paths, shared-memory attributes
        run()
    torch.cuda.synchronize()
    res = {k: [] for k in runs}
    positions = {}
    for _ in range(REPEATS):
        for name, run in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ln = run()
            e1.record()
            torch.cuda.synchronize()
            positions[name] = int(ln.max())
            res[name].append(e0.elapsed_time(e1) * 1e3 / positions[name])
    del runs
    torch.cuda.empty_cache()
    env = dict(os.environ, B200ST_NO_PDL="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--profile"], capture_output=True, text=True, env=env)
    kernels = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else {"error": r.stderr[-2000:]}
    info = gpu_info()
    out = {"gpu": info, "workload": "speech_transformer_s fp16 shadow, %d utterances [%d,%d,80] x %d samples = %d rows, %d positions "
                                    "(EOS masked), search only" % (UTT, UTT, T, SAMPLES, UTT * SAMPLES, STEPS),
           "us_per_token": {k: {"median": sorted(v)[len(v) // 2], "min": min(v), "max": max(v), "runs": v} for k, v in res.items()},
           "positions": positions, "selection_kernel_us_per_token": kernels}
    print("GPU %s, power limit %s, SM clock %s (max %s)" % (info.get("name"), info.get("power.limit"), info.get("clocks.sm"),
                                                            info.get("clocks.max.sm")))
    for k, v in out["us_per_token"].items():
        sel = kernels.get(k, {}) if isinstance(kernels, dict) else {}
        print("%-14s %8.1f us/token (min %.1f, max %.1f, %d positions)  selection kernel %s us/token" %
              (k, v["median"], v["min"], v["max"], positions[k], ", ".join("%s %.1f" % kv for kv in sel.items()) or "n/a"))
    if "error" in kernels:
        print("profile run failed:", kernels["error"])
    path = os.path.join(tempfile.gettempdir(), "sampling_bench.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print("written to", path)


if __name__ == "__main__":
    profile() if "--profile" in sys.argv else main()
