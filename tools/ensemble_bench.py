"""Ensemble beam search on the wide step: speech_transformer_s members, fp16 shadow weights, 64 utterances x beam 4 (256 rows),
inputs [64, 2000, 80] (Tm 500), 150 decoding steps forced by minimum_decode_length (EOS masked until then), random-init
weights (one seed per member).

Reports us per token (search only: CUDA events around the search; encoders and cache set-up are outside) for the plain
single-model beam_search and for ensembles of 1, 2 and 3 members, with the sum of the members' single-model steps beside
each ensemble.  A separate torch.profiler pass over one 2-member search gives the mean kernel time of the mixing kernel and
of the selection kernel, and the bytes the mixing kernel must move (computed from shapes) against the H100 SXM data-sheet
HBM bandwidth of 3.35 TB/s.  Prints the card's name and power limit read in the same run and writes
bench_out/ensemble_bench.json.

    python tools/ensemble_bench.py
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STEPS, T, V, BEAM, U, REPEATS = 150, 2000, 8192, 4, 64, 3
HBM = 3.35e12


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
        raise SystemExit("ensemble_bench.py needs a CUDA device")
    lib.load()
    info = gpu_info()
    hp = dict(speech_transformer_hparams("speech_transformer_s")["model.params"])
    tm = {"vocab_size": V, "eos_id": V - 1, "bos_id": V - 2, "unk_id": V - 3}
    rts = []
    for seed in (1234, 1235, 1236):
        model = SpeechTransformer.new(hp, {"audio_feature_dim": 80, "audio_feature_channels": 1}, tm, precision="fp16")
        model.init_parameters(seed)
        rts.append(model.runtime)
    g = torch.Generator().manual_seed(5)
    inputs = dict(src=torch.randn(U, T, 80, 1, generator=g), src_length=torch.full((U,), T, dtype=torch.long))
    bos, eos, unk = tm["bos_id"], tm["eos_id"], tm["unk_id"]
    kw = dict(beam_size=BEAM, length_penalty=-1.0, maximum_decode_length=STEPS, extra_decode_length=STEPS,
              minimum_decode_length=STEPS - 1, use_shadow=True)
    memories = [D.encode(rt, inputs) for rt in rts]

    def caches(n):
        return [D.create_decoding_cache(rt, enc, bias, STEPS, use_shadow=True, beam=BEAM) for rt, (enc, bias) in zip(rts[:n], memories[:n])]

    def timed(fn):
        fn()                                              # warm-up: graph capture, module loads, tensor maps
        best = None
        for _ in range(REPEATS):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / STEPS
            best = us if best is None else min(best, us)
        return best

    def plain(i):
        c = caches(i + 1)[i]
        return lambda: D.beam_search(rts[i], None, bos, eos, unk, cache=c, **kw)

    def ensemble(n):
        c = caches(n)
        return lambda: D.ensemble_beam_search(rts[:n], None, bos, eos, unk, weights="average", caches=c, **kw)

    res = {"gpu": info, "steps": STEPS, "beam": BEAM, "utterances": U, "rows": U * BEAM, "us_per_token": {}}
    single = [timed(plain(i)) for i in range(3)]
    res["us_per_token"]["beam_search member %d" % 1] = round(single[0], 1)
    print("[%s, power limit %s] %d utterances x beam %d (%d rows), %d steps" % (info.get("name"), info.get("power.limit"), U, BEAM,
                                                                            U * BEAM, STEPS), flush=True)
    print("  plain beam_search, member 1:          %8.1f us/token  (members 2, 3 alone: %.1f, %.1f)" % (single[0], single[1], single[2]),
          flush=True)
    for n in (1, 2, 3):
        us = timed(ensemble(n))
        res["us_per_token"]["ensemble of %d" % n] = round(us, 1)
        res["us_per_token"]["sum of %d single-model steps" % n] = round(sum(single[:n]), 1)
        print("  ensemble of %d member(s):              %8.1f us/token  (sum of the members' single-model steps %.1f)" %
              (n, us, sum(single[:n])), flush=True)

    # kernel times of one 2-member search, in a profiled run of its own
    try:
        from torch.profiler import ProfilerActivity, profile
        fn = ensemble(2)
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.events():
            for key in ("ensemble_logprob_kernel", "beam_select_kernel"):
                if key in e.name:
                    kern.setdefault(key, []).append(e.device_time if hasattr(e, "device_time") else e.cuda_time)
        mix_bytes = 3 * U * BEAM * V * 4                  # reads both members' logits [256, 8192] fp32, writes one
        for key, t in kern.items():
            mean = sum(t) / len(t)
            row = {"launches": len(t), "mean_us": round(mean, 2)}
            if key == "ensemble_logprob_kernel":
                row.update(bytes=mix_bytes, GB_per_s=round(mix_bytes / (mean * 1e-6) / 1e9, 1),
                           share_of_3_35TB_s=round(mix_bytes / (mean * 1e-6) / HBM, 3))
            res[key] = row
            print("  %-26s %4d launches, mean %7.2f us%s" % (key, len(t), mean, (", %.1f MB -> %.0f GB/s (%.0f%% of 3.35 TB/s)" % (
                mix_bytes / 1e6, row["GB_per_s"], 100 * row["share_of_3_35TB_s"])) if "GB_per_s" in row else ""), flush=True)
    except Exception as e:  # noqa
        res["profile_error"] = str(e)
        print("  kernel profile not available: %s" % e, flush=True)
    os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
    with open(os.path.join(ROOT, "bench_out", "ensemble_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
