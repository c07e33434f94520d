"""Beam search over many utterances per call: speech_transformer_s, fp16 shadow weights, beam 4, inputs [B, 2000, 80]
(Tm 500), 150 decoding steps forced by minimum_decode_length (EOS masked until then), random-init weights.

1. For 2, 16 and 64 utterances per call (8, 64 and 256 rows per step; 8 rows is the GEMV step, more the wide step):
   us per token (search only, CUDA events around the search; the encoder and the cache set-up are outside), row-tokens/s,
   and the bytes a token must read computed from shapes (16-bit decoder weights, fp32 cross K/V, fp32 self K/V at the mean
   position) with the rate that implies against the H100 SXM data-sheet HBM bandwidth of 3.35 TB/s.
2. The same 64 utterances decoded as 32 calls of 2 and as 1 call of 64, wall clock including the encoder passes.

Prints the card's name and power limit read in the same run, and writes bench_out/decode_rows_bench.json.

    python tools/decode_rows_bench.py
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STEPS, T, V, BEAM, REPEATS = 150, 2000, 8192, 4, 3
HBM = 3.35e12


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # noqa
        return {"error": str(e)}


def token_bytes(cfg, U, Tm, mean_pos):
    """Bytes one decoding step reads at U utterances x beam: the decoder's 16-bit weights once, the fp32 cross K/V of every
    utterance once (the wide step reads it once per utterance), the fp32 self K/V of every row up to the mean position."""
    d, f, L, Vv = cfg["d"], cfg["ffn"], cfg["dec_layers"], cfg["vocab"]
    weights = 2 * (L * (3 * d * d + d * d + d * d + d * d + 2 * d * f) + Vv * d)
    cross = 4 * L * U * Tm * 2 * d
    self_kv = 4 * L * U * BEAM * mean_pos * 2 * d
    return weights, cross, self_kv


def main():
    import torch
    from neurst_b200 import decode as D
    from neurst_b200 import lib
    from neurst_b200.models import SpeechTransformer, speech_transformer_hparams
    from oracle import restatement as R
    if not torch.cuda.is_available():
        raise SystemExit("decode_rows_bench.py needs a CUDA device")
    lib.load()
    info = gpu_info()
    hp = dict(speech_transformer_hparams("speech_transformer_s")["model.params"])
    tm = {"vocab_size": V, "eos_id": V - 1, "bos_id": V - 2, "unk_id": V - 3}
    model = SpeechTransformer.new(hp, {"audio_feature_dim": 80, "audio_feature_channels": 1}, tm, precision="fp16")
    model.init_parameters(1234)
    rt = model.runtime
    cfg = dict(R.CONFIGS["speech_transformer_s"])
    g = torch.Generator().manual_seed(5)
    src64 = torch.randn(64, T, 80, 1, generator=g)
    lens64 = torch.full((64,), T, dtype=torch.long)
    bos, eos, unk = tm["bos_id"], tm["eos_id"], tm["unk_id"]
    kw = dict(beam_size=BEAM, length_penalty=-1.0, maximum_decode_length=STEPS, extra_decode_length=STEPS,
              minimum_decode_length=STEPS - 1, use_shadow=True)

    def search(inputs):
        return D.beam_search(rt, inputs, bos, eos, unk, **kw)

    res = {"gpu": info, "steps": STEPS, "beam": BEAM, "T": T, "per_call": {}}
    for U in (2, 16, 64):
        enc, bias = D.encode(rt, dict(src=src64[:U], src_length=lens64[:U]))
        Tm = enc.shape[1]

        def run():
            cache = D.create_decoding_cache(rt, enc, bias, STEPS, use_shadow=True, beam=BEAM)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            D.beam_search(rt, None, bos, eos, unk, cache=cache, **kw)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) * 1e3
        run()                                             # warm-up: graph capture, module loads, tensor maps
        us = min(run() for _ in range(REPEATS))
        us_tok = us / STEPS
        w, c, s = token_bytes(cfg, U, Tm, STEPS / 2)
        total = w + c + s
        row = {"rows": U * BEAM, "Tm": Tm, "us_per_token": round(us_tok, 2),
               "row_tokens_per_s": round(U * BEAM * STEPS / (us * 1e-6)),
               "bytes_per_token": {"weights": w, "cross_kv": c, "self_kv_mean": s, "total": total},
               "GB_per_s": round(total / (us_tok * 1e-6) / 1e9, 1), "share_of_3.35TB_s": round(total / (us_tok * 1e-6) / HBM, 3)}
        res["per_call"][U] = row
        print("[%s, power limit %s] %3d utterances x beam %d (%3d rows): %8.1f us/token  %10.0f row-tokens/s  %6.1f MB/token  "
              "%7.1f GB/s (%.1f%% of 3.35 TB/s)" % (info.get("name"), info.get("power.limit"), U, BEAM,
                                                     U * BEAM, us_tok, row["row_tokens_per_s"], total / 1e6, row["GB_per_s"],
                                                     100 * row["share_of_3.35TB_s"]), flush=True)
        del enc, bias

    def wall(per_call):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(0, 64, per_call):
            search(dict(src=src64[i:i + per_call], src_length=lens64[i:i + per_call]))
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    wall(2), wall(64)                                     # warm-up
    times = {2: [], 64: []}
    for _ in range(REPEATS):                              # alternated
        times[2].append(wall(2))
        times[64].append(wall(64))
    res["64_utterances_wall_s"] = {"32_calls_of_2": round(min(times[2]), 3), "1_call_of_64": round(min(times[64]), 3)}
    print("64 utterances, encoder included: 32 calls of 2 %.3f s, 1 call of 64 %.3f s (%.1fx)" %
          (min(times[2]), min(times[64]), min(times[2]) / min(times[64])), flush=True)
    os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
    with open(os.path.join(ROOT, "bench_out", "decode_rows_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
