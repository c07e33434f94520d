"""Streaming simultaneous translation (b200st_stream_*) at waitk_transformer_big (d=1024, 16 heads, 6+6 layers, ffn 4096),
random-init weights, V = 32000 on both sides, with 1 and 3 members, from the fp16 shadow and from the fp32 weights:

  read      microseconds per READ of a 1-, 2- and 4-token word appended to a source of 10 / 40 / 100 tokens (every member
            encodes the new rows and appends their cross K/V);
  write     microseconds per WRITE (the captured step of every member, the mixture, the argmax) and its pinned id read;
  reencode  the same READ done the only other way: b200st_encode of the whole prefix plus b200st_decode_init, per member.

Each number is the mean over timed repetitions between device synchronisations, after a warm-up.  Prints the GPU name and
power limit next to a table, and the JSON of every number (also to --json PATH).  Without a GPU it fails.

    python tools/simul_bench.py [--json PATH]
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from mt_bench import gpu_info, meta  # noqa: E402

V = 32000


def _members(n, precision):
    from neurst_b200.models import WaitkTransformer, waitk_transformer_hparams
    hp = waitk_transformer_hparams("waitk_transformer_big")
    return [WaitkTransformer.new(hp["model.params"], meta(V), meta(V), precision=precision, wait_k=3).init_parameters(i + 1)
            for i in range(n)]


def _time(fn, reps, setup=None):
    import torch
    total = 0.0
    for _ in range(reps):
        if setup:
            setup()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        total += time.perf_counter() - t0
    return total / reps * 1e6


def run(n, precision, reps=20):
    import torch
    from neurst_b200 import decode as D
    from neurst_b200.simultaneous import StreamingSession
    models = _members(n, precision)
    shadow = precision != "fp32"
    s = StreamingSession(models, use_shadow=shadow, max_src=128, max_trg=128)
    g = torch.Generator().manual_seed(3)
    src = torch.randint(0, V - 3, (110,), generator=g)
    out = {"read_us": {}, "reencode_us": {}}
    for L in (10, 40, 100):
        for w in (1, 2, 4):
            def prefix():
                s.reset()
                s.read(src[:L])
            _time(lambda: s.read(src[L:L + w]), 3, prefix)
            out["read_us"]["%d+%d" % (L, w)] = _time(lambda: s.read(src[L:L + w]), reps, prefix)

            def reencode():
                x = dict(src=src[None, :L + w], src_padding=torch.zeros(1, L + w))
                for m in models:
                    enc, bias = D.encode(m.runtime, x)
                    D.create_decoding_cache(m.runtime, enc, bias, 128, use_shadow=shadow)
            reencode()
            out["reencode_us"]["%d+%d" % (L, w)] = _time(reencode, reps)
    s.reset()
    s.read(src[:40])
    for _ in range(3):
        s.write()
    steps = 60
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        s.write()
    out["write_us"] = (time.perf_counter() - t0) / steps * 1e6
    return out


def main():
    info = gpu_info()
    res = {"gpu": info, "model": "waitk_transformer_big, V=%d" % V, "runs": {}}
    for precision in ("fp16", "fp32"):
        for n in (1, 3):
            key = "%s_shadow x%d" % (precision, n) if precision != "fp32" else "fp32 x%d" % n
            res["runs"][key] = run(n, precision)
    print("%s, power limit %s" % (info.get("name"), info.get("power.limit")))
    print("| weights x members | READ 1/2/4 tokens @10 (us) | @40 | @100 | re-encode 1/2/4 @10 | @40 | @100 | WRITE (us) |")
    print("|---|---|---|---|---|---|---|---|")
    for key, r in res["runs"].items():
        cells = []
        for what in ("read_us", "reencode_us"):
            for L in (10, 40, 100):
                cells.append(" / ".join("%.0f" % r[what]["%d+%d" % (L, w)] for w in (1, 2, 4)))
        print("| %s | %s | %.0f |" % (key, " | ".join(cells), r["write_us"]))
    print(json.dumps(res))
    if "--json" in sys.argv:
        with open(sys.argv[sys.argv.index("--json") + 1], "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
