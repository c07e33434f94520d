"""Wait-k simultaneous translation on the device at transformer_base (d=512, 6+6 layers, ffn 2048), fp16, random-init
weights, V = 8192 on both sides:

  train    one captured CUDA-graph training step (the trainer's bucket step) of 192 pairs x 64 source and 64 target
           positions: the plain Transformer, then the WaitkTransformer (monotonic encoder, wait-k cross-attention with a
           k drawn from [3, 5, 7] per step) on the same bucket.  Reports ms per step over timed steps that end in a device
           synchronise.
  decode   64 sentences of 40 source tokens, maximum_decode_length 60 from the fp16 shadow weights: greedy and beam 4 at
           k = 3 against no lag (wait_k = 0), the same weights.  Reports ms per decoded position (time of the search over
           its number of steps), mean of the timed calls.

Prints the GPU name and power limit next to the numbers.  Without a GPU it fails: nothing is measured on the CPU.

    python tools/waitk_bench.py
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from mt_bench import gpu_info, meta  # noqa: E402


def _model(waitk, V):
    from neurst_b200.models import Transformer, WaitkTransformer, transformer_hparams, waitk_transformer_hparams
    if waitk:
        hp = waitk_transformer_hparams("waitk_transformer_base")
        m = WaitkTransformer.new(hp["model.params"], meta(V), meta(V), precision="fp16", label_smoothing=0.1, wait_k=[3, 5, 7],
                                 random_seed=1)
    else:
        hp = transformer_hparams("transformer_base")
        m = Transformer.new(hp["model.params"], meta(V), meta(V), precision="fp16", label_smoothing=0.1)
    return m.init_parameters(1), hp


def train(steps=20, warmup=3, B=192, T=64, Lq=64, V=8192):
    import torch
    from neurst_b200.trainer import DataParallelTrainer
    g = torch.Generator().manual_seed(2)
    trg = torch.randint(0, V - 3, (B, Lq), generator=g)
    trg[:, -1] = V - 1
    batch = {"src": torch.randint(0, V - 3, (B, T), generator=g), "src_padding": torch.zeros(B, T),
             "trg": trg, "trg_input": torch.cat([torch.full((B, 1), V - 2), trg[:, :-1]], 1), "trg_length": torch.full((B,), Lq)}
    batch = {k: v.cuda() for k, v in batch.items()}
    res = {}
    for name in ("transformer", "waitk_transformer"):
        model, hp = _model(name != "transformer", V)
        tr = DataParallelTrainer(model, hp["optimizer.params"], hp["lr_schedule.params"], use_cuda_graph=True)
        for i in range(warmup):
            tr.train_step(batch, seed=i + 1)
        torch.cuda.synchronize()
        t0 = time.time()
        for i in range(steps):
            tr.train_step(batch, seed=warmup + i + 1)
        torch.cuda.synchronize()
        res[name] = {"ms_per_step": (time.time() - t0) / steps * 1e3}
        del tr, model
    res["bucket"] = {"B": B, "T": T, "L": Lq}
    return res


def decode(calls=3, U=64, T=40, V=8192, max_len=60):
    import torch
    from neurst_b200 import decode as D
    model, _ = _model(False, V)
    rt = model.runtime
    g = torch.Generator().manual_seed(5)
    inputs = {"src": torch.randint(0, V - 3, (U, T), generator=g), "src_padding": torch.zeros(U, T)}
    inputs["src"][:, -1] = V - 1
    res = {}
    for search, beam in (("greedy", 1), ("beam4", 4)):
        for k in (0, 3):
            def run():
                if beam == 1:
                    ids, _, length = D.greedy_search(rt, inputs, V - 2, V - 1, V - 3, max_len, 50, 0, use_shadow=True, wait_k=k)
                else:
                    ids, _, _, length = D.beam_search(rt, inputs, V - 2, V - 1, V - 3, beam_size=beam, maximum_decode_length=max_len,
                                                      use_shadow=True, wait_k=k)
                return int(length.max())
            run()
            torch.cuda.synchronize()
            times, steps = [], 0
            for _ in range(calls):
                t0 = time.time()
                steps = run()
                torch.cuda.synchronize()
                times.append(time.time() - t0)
            res["%s_k%d" % (search, k)] = {"ms_per_position": sum(times) / len(times) / max(steps, 1) * 1e3, "positions": steps}
    res["sentences"], res["source_tokens"] = U, T
    return res


def main():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("waitk_bench measures on a CUDA device: not measured")
    print(json.dumps({"gpu": gpu_info(), "train": train(), "decode": decode()}))


if __name__ == "__main__":
    main()
