"""Machine translation and cascade ST on the device, random-init weights:

  mt_train   transformer_s (d=256, 6+6 layers, ffn 2048, V = 8192 on both sides) training at the MT recipe's 25,000-token
             batches, fp16, one captured CUDA graph per step (the trainer's bucket step): one bucket of 390 pairs x 64 source
             and 64 target positions (24,960 target tokens, every row full).  Reports target tokens/s over timed steps
             that end in a device synchronise.
  cascade    64-utterance groups ([64,1000,80] fbank) through speech_transformer_s (ASR) then transformer_s (MT), beam 4 on
             both stages, fp16 shadow weights, maximum_decode_length 100: ASR search, b200st_cascade_source, MT search.
             Reports the time per utterance of the whole group (encoders included), mean of the timed groups.

Prints the GPU name and power limit next to the numbers.  Without a GPU it fails: nothing is measured on the CPU.

    python tools/mt_bench.py
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = "name,power.limit"
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def meta(V):
    return {"vocab_size": V, "unk_id": V - 3, "bos_id": V - 2, "eos_id": V - 1, "pad_id": V - 1}


def mt_train(steps=20, warmup=3, B=390, T=64, Lq=64, V=8192):
    import torch
    from neurst_b200.models import Transformer, transformer_hparams
    from neurst_b200.trainer import DataParallelTrainer
    hp = transformer_hparams("transformer_s")
    model = Transformer.new(hp["model.params"], meta(V), meta(V), precision="fp16", label_smoothing=0.1).init_parameters(1)
    tr = DataParallelTrainer(model, hp["optimizer.params"], hp["lr_schedule.params"], use_cuda_graph=True)
    g = torch.Generator().manual_seed(2)
    trg = torch.randint(0, V - 3, (B, Lq), generator=g)
    trg[:, -1] = V - 1
    batch = {"src": torch.randint(0, V - 3, (B, T), generator=g), "src_padding": torch.zeros(B, T),
             "trg": trg, "trg_input": torch.cat([torch.full((B, 1), V - 2), trg[:, :-1]], 1),
             "trg_length": torch.full((B,), Lq)}
    batch = {k: v.cuda() for k, v in batch.items()}
    for i in range(warmup):
        tr.train_step(batch, seed=i + 1)
    torch.cuda.synchronize()
    t0 = time.time()
    for i in range(steps):
        loss = tr.train_step(batch, seed=warmup + i + 1)
    torch.cuda.synchronize()
    dt = (time.time() - t0) / steps
    return {"ms_per_step": dt * 1e3, "trg_tokens_per_step": B * Lq, "trg_tokens_per_sec": B * Lq / dt,
            "src_tokens_per_sec": B * T / dt, "loss": float(loss)}


def cascade(groups=3, U=64, T=1000, V=8192, beam=4, max_len=100):
    import torch
    from neurst_b200 import decode as D
    from neurst_b200.models import SpeechTransformer, Transformer, speech_transformer_hparams, transformer_hparams
    asr = SpeechTransformer.new(speech_transformer_hparams("speech_transformer_s")["model.params"],
                                {"audio_feature_dim": 80, "audio_feature_channels": 1}, meta(V), precision="fp16").init_parameters(3)
    mt = Transformer.new(transformer_hparams("transformer_s")["model.params"], meta(V), meta(V), precision="fp16").init_parameters(4)
    remap = torch.arange(V, dtype=torch.int32).cuda()                    # a shared vocabulary (MuST-C's vocab.en)
    g = torch.Generator().manual_seed(5)
    audio = torch.randn(U, T, 80, 1, generator=g).cuda()
    lens = torch.full((U,), T, dtype=torch.long).cuda()
    kw = dict(beam_size=beam, length_penalty=0.6, maximum_decode_length=max_len, use_shadow=True)

    def run():
        ids, _ = asr.beam_search({"src": audio, "src_length": lens}, **kw)
        src, pad, _ = D.cascade_source(ids, remap, V - 1, V, V - 1, V - 1, V - 3)
        out, _ = mt.beam_search({"src": src, "src_padding": pad}, **kw)
        return src.shape[1], out
    run()
    torch.cuda.synchronize()
    times = []
    for _ in range(groups):
        t0 = time.time()
        width, _ = run()
        torch.cuda.synchronize()
        times.append(time.time() - t0)
    return {"ms_per_utterance": sum(times) / len(times) / U * 1e3, "ms_per_group": [t * 1e3 for t in times],
            "utterances_per_group": U, "mt_source_positions": width}


def main():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mt_bench measures on a CUDA device: not measured")
    res = {"gpu": gpu_info(), "mt_train": mt_train(), "cascade": cascade()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
