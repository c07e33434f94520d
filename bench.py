#!/usr/bin/env python
"""bench.py — audio-frames/sec (fwd+bwd[+all-reduce]+Adam) of SpeechTransformer-base on N H100s.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--dump-outputs DIR]   # this repo's CUDA path (libb200st)
  python bench.py --impl reference [--steps K] [--warmup W]      # the reference algorithm's CPU path (oracle port)
  torchrun --nnodes=1 --nproc-per-node N ... bench.py --gpus N   # one rank per GPU, NCCL

Workload (BASELINE.json configs[1], SURVEY.md §8d cfg-2): speech_transformer_s (conv2d subsample + 12 enc / 6 dec,
d=256, ffn=2048, V=8192), synthetic fbank [32,1000,80] per GPU, L=88, dropout 0.1, label smoothing 0.1, bf16 tensor-core
operands with fp32 accumulation / residual stream / statistics / loss / Adam.  One JSON line on stdout (rank 0).
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

WORKLOADS = {
    # BASELINE.json configs[1] (SURVEY §8d cfg-2): the configuration the headline metric is quoted on
    "cfg2": dict(hparams="speech_transformer_s", B=32, T=1000, F=80, L=88, V=8192, d=256, H=4, ffn=2048),
    # configs[2] (cfg-3): global [64,1500,80] over 8 GPUs = 8 utterances per GPU (strong-scaling share); "cfg3w" = 64 per GPU
    "cfg3": dict(hparams="speech_transformer_s", B=8, T=1500, F=80, L=128, V=8192, d=256, H=4, ffn=2048),
    "cfg3w": dict(hparams="speech_transformer_s", B=64, T=1500, F=80, L=128, V=8192, d=256, H=4, ffn=2048),
    # configs[3] (cfg-4): speech_transformer_m, frame budget 24000 / GPU, length buckets, ragged src_length (see run_gpu)
    "cfg4": dict(hparams="speech_transformer_m", B=8, T=3000, F=80, L=152, V=8192, d=512, H=8, ffn=2048, ragged=True),
}
WORKLOAD = WORKLOADS["cfg2"]
# SURVEY.md §8(d): 2*M*N*K of every contraction, fwd+bwd = 3x fwd, padded positions counted
MFLOP_PER_FRAME = 53.24


def flops_per_step(B, T, L, V=8192, d=256, H=4, ffn=2048, C=256, F=80, enc=12, dec=6):
    T1, F1 = (T + 1) // 2, (F + 1) // 2
    T2, F2 = (T1 + 1) // 2, (F1 + 1) // 2
    M, Md, dh = B * T2, B * L, d // H
    fwd = 2 * 9 * 1 * C * B * T1 * F1 + 2 * 9 * C * C * B * T2 * F2 + 2 * M * (F2 * C) * d
    fwd += enc * (2 * M * d * 3 * d + 2 * M * d * d + 4 * B * H * T2 * T2 * dh + 4 * M * d * ffn)
    fwd += dec * (2 * Md * d * 4 * d + 4 * B * H * L * L * dh)
    fwd += dec * (2 * Md * d * 2 * d + 2 * M * d * 2 * d + 4 * B * H * L * T2 * dh)
    fwd += dec * 4 * Md * d * ffn + 2 * Md * d * V
    return 3.0 * fwd


def load_peaks():
    """Data-sheet peaks of the H100 SXM (dense 16-bit tensor rate, HBM3 bandwidth, 700 W card): the denominators of the
    `frac` fields, not rates this program has reached."""
    return dict(tflops_sustained=989.0, hbm_gbs=3350.0, source="NVIDIA H100 SXM data sheet")


def dump_outputs(out_dir, trainer, losses):
    """What a caller of the timed path holds after its last step, as float32 .npy files: the loss of every timed step and the
    parameters the last step left behind (a fixed, seeded sample of at most 4 Mi elements: the arena is larger than 64 MB)."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "loss.npy"), np.asarray([float(x) for x in losses], dtype=np.float32))
    params = trainer.rt.params.detach().reshape(-1).float()
    n = params.numel()
    if n > (1 << 22):
        idx = torch.from_numpy(np.sort(np.random.RandomState(1234).choice(n, 1 << 22, replace=False))).to(params.device)
        params = params[idx]
    np.save(os.path.join(out_dir, "params_sample.npy"), params.cpu().numpy())


class ClockSampler(threading.Thread):
    """One long-lived `nvidia-smi -lms 20` process; lines are stamped on arrival and only those that fall inside the
    marked timed windows (resident + e2e regions, GPU under load) are summarised."""

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.stop_flag, self.raw, self.windows, self.proc = index, False, [], [], None
        import atexit
        atexit.register(self.stop)          # never leave the nvidia-smi loop behind, whatever path the process exits by

    def run(self):
        q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
            "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q, "--format=csv,noheader,nounits",
                                          "-lms", "20"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            for line in self.proc.stdout:
                f = [x.strip() for x in line.strip().split(",")]
                if len(f) >= 6:
                    self.raw.append((time.time(), f))
                if self.stop_flag:
                    break
        except Exception:
            pass

    def mark(self, t0, t1):
        self.windows.append((t0, t1))

    def stop(self):
        self.stop_flag = True
        if self.proc is not None:
            try:
                self.proc.terminate()            # the exact child we started
            except Exception:
                pass

    @property
    def samples(self):
        inside = [f for (t, f) in self.raw if any(a <= t <= b for a, b in self.windows)]
        return inside if inside else [f for (_, f) in self.raw[-3:]]

    def summary(self):
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["unavailable"]}
        mhz = sorted(float(s[0]) for s in self.samples if s[0].replace(".", "").isdigit())
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(s[2 + i].lower().startswith("active") for s in self.samples)]
        return {"sm_mhz": mhz[len(mhz) // 2] if mhz else None, "sm_max_mhz": float(self.samples[0][1]), "reasons": reasons,
                "samples": len(self.samples)}


# ------------------------------------------------------------------------------------------------------
# CPU arm: the reference algorithm on host cores (oracle port — the reference's TF2 path cannot run: no TF wheel,
# and the reference tree is not present where the benchmark runs; its PyTorch mirror has no working backward, SURVEY §8c)
# ------------------------------------------------------------------------------------------------------
def cpu_reference_step_time(B, T, L, steps, warmup, threads):
    import torch
    from oracle import restatement as R
    torch.set_num_threads(threads)
    cfg = dict(R.CONFIGS["speech_transformer_s"])
    P = R.init_params(cfg, seed=1234)
    for v in P.values():
        v.requires_grad_(True)
    from neurst_b200.trainer import synthetic_batch
    batch = synthetic_batch(B, T, L, cfg["vocab"], seed=1234)
    g = torch.Generator().manual_seed(7)

    def masks():
        d, H, f = cfg["d"], cfg["heads"], cfg["ffn"]
        T2 = R.length_after_conv(T)
        m = {}

        def mk(name, shape):
            m[name] = torch.rand(shape, generator=g) >= 0.1
        mk("enc.in_drop", (B, T2, d)); mk("dec.in_drop", (B, L, d))
        for i in range(cfg["enc_layers"]):
            mk("enc.%d.att.attn_drop" % i, (B, H, T2, T2)); mk("enc.%d.att.post_drop" % i, (B, T2, d))
            mk("enc.%d.ffn.ffn_drop" % i, (B, T2, f)); mk("enc.%d.ffn.post_drop" % i, (B, T2, d))
        for i in range(cfg["dec_layers"]):
            mk("dec.%d.self.attn_drop" % i, (B, H, L, L)); mk("dec.%d.self.post_drop" % i, (B, L, d))
            mk("dec.%d.cross.attn_drop" % i, (B, H, L, T2)); mk("dec.%d.cross.post_drop" % i, (B, L, d))
            mk("dec.%d.ffn.ffn_drop" % i, (B, L, f)); mk("dec.%d.ffn.post_drop" % i, (B, L, d))
        return R.Masks(0.1, m)

    times = []
    for it in range(warmup + steps):
        t0 = time.perf_counter()
        logits = R.speech_transformer_forward(P, cfg, batch["src"], batch["src_length"], batch["trg_input"], masks())
        loss = R.reduce_loss(logits, batch["trg"], batch["trg_length"], 0.1)
        grads = torch.autograd.grad(loss, list(P.values()))
        with torch.no_grad():   # Adam-free SGD touch so the step is not optimised away; Adam cost is negligible on CPU
            for p_, g_ in zip(P.values(), grads):
                p_.sub_(1e-9 * g_)
        dt = time.perf_counter() - t0
        if it >= warmup:
            times.append(dt)
    times.sort()
    return times[len(times) // 2], float(loss.detach())


def cpu_reference_forward_time(B, T, L, steps, warmup, threads):
    """The UNMODIFIED reference `neurst_pt` SpeechTransformer (staged under oracle/_ref by oracle/build_ref.py), forward only
    (its autograd does not run on this torch, SURVEY 8c), training mode (dropout on), same synthetic batch."""
    import torch
    from oracle import build_ref
    from oracle import restatement as R
    torch.set_num_threads(threads)
    cfg = dict(R.CONFIGS["speech_transformer_s"])
    model = build_ref.reference_speech_transformer(cfg, cfg["vocab"])
    from neurst_b200.trainer import synthetic_batch
    batch = synthetic_batch(B, T, L, cfg["vocab"], seed=1234)
    times = []
    with torch.no_grad():
        for it in range(warmup + steps):
            t0 = time.perf_counter()
            logits = model({"src": batch["src"].clone(), "src_length": batch["src_length"], "trg_input": batch["trg_input"]}, is_training=True)
            dt = time.perf_counter() - t0
            if it >= warmup:
                times.append(dt)
    times.sort()
    return times[len(times) // 2], float(logits.float().abs().mean())


def cpu_threads():
    """Threads of the CPU arm.  The oracle's ops at the bounded sample size stop scaling near 16 intra-op threads, and
    on a shared host more OpenMP threads than free cores is catastrophically slow (spin-waits) — measured: 8 threads
    378 frames/s, 128 threads 112 frames/s on an idle box and > 400 s per step on a loaded one."""
    env = os.environ.get("B200ST_CPU_THREADS")
    return int(env) if env else max(1, min(len(os.sched_getaffinity(0)), 16))


def cpu_sample(B, T, L, steps, warmup, threads, timeout_s, which="--cpu-worker"):
    """Runs the oracle sample in a child process (exact PID, killed on timeout) so that the bench always terminates."""
    env = dict(os.environ, OMP_NUM_THREADS=str(threads), MKL_NUM_THREADS=str(threads), OMP_WAIT_POLICY="PASSIVE",
               KMP_BLOCKTIME="0", CUDA_VISIBLE_DEVICES="")
    cmd = [sys.executable, os.path.abspath(__file__), which, "%d,%d,%d,%d,%d,%d" % (B, T, L, steps, warmup, threads)]
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, env=env)
    try:
        out, _ = proc.communicate(timeout=timeout_s)
        for line in reversed(out.strip().splitlines()):
            if line.startswith("{"):
                return json.loads(line)
    except subprocess.TimeoutExpired:
        proc.kill()
        proc.communicate()
    return None


def cpu_baseline_object(steps, warmup):
    """Bounded CPU sample of the cfg-2 workload: B=2 full-length utterances; a loaded host falls back to one shorter
    utterance rather than stalling the bench."""
    threads = cpu_threads()
    T, L = WORKLOAD["T"], WORKLOAD["L"]
    for (B, Tn, Ln, budget) in ((2, T, L, 150), (1, T // 4, L // 4, 90)):
        r = cpu_sample(B, Tn, Ln, steps, warmup, threads, budget)
        if r is not None:
            sample = "oracle port (fp32 torch-CPU restatement of the reference graph) fwd+bwd, dropout on, B=%d x T=%d frames " \
                     "per step, median of %d step(s) after %d warm-up" % (B, Tn, steps, warmup)
            obj = {"value": B * Tn / r["sec"], "unit": "frames/s", "cores": threads, "kind": "port", "sample": sample}
            # beside it: the unmodified reference itself, for the part of the step it can run (forward only)
            rf = cpu_sample(B, Tn, Ln, steps, warmup, threads, 90, which="--cpu-ref-worker")
            if rf is not None and rf.get("sec"):
                obj["reference_forward"] = {"value": B * Tn / rf["sec"], "unit": "frames/s (forward only)", "kind": "reference", "cores": threads,
                                            "sample": "unmodified reference neurst_pt.SpeechTransformer.forward(is_training=True) staged under oracle/_ref "
                                                      "(oracle/build_ref.py), same batch; the reference has no runnable backward"}
            return obj, r["sec"], (B, Tn, Ln)
    return None, None, None


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    steps, warmup = max(1, min(args.steps, 3)), max(1, min(args.warmup, 1))
    cpu, sec, shape = cpu_baseline_object(steps, warmup)
    if cpu is None:
        print(json.dumps({"impl": "reference", "unavailable": "CPU oracle sample exceeded its time budget on this host"}), flush=True)
        return
    val = cpu["value"]
    line = {
        "impl": "reference", "metric": "audio_frames_per_sec_fwd_bwd", "value": val, "unit": "frames/s", "n_gpus": 0,
        "steps": steps, "warmup": warmup, "ms_per_step": sec * 1e3, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "speech_transformer_s fbank[%d,%d,80] L=%d V=8192 (bounded CPU sample of cfg-2)" % shape},
        "cpu_baseline": cpu,
        "e2e": {"value": val, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line), flush=True)


def cpu_ref_worker(spec):
    B, T, L, steps, warmup, threads = [int(x) for x in spec.split(",")]
    try:
        sec, chk = cpu_reference_forward_time(B, T, L, steps, warmup, threads)
        print(json.dumps({"sec": sec, "check": chk}), flush=True)
    except Exception as e:       # no staged reference on this box: the port number stands alone
        print(json.dumps({"sec": None, "error": str(e)[:200]}), flush=True)


def cpu_worker(spec):
    B, T, L, steps, warmup, threads = [int(x) for x in spec.split(",")]
    sec, loss = cpu_reference_step_time(B, T, L, steps, warmup, threads)
    print(json.dumps({"sec": sec, "loss": loss}), flush=True)


# ------------------------------------------------------------------------------------------------------
# GPU arm
# ------------------------------------------------------------------------------------------------------
def encoder_block_roofline(WL, dtype, peaks, iters=20):
    import torch
    from neurst_b200.layers import TransformerEncoder
    B, T, d, H, ffn = WL["B"], WL["T"], WL["d"], WL["H"], WL["ffn"]
    T2 = ((T + 1) // 2 + 1) // 2
    nl = 12
    enc = TransformerEncoder(nl, d, H, ffn, attention_dropout_rate=0.1, ffn_dropout_rate=0.1, layer_postprocess_dropout_rate=0.1,
                             precision=dtype)
    g = torch.Generator().manual_seed(3)
    P = {k: (torch.randn(shp, generator=g) * (0.05 if len(shp) > 1 else 0.0) + (1.0 if k.endswith("gamma") else 0.0))
         for k, (_, shp) in enc.runtime.table.items()}
    enc.load_parameters(P)
    enc.frozen_parameters = True          # no 16-bit shadow refresh inside the timed calls
    x = torch.randn(B, T2, d, device="cuda")
    pad = torch.zeros(B, T2, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            enc(x, pad, is_training=True)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()           # one graph = the 12-layer forward (no host launch gaps between the kernels)
    with torch.cuda.graph(graph):
        enc(x, pad, is_training=True)
    graph.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    us_layer = e0.elapsed_time(e1) * 1e3 / iters / nl
    M, dh = B * T2, d // H
    gf = (2 * M * d * 3 * d + 2 * M * d * d + 4 * B * H * T2 * T2 * dh + 4 * M * d * ffn) / 1e9
    tf = gf / us_layer * 1e3           # GFLOP / us = PFLOP/s
    return {"what": "TransformerEncoder forward (dropout on) replayed as one CUDA graph, time / 12 layers (includes 1/12 of the "
                    "input cast and final LayerNorm)", "fwd_us_per_layer": us_layer, "gflop_per_layer": gf, "achieved": tf,
            "unit": "TFLOP/s", "frac": tf / peaks["tflops_sustained"]}


def run_decode(args):
    """BASELINE configs[4] (cfg-5): greedy decode of one [1,2000,80] utterance, speech_transformer_s, 200 steps."""
    import torch
    from neurst_b200 import lib, decode as D
    from neurst_b200.models import SpeechTransformer, speech_transformer_hparams
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device: the product path has no CPU fallback")
    lib.load()
    V, T, steps = 8192, 2000, 200
    sampler = ClockSampler(0)
    sampler.start()
    t_w0 = time.time()
    hp = dict(speech_transformer_hparams("speech_transformer_s")["model.params"])
    tm = {"vocab_size": V, "eos_id": V - 1, "bos_id": V - 2, "unk_id": V - 3}
    out = {}
    for dtype, shadow in (("fp32", False), ("fp16", True)):
        model = SpeechTransformer.new(hp, {"audio_feature_dim": 80, "audio_feature_channels": 1}, tm, precision=dtype)
        model.init_parameters(1234)
        rt = model.runtime
        g = torch.Generator().manual_seed(5)
        src = torch.randn(1, T, 80, 1, generator=g).pin_memory()
        inputs = dict(src=src, src_length=torch.tensor([T]))
        # never-EOS decoding: minimum_decode_length = steps forces all 200 positions to be decoded
        kw = dict(maximum_decode_length=steps, extra_decode_length=steps, minimum_decode_length=steps, use_shadow=shadow)
        for _ in range(2):
            D.greedy_search(rt, inputs, tm["bos_id"], tm["eos_id"], tm["unk_id"], **kw)
        torch.cuda.synchronize()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        enc, bias = D.encode(rt, {k: v.cuda(non_blocking=True) for k, v in inputs.items()})
        cache = D.create_decoding_cache(rt, enc, bias, steps, shadow)
        e[1].record()
        ids, lp, ln = D.greedy_search(rt, inputs, tm["bos_id"], tm["eos_id"], tm["unk_id"], cache=cache, **kw)
        mode = int(rt.lib.b200st_greedy_used_graph())          # 2 = persistent cooperative kernel
        host_ids = ids.cpu()
        e[2].record()
        torch.cuda.synchronize()
        enc_ms, dec_ms = e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2])
        # the same search as a per-token CUDA graph (the earlier version), for the comparison
        cache2 = D.create_decoding_cache(rt, enc, bias, steps, shadow)
        D.greedy_search(rt, inputs, tm["bos_id"], tm["eos_id"], tm["unk_id"], cache=cache2, persistent=False, **kw)    # warm-up
        cache2 = D.create_decoding_cache(rt, enc, bias, steps, shadow)
        g0, g1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        g0.record()
        D.greedy_search(rt, inputs, tm["bos_id"], tm["eos_id"], tm["unk_id"], cache=cache2, persistent=False, **kw)
        g1.record()
        torch.cuda.synchronize()
        out[dtype] = dict(encode_ms=enc_ms, decode_ms=dec_ms, us_per_token=dec_ms * 1e3 / steps, tokens=int(ln[0]),
                          weights="16-bit shadow" if shadow else "fp32 master", mode=mode,
                          us_per_token_graph_replay=g0.elapsed_time(g1) * 1e3 / steps)
    sampler.mark(t_w0, time.time())
    sampler.stop()
    wbytes = 10.8e6          # decoder + tied embedding parameters read per token
    peaks = load_peaks()
    best = out["fp16"]
    floor_us = wbytes * 2 / (peaks["hbm_gbs"] * 1e9) * 1e6
    line = {"metric": "greedy_decode_tokens_per_sec", "value": 1e6 / best["us_per_token"], "unit": "tokens/s", "n_gpus": 1,
            "steps": steps, "warmup": 2, "ms_per_step": best["us_per_token"] / 1e3, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "fp32 arithmetic, fp16 weights (fp32-weight variant alongside)", "data": "synthetic",
            "config": {"workload": "cfg-5: speech_transformer_s greedy decode, one utterance [1,2000,80], 200 steps, preallocated "
                                   "KV caches, ONE persistent cooperative kernel for the whole search", "per_precision": out},
            "roofline": {"bound": "hbm", "achieved": wbytes * 2 / (best["us_per_token"] * 1e-6) / 1e9, "peak": peaks["hbm_gbs"],
                         "unit": "GB/s", "frac": floor_us / best["us_per_token"], "traffic": None,
                         "note": "algorithmic bytes per token = 21.6 MB of 16-bit decoder + embedding weights (+ 6 MB fp32 cross "
                                 "K/V); floor %.1f us/token" % floor_us},
            "e2e": {"value": steps / ((best["encode_ms"] + best["decode_ms"]) * 1e-3), "unit": "tokens/s (encoder pass + cache "
                    "build + 200 steps + ids D2H)", "h2d_bytes_per_step": T * 80 * 4, "d2h_bytes_per_step": steps * 8},
            "clocks": sampler.summary(),
            "gpu_launches": 2}
    print(json.dumps(line), flush=True)



def run_gpu(args):
    import torch
    import torch.distributed as dist
    from neurst_b200 import lib
    from neurst_b200.trainer import build_speech_transformer_trainer, synthetic_batch

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py needs a CUDA device: the product path has no CPU fallback")
    torch.cuda.set_device(local_rank)
    if world > 1:
        # bounded failure with a diagnosis: if a rank is still here after the watchdog period, dump every thread's stack and exit
        import faulthandler
        faulthandler.dump_traceback_later(int(os.environ.get("B200ST_BENCH_WATCHDOG_S", "480")), exit=True)
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        import datetime
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank), timeout=datetime.timedelta(seconds=180))
    lib.load()
    WL = WORKLOADS[args.workload]
    B, T, L, V = WL["B"], WL["T"], WL["L"], WL["V"]
    trainer, _ = build_speech_transformer_trainer(WL["hparams"], V, precision=args.dtype, label_smoothing=0.1, seed=1234,
                                                  use_cuda_graph=not args.no_graph)
    dev = torch.device("cuda", local_rank)

    # resident-input arm: a few distinct batches already in HBM (activations per step ~4 GB >> 50 MB L2)
    n_batches = 4
    if WL.get("ragged"):
        # cfg-4: frame budget 24000 / GPU over the reference's length buckets (neurst/tasks/speech2text.py:38-56,296-310):
        # every rank takes the SAME (T bucket, B = 24000 // T rounded to 8) each step, src_length ~ U(0.6 T, T)
        buckets = [(3000, 8, 152), (2000, 8, 152), (1200, 16, 104), (600, 40, 56)]
        shapes = [buckets[i % len(buckets)] for i in range(n_batches)]
    else:
        shapes = [(T, B, L)] * n_batches
    lens = "ragged" if WL.get("ragged") else "full"
    dev_batches = [synthetic_batch(b_, t_, l_, V, seed=1234 + rank * 100 + i, lengths=lens, device=dev) for i, (t_, b_, l_) in enumerate(shapes)]
    host_batches = [synthetic_batch(b_, t_, l_, V, seed=1234 + rank * 100 + i, lengths=lens, pin=True) for i, (t_, b_, l_) in enumerate(shapes)]
    frames_per_cycle = sum(t_ * b_ for (t_, b_, _) in shapes)
    real_frames_per_cycle = sum(int(b["src_length"].sum()) for b in host_batches)
    h2d = sum(v.numel() * v.element_size() for v in host_batches[0].values())

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(step_fn, steps):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            step_fn(i)
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms)

    losses = []

    def resident_step(i):
        losses.append(trainer.train_step(dev_batches[i % n_batches], seed=i + 1))

    # e2e: the public host loop (neurst_b200.trainer.HostPipeline): every step copies its inputs from pinned host memory
    # and reads its loss back; the copy of step i+1 and the read of step i-1 overlap the kernels of step i.
    from neurst_b200.trainer import HostPipeline
    import itertools
    pipe = HostPipeline(trainer)
    e2e_iter = pipe.run(itertools.cycle(host_batches), seed0=1000)

    def e2e_step(i):
        v = next(e2e_iter)
        if v is not None:
            losses.append(v)

    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()                              # started before the warm-up so that it is streaming by the timed region
    for i in range(max(3, args.warmup)):
        resident_step(i)
    launches0 = lib.launch_count()
    t_w0 = time.time()
    ms_total = timed(resident_step, args.steps)
    sampler.mark(t_w0, time.time())
    launches = lib.launch_count() - launches0
    loss_val = float(losses[-1])
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, trainer, losses[-args.steps:])
    for i in range(2):
        e2e_step(i)
    t_w0 = time.time()
    ms_e2e = timed(e2e_step, args.steps)
    sampler.mark(t_w0, time.time())
    sampler.stop()

    # roofline pass (not timed): per-launch CUDA events around the wgmma GEMM launches of ONE step
    # (every rank runs the same steps — train_step contains the gradient all-reduce — only rank 0 reports)
    torch.cuda.synchronize()
    lib.profile_begin()
    trainer.use_cuda_graph = False          # eager launches so each GEMM can be bracketed by events
    pe0, pe1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    pe0.record()
    resident_step(0)
    pe1.record()
    torch.cuda.synchronize()
    gms, gfl, gn = lib.profile_end()
    gemm = dict(ms=gms, flops=gfl, launches=gn, step_ms=pe0.elapsed_time(pe1))   # same (eager, single-stream) step
    barrier()
    # kernels per step: counted on one eagerly launched step (a CUDA-graph replay re-issues the same kernel nodes)
    trainer.use_cuda_graph = False
    l0 = lib.launch_count()
    resident_step(1)
    torch.cuda.synchronize()
    launches_per_step = lib.launch_count() - l0
    barrier()

    # north-star sub-target: forward time of ONE encoder self-attention + FFN block (23.02 GFLOP at cfg-2), measured on the
    # encoder stack alone (b200st_encoder_forward: 12 layers + final LN, dropout on) with CUDA events
    enc_block = None
    if rank == 0 and not WL.get("ragged"):
        try:
            enc_block = encoder_block_roofline(WL, args.dtype, load_peaks())
        except Exception as e:      # never lose the headline line over the side measurement
            enc_block = {"error": str(e)[:200]}
    cpu = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        cpu, _, _ = cpu_baseline_object(3, 1)
        if cpu is None:
            cpu = {"value": None, "unit": "frames/s", "cores": cpu_threads(), "kind": "port",
                   "sample": "oracle sample exceeded its time budget on this host (loaded CPU)"}
    def leave(code=0):
        # Multi-rank exit: every rank has passed the final barrier; the NCCL communicators (torch's and the library's) are
        # left to the process teardown — ncclCommDestroy is an intra-node collective and a destructor-time call on one rank
        # while another is already gone blocks forever — so the ranks exit without running destructors.
        sys.stdout.flush(); sys.stderr.flush()
        if world > 1:
            os._exit(code)

    if world > 1:
        barrier()                # rank 0 has finished its rank-0-only measurements; all ranks leave together
    if rank != 0:
        leave(0)
        return

    peaks = load_peaks()
    ms_step = ms_total / args.steps
    step_shapes = [shapes[i % n_batches] for i in range(args.steps)]
    frames = world * sum(t_ * b_ for (t_, b_, _) in step_shapes) / args.steps            # padded frames per step (the metric)
    real_frames = world * sum(int(host_batches[i % n_batches]["src_length"].sum()) for i in range(args.steps)) / args.steps
    value = frames / (ms_step * 1e-3)
    fl = sum(flops_per_step(b_, t_, l_, V, WL["d"], WL["H"], WL["ffn"]) for (t_, b_, l_) in step_shapes) / args.steps
    ach = fl / (ms_step * 1e-3) / 1e12
    clocks = sampler.summary()
    line = {
        "metric": "audio_frames_per_sec_fwd_bwd", "value": value, "unit": "frames/s", "n_gpus": world, "steps": args.steps,
        "warmup": max(3, args.warmup), "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": {"fp16": "fp16 (mixed_float16: fp16 operands/activations, fp32 accumulate + master weights, dynamic loss scale)",
                  "bf16": "bf16", "fp32": "f32"}[args.dtype], "data": "synthetic",
        "config": {"workload": "%s: %s (conv2d subsample + 12enc/6dec, d=%d) synthetic fbank %s per GPU, V=8192, dropout 0.1, "
                               "label_smoothing 0.1, Adam+noam" % (args.workload, WL["hparams"], WL["d"],
                                                                   "[%d,%d,80] L=%d" % (B, T, L) if not WL.get("ragged") else
                                                                   "length buckets %s (T,B,L), src_length~U(0.6T,T)" % (shapes,)),
                   "global_batch_frames": frames, "real_frames_per_sec": real_frames / (ms_step * 1e-3), "parallelism": "dp%d" % world, "cuda_graph": not args.no_graph, "kernels_per_step": int(launches_per_step),
                   "l2_policy": "inputs+activations per step (~4 GB) exceed the 50 MB L2; 4 rotating input batches",
                   "loss_last_step": loss_val,
                   "loss_scale_state": (dict(zip(("scale", "finite_steps_in_a_row", "last_step_skipped", "skipped_steps", "applied_steps",
                                                  "global_grad_norm"), [float(x) for x in trainer.rt.loss_scale_state[:6].tolist()]))
                                        if getattr(trainer.rt, "loss_scale_state", None) is not None else None)},
        "clocks": clocks,
        "e2e": {"value": frames / (ms_e2e / args.steps * 1e-3), "unit": "frames/s", "h2d_bytes_per_step": h2d,
                "d2h_bytes_per_step": 4, "ms_per_step": ms_e2e / args.steps},
        "gpu_launches": int(launches_per_step * args.steps),
    }
    # roofline of the GEMM kernel family (tc_gemm_kernel / tc_wgrad_group_kernel): algorithmic FLOPs of those launches / their
    # durations: the GEMMs of one eagerly launched step are recorded and each is replayed back to back inside the library
    # with CUDA events around the repetitions (a graph replay cannot be bracketed per kernel).  DRAM traffic is not measured.
    step_rf = {"achieved": ach, "frac": ach / peaks["tflops_sustained"],
               "algorithmic_flops_per_step": fl, "mflop_per_frame": fl / (frames / world) / 1e6,
               "note": "all kernels of the step / step time"}
    if gemm and gemm["ms"] > 0:
        g_tf = gemm["flops"] / (gemm["ms"] * 1e-3) / 1e12
        line["roofline"] = {"bound": "tensor", "kernel": "tc_gemm_kernel (all instantiations) + tc_wgrad_group_kernel (wgmma GEMMs outside the fused FFN / attention kernels)", "achieved": g_tf,
                            "peak": peaks["tflops_sustained"], "unit": "TFLOP/s", "frac": g_tf / peaks["tflops_sustained"],
                            "traffic": None, "peak_source": peaks["source"], "launches_per_step": gemm["launches"],
                            "avg_launch_us": gemm["ms"] * 1e3 / max(1, gemm["launches"]),
                            "algorithmic_flops_per_launch": gemm["flops"] / max(1, gemm["launches"]),
                            "share_of_step": gemm["ms"] / ms_step,
                            "share_note": "sum of the per-launch GEMM durations (each GEMM of one step replayed back to back, "
                                          "CUDA events, no host gaps) / timed step",
                            "step": step_rf}
    else:
        line["roofline"] = {"bound": "tensor", "kernel": "whole step", "achieved": ach, "peak": peaks["tflops_sustained"],
                            "unit": "TFLOP/s", "frac": ach / peaks["tflops_sustained"], "traffic": None,
                            "peak_source": peaks["source"], "step": step_rf}
    if enc_block:
        line["roofline"]["encoder_block"] = enc_block
    if cpu:
        line["cpu_baseline"] = cpu
    print(json.dumps(line), flush=True)
    leave(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10, help="timed training steps (the decode workload always decodes its 200 tokens)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--dump-outputs", default="", metavar="DIR",
                    help="training workloads only: after the timed steps write their losses and a seeded sample of the updated "
                         "parameters to DIR/*.npy; split-K and FFN-slice reductions use fp32 atomics, so two runs agree to rounding, "
                         "not bit for bit")
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--cpu-worker", default="", help=argparse.SUPPRESS)
    ap.add_argument("--cpu-ref-worker", default="", help=argparse.SUPPRESS)
    ap.add_argument("--no-graph", action="store_true", help="launch every kernel eagerly instead of replaying the CUDA graph")
    ap.add_argument("--dtype", default="fp16", choices=["fp16", "bf16", "fp32"],
                    help="fp16 = the reference's mixed_float16 (default: logits within 3.2e-3 of the fp64 oracle); bf16; fp32 parity mode")
    ap.add_argument("--workload", default="cfg2", choices=sorted(WORKLOADS) + ["decode"],
                    help="cfg2 = BASELINE headline [32,1000,80]; cfg3 / cfg3w = [8|64,1500,80]; cfg4 = speech_transformer_m ragged buckets; "
                         "decode = cfg-5 greedy decode")
    args = ap.parse_args()
    if args.dump_outputs and (args.impl == "reference" or args.workload == "decode"):
        ap.error("--dump-outputs is implemented for the training workloads of the CUDA path only")
    if args.cpu_ref_worker:
        cpu_ref_worker(args.cpu_ref_worker)
        return
    if args.cpu_worker:
        cpu_worker(args.cpu_worker)
        return
    if args.impl == "reference":
        run_reference(args)
        return
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.gpus > 1 and world == 1:
        # convenience: re-launch under torchrun when invoked directly with --gpus N
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(args.gpus),
               "--master-addr", "127.0.0.1", "--master-port", os.environ.get("MASTER_PORT", "29533"), __file__,
               "--gpus", str(args.gpus), "--steps", str(args.steps), "--warmup", str(args.warmup)]
        cmd += ["--dtype", args.dtype, "--workload", args.workload]
        if args.no_cpu_baseline:
            cmd.append("--no-cpu-baseline")
        if args.dump_outputs:
            cmd += ["--dump-outputs", args.dump_outputs]
        sys.exit(subprocess.call(cmd))
    if args.workload == "decode":
        run_decode(args)
        return
    run_gpu(args)


if __name__ == "__main__":
    main()
