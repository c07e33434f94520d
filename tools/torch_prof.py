"""Kernel-time breakdown of one eager training step (cfg-2) with torch.profiler (CUPTI), aggregated by kernel.

Usage: python tools/torch_prof.py [--dtype fp16|bf16|fp32]   (default fp16, the precision bench.py times)

Also prints the per-launch times of the attention and fused FFN kernels, and for the fused FFN the median time and rate
per direction and row count."""
import argparse, collections, json, os, re, subprocess, sys, tempfile
os.environ.setdefault("B200ST_NO_PDL", "1")   # with PDL a dependent kernel's duration includes its wait on the predecessor
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from torch.profiler import profile, ProfilerActivity
from neurst_b200.trainer import build_speech_transformer_trainer, synthetic_batch
ap = argparse.ArgumentParser()
ap.add_argument("--dtype", default="fp16", choices=["fp16", "bf16", "fp32"])
args = ap.parse_args()
# a kernel time belongs with the card and power limit it was measured at
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
print("device:", smi.stdout.strip() or torch.cuda.get_device_name(0))
tr, _ = build_speech_transformer_trainer("speech_transformer_s", 8192, precision=args.dtype, label_smoothing=0.1)
b = synthetic_batch(32, 1000, 88, 8192, device="cuda")
for i in range(3):
    tr.train_step(b, seed=i + 1)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    tr.train_step(b, seed=9)
    torch.cuda.synchronize()
agg = collections.defaultdict(lambda: [0, 0.0])
seq = collections.defaultdict(list)
tot = 0.0
for e in prof.events():
    if e.device_type is not None and "cuda" in str(e.device_type).lower():
        name = e.name.replace("(anonymous namespace)::", "")
        name = re.sub(r"\(.*", "", name)
        name = re.sub(r"^void ", "", name)
        agg[name[:80]][0] += 1
        seq[name[:80]].append(e.device_time if hasattr(e, 'device_time') else e.cuda_time)
        agg[name[:80]][1] += e.device_time if hasattr(e, "device_time") else e.cuda_time
        tot += e.device_time if hasattr(e, "device_time") else e.cuda_time
print("total kernel us", tot)
for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:28]:
    print("%-82s n=%5d total=%9.1f avg=%8.1f share=%.3f" % (k, n, t, t / n, t / tot))
for k in seq:
    if "attn_" in k or "cast_rows" in k or "fused_mlp" in k:
        print(k, " ".join("%.1f" % t for t in seq[k]))

# The fused FFN kernel runs under one name at the encoder's M = B*T/4 rows and the decoder's M = B*L rows; the trace's grid
# (m_tiles * splits CTAs) tells them apart.  Template argument 2 is the direction: MN-major weights (true) = forward,
# K-major (false) = backward.  4*M*d*ffn FLOP per launch.
with tempfile.TemporaryDirectory() as tmp:
    path = os.path.join(tmp, "trace.json")
    prof.export_chrome_trace(path)
    trace = json.load(open(path))
d, ffn = tr.rt.config.d, tr.rt.config.ffn
rows = {(M + 127) // 128: M for M in (32 * 1000 // 4, 32 * 88)}
mlp = collections.defaultdict(list)
for ev in trace.get("traceEvents", []):
    if ev.get("cat") == "kernel" and "fused_mlp_fwd_kernel" in ev.get("name", ""):
        grid = ev["args"]["grid"][0]
        M = next((m for mt, m in rows.items() if grid % mt == 0), 0)
        mlp[("forward" if ", true," in ev["name"] else "backward", M, grid)].append(ev["dur"])
for (direction, M, grid), ts in sorted(mlp.items(), key=lambda kv: (kv[0][0] != "forward", -kv[0][1])):
    ts = sorted(ts)
    med = ts[len(ts) // 2]
    print("fused_mlp %-8s M=%5d grid=%3d n=%2d median=%6.1f us min=%6.1f max=%6.1f  %.0f TFLOP/s  [%s]" %
          (direction, M, grid, len(ts), med, ts[0], ts[-1], 4.0 * M * d * ffn / (med * 1e-6) / 1e12, " ".join("%.1f" % t for t in ts)))
