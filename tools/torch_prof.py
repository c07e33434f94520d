"""Kernel-time breakdown of one eager training step (cfg-2) with torch.profiler (CUPTI), aggregated by kernel.

Usage: python tools/torch_prof.py [--dtype fp16|bf16|fp32]   (default fp16, the precision bench.py times)"""
import argparse, collections, os, re, sys
os.environ.setdefault("B200ST_NO_PDL", "1")   # with PDL a dependent kernel's duration includes its wait on the predecessor
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from torch.profiler import profile, ProfilerActivity
from neurst_b200.trainer import build_speech_transformer_trainer, synthetic_batch
ap = argparse.ArgumentParser()
ap.add_argument("--dtype", default="fp16", choices=["fp16", "bf16", "fp32"])
args = ap.parse_args()
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
    if "attn_" in k or "cast_rows" in k:
        print(k, " ".join("%.1f" % t for t in seq[k]))
