"""Per-launch wgmma GEMM timing of one training step (cfg-2) -> bench_out/gemm_step.csv + aggregated summary."""
import collections, csv, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
os.environ["B200ST_PROFILE_CSV"] = os.path.join(ROOT, "bench_out", "gemm_step.csv")
import torch
from neurst_b200 import lib
from neurst_b200.trainer import build_speech_transformer_trainer, synthetic_batch
tr, _ = build_speech_transformer_trainer("speech_transformer_s", 8192, precision="bf16", label_smoothing=0.1)
b = synthetic_batch(32, 1000, 88, 8192, device="cuda")
for i in range(3):
    tr.train_step(b, seed=i + 1)
torch.cuda.synchronize()
lib.profile_begin()
tr.train_step(b, seed=9)
torch.cuda.synchronize()
print(lib.profile_end())
agg = collections.OrderedDict()
for r in csv.DictReader(open(os.environ["B200ST_PROFILE_CSV"])):
    k = (r["M"], r["N"], r["K"], r["batch"], r["bn"], r["splitk"], r["a_mn"], r["b_mn"], r["epi"])
    a = agg.setdefault(k, [0, 0.0, 0.0])
    a[0] += 1; a[1] += float(r["us"]); a[2] = float(r["tflops"])
print("%8s %6s %7s %5s %4s %3s %2s %2s %3s | %4s %9s %8s %7s" % ("M", "N", "K", "batch", "bn", "sk", "aM", "bM", "epi", "n", "total_us", "avg_us", "TF"))
for k, (n, us, tf) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print("%8s %6s %7s %5s %4s %3s %2s %2s %3s | %4d %9.1f %8.1f %7.1f" % (k + (n, us, us / n, tf)))
