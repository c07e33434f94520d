"""C-level timing (no Python overhead) of the wgmma GEMM at the model's shapes. Results -> bench_out/gemm_perf.json"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa
from neurst_b200 import lib  # noqa

L = lib.load()
dev = "cuda"
res = {}


def rnd(*s):
    return torch.randn(*s, device=dev).to(torch.bfloat16)


def run(tag, M, N, K, out_dtype=torch.bfloat16, bn=0, stages=0, a_mn=False, b_mn=False, **kw):
    L.b200st_debug_tc(bn, stages, 0)
    A = rnd(K, M) if a_mn else rnd(M, K)
    B = rnd(K, N) if b_mn else rnd(N, K)
    Cc = torch.zeros(M, N, device=dev, dtype=out_dtype)
    ms = lib.gemm_bench(A, B, Cc, iters=30, a_mn=a_mn, b_mn=b_mn, **kw)
    r = dict(ms=ms, tflops=2.0 * M * N * K / ms / 1e9)
    res[tag] = r
    print(tag, r, flush=True)


for bn in (0, 64, 128, 256):
    run("ffn1_M8192_N2048_K256_bn%d" % bn, 8192, 2048, 256, bn=bn)
run("ffn1_f32out", 8192, 2048, 256, out_dtype=torch.float32)
for st in (2, 4):
    run("ffn1_bn128_stages%d" % st, 8192, 2048, 256, bn=128, stages=st)
for bn in (0, 128, 256):
    run("ffn2_M8192_N256_K2048_bn%d" % bn, 8192, 256, 2048, bn=bn)
run("qkv_M8192_N768_K256", 8192, 768, 256)
run("qkv_bmn", 8192, 768, 256, b_mn=True)
run("out_M8192_N256_K256", 8192, 256, 256)
for bn in (0, 128, 256):
    run("conv2_M160000_N256_K2304_bn%d" % bn, 160000, 256, 2304, bn=bn)
run("dense_M8000_N256_K5120", 8000, 256, 5120)
run("logits_M2816_N8192_K256", 2816, 8192, 256, out_dtype=torch.float32)
run("big_8192", 8192, 8192, 8192)
run("big_4096", 4096, 4096, 4096)
# wgrad forms (split-K, fp32 accumulate)
run("wgrad_ffn_K8000", 256, 2048, 8000, out_dtype=torch.float32, a_mn=True, b_mn=True, accumulate=True, splitk=0)
run("wgrad_conv2_K160000", 2304, 256, 160000, out_dtype=torch.float32, a_mn=True, b_mn=True, accumulate=True, splitk=0)
os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
json.dump(res, open(os.path.join(ROOT, "bench_out", "gemm_perf.json"), "w"), indent=1)
