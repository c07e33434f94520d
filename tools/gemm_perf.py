"""C-level timing (no Python overhead) of the wgmma GEMM at the model's shapes and epilogues, with the tile configuration
the library picks. Results -> bench_out/gemm_perf.json"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa
from neurst_b200 import lib  # noqa

dev = "cuda"
res = {}


def rnd(*s):
    return torch.randn(*s, device=dev).to(torch.bfloat16)


def run(tag, M, N, K, out_dtype=torch.bfloat16, a_mn=False, b_mn=False, **kw):
    A = rnd(K, M) if a_mn else rnd(M, K)
    B = rnd(K, N) if b_mn else rnd(N, K)
    Cc = torch.zeros(M, N, device=dev, dtype=out_dtype)
    ms = lib.gemm_bench(A, B, Cc, iters=50, a_mn=a_mn, b_mn=b_mn, **kw)
    r = dict(ms=ms, tflops=2.0 * M * N * K / ms / 1e9)
    res[tag] = r
    print("%-40s %8.1f us %8.1f TF" % (tag, ms * 1e3, r["tflops"]), flush=True)


# FFN1 [M, 256] x [256, 2048] and its epilogues
for M in (8000, 8192):
    run("ffn1 M=%d" % M, M, 2048, 256)
    run("ffn1 b_mn M=%d" % M, M, 2048, 256, b_mn=True)
bias = torch.randn(2048, device=dev)
run("ffn1 bias", 8000, 2048, 256, b_mn=True, bias=bias)
run("ffn1 bias relu", 8000, 2048, 256, b_mn=True, bias=bias, relu=True)
run("ffn1 bias relu drop(philox)", 8000, 2048, 256, b_mn=True, bias=bias, relu=True, dropout=(0.1, 1, 2))
run("ffn1 mask", 8000, 2048, 256, mask_src=rnd(8000, 2048))
run("ffn1 f32 out", 8000, 2048, 256, out_dtype=torch.float32)
run("ffn1 f32 out + residual", 8000, 2048, 256, out_dtype=torch.float32, residual=torch.randn(8000, 2048, device=dev))
# FFN2, attention projections
bias2, res2 = torch.randn(256, device=dev), torch.randn(8000, 256, device=dev)
run("ffn2 M=8192", 8192, 256, 2048)
run("ffn2 M=8000", 8000, 256, 2048)
run("ffn2 f32 bias res", 8000, 256, 2048, out_dtype=torch.float32, bias=bias2, residual=res2, b_mn=True)
run("qkv", 8192, 768, 256)
run("qkv b_mn", 8192, 768, 256, b_mn=True)
run("qkv bias", 8000, 768, 256, b_mn=True, bias=torch.randn(768, device=dev))
run("out-proj M=8192", 8192, 256, 256)
run("out-proj M=8000", 8000, 256, 256)
run("out-proj f32 bias res", 8000, 256, 256, out_dtype=torch.float32, bias=bias2, residual=res2, b_mn=True)
# front-end, output layer, large squares
run("conv2 M=160000", 160000, 256, 2304)
run("dense M=8000 K=5120", 8000, 256, 5120)
run("logits f32 out", 2816, 8192, 256, out_dtype=torch.float32)
run("big 8192", 8192, 8192, 8192)
run("big 4096", 4096, 4096, 4096)
# weight gradients (MN-major operands, fp32 accumulate): split-K picked by the library, then fixed factors
wg = dict(out_dtype=torch.float32, a_mn=True, b_mn=True, accumulate=True)
run("wgrad ffn 256x2048xK8000 auto", 256, 2048, 8000, splitk=0, **wg)
for sk in (1, 2, 4, 8, 16):
    run("wgrad ffn 256x2048xK8000 splitk=%d" % sk, 256, 2048, 8000, splitk=sk, **wg)
for sk in (1, 4, 8, 13, 26):
    run("wgrad qkv 256x768xK8000 splitk=%d" % sk, 256, 768, 8000, splitk=sk, **wg)
run("wgrad conv2 2304x256xK160000 auto", 2304, 256, 160000, splitk=0, **wg)
os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
json.dump(res, open(os.path.join(ROOT, "bench_out", "gemm_perf.json"), "w"), indent=1)
