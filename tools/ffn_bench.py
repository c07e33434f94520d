"""Fused FFN kernel alone (fused_mlp_fwd / fused_mlp_bwd) at the speech Transformer's shapes: time per launch, rate and
weight bytes, and a timeline of where each warpgroup's time goes inside the CTA.

Usage: python tools/ffn_bench.py [--iters 200] [--dtype fp16|bf16] [--shapes 8000,2816] [--d 256] [--ffn 2048]

The library's other objects come from the in-tree build (neurst_b200/csrc/build); tools/ffn_bench.cu, which includes
tc_gemm.cu, is compiled with the library's flags into bench_out/libffn_bench.so and, with -DB200ST_MLP_TIMELINE, into
bench_out/libffn_bench_tl.so.  Times come from CUDA events around `--iters` back-to-back launches (PDL off, as in
tools/torch_prof.py, so that a launch's time does not include its wait on the one before).  The timeline is one launch of
the stamped build, after warm-up: per warpgroup, the mean of each phase over the CTAs, per 64-column hidden half and for
the fixed parts (prologue, output tail).  Writes bench_out/ffn_bench.json."""
import argparse, ctypes, hashlib, json, os, subprocess, sys
os.environ.setdefault("B200ST_NO_PDL", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "bench_out")
SLOTS = 256          # kMlpTlSlots in tc_gemm.cu
PHASES = ["epilogue", "turn wait", "ring wait", "issue", "wgmma wait", "release"]


def build_libs():
    from neurst_b200.csrc import build as B
    B.build()
    objs = [os.path.join(B.OBJ, f[:-3] + ".o") for f in B._sources() if f != "tc_gemm.cu"]
    os.makedirs(OUT, exist_ok=True)
    digest = B._digest() + hashlib.sha256(open(os.path.join(ROOT, "tools", "ffn_bench.cu"), "rb").read()).hexdigest()
    libs = {}
    for name, extra in (("libffn_bench.so", []), ("libffn_bench_tl.so", ["-DB200ST_MLP_TIMELINE"])):
        obj = os.path.join(OUT, name[:-3] + ".o")
        lib = os.path.join(OUT, name)
        libs[name] = lib
        stamp = lib + ".digest"
        if os.path.exists(lib) and os.path.exists(stamp) and open(stamp).read() == digest:
            continue
        for cmd in ([B.NVCC] + B.FLAGS + extra + ["-c", os.path.join(ROOT, "tools", "ffn_bench.cu"), "-o", obj],
                    [B.NVCC, "-shared", "-o", lib, obj] + objs + ["-cudart", "static"]):
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise SystemExit("build failed: %s\n%s%s" % (" ".join(cmd), r.stdout, r.stderr))
        open(stamp, "w").write(digest)
    return libs


def bind(path):
    L = ctypes.CDLL(path)
    vp, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    L.ffnb_fwd.argtypes = [vp, i, i, i, i, vp, vp, vp, vp, f, vp, f, vp, vp, vp, vp, vp]
    L.ffnb_bwd.argtypes = [vp, i, i, i, i, vp, vp, vp, f, vp, vp, vp, vp]
    L.ffnb_grid.argtypes = [i, i]
    L.ffnb_set_timeline.argtypes = [vp]
    return L


def card():
    import torch
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip() or torch.cuda.get_device_name(0)


def make_case(M, d, ffn, dtype):
    import torch
    g = torch.Generator(device="cuda").manual_seed(M)
    t = torch.float16 if dtype == "fp16" else torch.bfloat16

    def packed_bits(n, keep=0.9):
        b = (torch.rand(n, generator=g, device="cuda") < keep).to(torch.int32).view(-1, 8)
        return (b << torch.arange(8, device="cuda", dtype=torch.int32)).sum(1).to(torch.uint8)
    return dict(
        X=torch.randn(M, d, generator=g, device="cuda").to(t), W1=(torch.randn(d, ffn, generator=g, device="cuda") * d ** -0.5).to(t),
        W2=(torch.randn(ffn, d, generator=g, device="cuda") * ffn ** -0.5).to(t), b1=torch.randn(ffn, generator=g, device="cuda") * 0.1,
        b2=torch.randn(d, generator=g, device="cuda") * 0.1, bits_ffn=packed_bits(M * ffn), bits_post=packed_bits(M * d),
        F1=torch.empty(M, ffn, device="cuda", dtype=t), out=torch.zeros(M, d, device="cuda"),
        dF1=torch.empty(M, ffn, device="cuda", dtype=t), dH=torch.zeros(M, d, device="cuda"))


def launcher(L, c, M, d, ffn, dtype, direction):
    import torch
    from neurst_b200 import lib as NL
    dt = NL.F16 if dtype == "fp16" else NL.BF16
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda x: ctypes.c_void_p(x.data_ptr())
    if direction == "forward":
        def run():
            if L.ffnb_fwd(p(c["X"]), dt, M, d, ffn, p(c["W1"]), p(c["b1"]), p(c["W2"]), p(c["b2"]), 0.1, p(c["bits_ffn"]), 0.1,
                          p(c["bits_post"]), p(c["F1"]), p(c["out"]), st, None):
                raise SystemExit("fused_mlp_fwd failed")
    else:
        def run():
            if L.ffnb_bwd(p(c["X"]), dt, M, d, ffn, p(c["W1"]), p(c["W2"]), p(c["F1"]), 1.0 / 0.9, p(c["dF1"]), p(c["dH"]), st, None):
                raise SystemExit("fused_mlp_bwd failed")
    return run


def time_us(run, iters):
    import torch
    for _ in range(10):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def timeline(L, run, grid, H, longest):
    """Mean time per phase (us) over the CTAs with the longest slice (H halves), per warpgroup: per hidden half (steps
    1 .. H - 1) and the fixed parts."""
    import torch
    buf = torch.zeros(grid * 2 * SLOTS, dtype=torch.int64, device="cuda")
    rc = L.ffnb_set_timeline(ctypes.c_void_p(buf.data_ptr()))
    if rc != 0:
        raise SystemExit("setting the timeline buffer failed (%d; 1: built without B200ST_MLP_TIMELINE)" % rc)
    for _ in range(4):           # every launch rewrites the same slots: the last one is read
        run()
    torch.cuda.synchronize()
    L.ffnb_set_timeline(None)
    t = buf.view(grid, 2, SLOTS).cpu().double()
    span = float(t[:, :, 6].max() - t[:, :, 0].min()) * 1e-3
    entry = float(t[:, 0, 0].max() - t[:, :, 0].min()) * 1e-3
    t = t[longest]
    ns_per_clk = (t[:, :, 6] - t[:, :, 0]).sum() / (t[:, :, 5] - t[:, :, 1]).sum()
    us = lambda clk: float(clk.mean()) * float(ns_per_clk) * 1e-3
    step = lambda s, e: t[:, :, 8 + 6 * s + e]
    res = {"sm_ghz": 1.0 / float(ns_per_clk)}
    for wg in range(2):
        sl = lambda x: x[:, wg]
        r = {}
        for e, name in enumerate(PHASES):
            acc = 0.0
            for s in range(1, H):
                nxt = step(s + 1, 0) if e == 5 else step(s, e + 1)
                acc += us(sl(nxt - step(s, e)))
            r[name] = acc / (H - 1)
        r["per half"] = us(sl(step(H, 0) - step(1, 0))) / (H - 1)
        r["prologue (entry to X arrived)"] = us(sl(t[:, :, 2] - t[:, :, 1]))
        r["step 0 (entry to wgmmas complete)"] = us(sl(step(0, 5) - t[:, :, 2]))
        r["last step (GEMM2 only)"] = us(sl(t[:, :, 3] - step(H, 0)))
        r["tail: staging in smem"] = us(sl(t[:, :, 4] - t[:, :, 3]))
        r["tail: ticket wait + bulk reductions"] = us(sl(t[:, :, 5] - t[:, :, 4]))
        r["CTA total"] = us(sl(t[:, :, 5] - t[:, :, 1]))
        res["wg%d" % wg] = r
    res["launch span (first entry to last exit)"] = span
    res["latest CTA entry"] = entry
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--dtype", default="fp16", choices=["fp16", "bf16"])
    ap.add_argument("--shapes", default="8000,2816", help="row counts M (encoder B*T/4 and decoder B*L at cfg-2)")
    ap.add_argument("--d", type=int, default=256)
    ap.add_argument("--ffn", type=int, default=2048)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("ffn_bench.py needs a CUDA device")
    libs = build_libs()
    Lp, Lt = bind(libs["libffn_bench.so"]), bind(libs["libffn_bench_tl.so"])
    dev = card()
    print("device:", dev)
    d, ffn = args.d, args.ffn
    report = dict(device=dev, dtype=args.dtype, d=d, ffn=ffn, iters=args.iters, pdl=False, cases=[])
    for M in [int(x) for x in args.shapes.split(",")]:
        c = make_case(M, d, ffn, args.dtype)
        grid = Lp.ffnb_grid(M, ffn)
        m_tiles = (M + 127) // 128
        splits, total = grid // m_tiles, ffn // 64
        H = -(-total // splits)                     # 64-column halves per slice (mlp_splits in tc_gemm.cu)
        longest = [i for i in range(grid) if total // splits + (i % splits < total % splits) == H]
        for direction in ("forward", "backward"):
            us = time_us(launcher(Lp, c, M, d, ffn, args.dtype, direction), args.iters)
            flop = 4.0 * M * d * ffn
            l2_bytes = m_tiles * 2 * d * ffn * 2       # every row tile streams both weight matrices once
            tl = timeline(Lt, launcher(Lt, c, M, d, ffn, args.dtype, direction), grid, H, longest)
            row = dict(direction=direction, M=M, ctas=grid, halves_per_cta=H, us=us, tflops=flop / us * 1e-6,
                       weight_bytes_l2_to_smem=l2_bytes, weight_tb_per_s=l2_bytes / us * 1e-6,
                       tensor_us_at_989=flop / 989e12 * 1e6, timeline=tl)
            report["cases"].append(row)
            print("%-8s M=%5d CTAs=%3d halves/CTA=%2d  %7.1f us  %6.1f TFLOP/s  weights L2->smem %.0f MB = %.2f TB/s  (tensor work at 989 TFLOP/s: %.1f us)"
                  % (direction, M, grid, H, us, row["tflops"], l2_bytes / 1e6, row["weight_tb_per_s"], row["tensor_us_at_989"]))
            for wg in (0, 1):
                r = tl["wg%d" % wg]
                print("   wg%d per half %.2f us: %s" % (wg, r["per half"], "  ".join("%s %.2f" % (k, r[k]) for k in PHASES)))
                print("       fixed: %s" % "  ".join("%s %.2f" % (k, v) for k, v in r.items() if k not in PHASES and k != "per half"))
            print("   launch span %.1f us (stamped build), latest CTA entry %.1f us, SM clock %.2f GHz"
                  % (tl["launch span (first entry to last exit)"], tl["latest CTA entry"], tl["sm_ghz"]))
    with open(os.path.join(OUT, "ffn_bench.json"), "w") as f:
        json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
