"""Speech front-end launches of the cfg-2 training step (speech_transformer_s, B = 32, T = 1000, F = 80, fp16), one by one.

Per launch: the average time over the eager steps of a torch.profiler run of its own, the bytes the launch must move at
least (each operand read once, each output written once, from the shapes) and the resulting GB/s.  The launches are found
by kernel name and by their place in the step:
  conv1 forward        conv1_fwd_c256_kernel
  im2col               im2col_row_kernel (explicit front-end only)
  conv2 forward        the first GEMM (tc_gemm_kernel / tc_gemm_conv_kernel) after conv1's forward on its stream
  conv2 data gradient  the GEMM launches right before conv1's backward on its stream (1 implicit launch over the four
                       parity classes, or 1 explicit)
  conv2 filter grad.   the last tc_wgrad_group_kernel or MN-major x MN-major tc_gemm_kernel on the side stream before
                       conv1's backward
  conv1 backward       conv1_bwd_xhat_c256_kernel
  conv1 filter grad.   the first GEMM after conv1's backward on its stream (explicit front-end only)
Also the front-end backward span: from the start of the last LayerNorm backward (LN2's) before conv1's backward on its
stream to the end of conv1's backward — the stretch of the step's critical path the lines above share.
With --compare DIR, also the whole step: bench.py in this tree and in DIR (another checkout, built), alternated --rounds
times per workload, median and range of ms_per_step.  Prints the card's name, power limit and clocks; writes
bench_out/front_bench.json.  Run from the repository root on a machine with an H100."""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, T, F, L, V, C = 32, 1000, 80, 88, 8192, 256


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {}


def launch_bytes(implicit):
    """Least bytes each front-end launch moves at cfg-2 in fp16 (e = 2 bytes per activation)."""
    e = 2
    T1, F1 = (T + 1) // 2, (F + 1) // 2
    T2, F2 = (T1 + 1) // 2, (F1 + 1) // 2
    R1, R2, P = B * T1 * F1, B * T2 * F2, 4 * B * T2 * F2
    tu = 128 // F2
    tiles = 4 * B * -(-T2 // tu) * 128 * C * e           # class-major tiles of the implicit data gradient
    src, xhat, rstd, W2 = B * T * F * 4, R1 * C * e, R1 * 4, 9 * C * C * e
    a_conv2 = P * C * e if implicit else R2 * 9 * C * e  # parity-class planes, or the column matrix
    out = {
        "conv1 forward": src + xhat + rstd + (P * C * e if implicit else 0),
        "conv2 forward": a_conv2 + W2 + R2 * C * e,
        "conv2 data gradient": R2 * C * e + W2 + (tiles if implicit else R2 * 9 * C * e),
        "conv2 filter gradient": a_conv2 + R2 * C * e + 9 * C * C * 4,
        "conv1 backward": src + xhat + rstd + (tiles if implicit else R2 * 9 * C * e + R1 * C * e + R1 * 16 * e),
    }
    if not implicit:
        out["im2col"] = xhat + R2 * 9 * C * e
        out["conv1 filter gradient"] = R1 * 16 * e + R1 * C * e
    return out


def profile(steps, out_dir, graph=False, keep=False):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    from neurst_b200.trainer import build_speech_transformer_trainer, synthetic_batch
    tr, _ = build_speech_transformer_trainer("speech_transformer_s", V, precision="fp16", label_smoothing=0.1, use_cuda_graph=graph)
    batch = synthetic_batch(B, T, L, V, device="cuda")
    for i in range(3):
        tr.train_step(batch, seed=i + 1)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(steps):
            tr.train_step(batch, seed=100 + i)
        torch.cuda.synchronize()
    path = os.path.join(out_dir, "front_bench.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    if not keep:
        os.remove(path)
    ev.sort(key=lambda e: e["ts"])
    return ev


def classify(ev):
    """{launch: [durations in us]} from the kernel events of the profiled steps (sorted by start)."""
    gemm = lambda e: "tc_gemm_kernel" in e["name"] or "tc_gemm_conv_kernel" in e["name"]
    stream = lambda e: e["args"].get("stream")
    out = {}
    add = lambda k, e: out.setdefault(k, []).append(e["dur"])
    for i, e in enumerate(ev):
        n = e["name"]
        if "conv1_fwd_c256_kernel" in n:
            add("conv1 forward", e)
            nxt = next((x for x in ev[i + 1:] if gemm(x) and stream(x) == stream(e)), None)
            if nxt:
                add("conv2 forward", nxt)
        elif "im2col_row_kernel" in n:
            add("im2col", e)
        elif "conv1_bwd_xhat_c256_kernel" in n:
            add("conv1 backward", e)
            ln2 = next((x for x in reversed(ev[:i]) if stream(x) == stream(e) and re.search(r"\bln_bwd(_vec)?_kernel", x["name"])), None)
            if ln2:
                out.setdefault("front-end backward span", []).append(e["ts"] + e["dur"] - ln2["ts"])
            j, dg = i - 1, 0.0
            while j >= 0:
                if stream(ev[j]) == stream(e):
                    if not gemm(ev[j]):
                        break
                    dg += ev[j]["dur"]
                j -= 1
            out.setdefault("conv2 data gradient", []).append(dg)
            wg = [x for x in ev[:i] if stream(x) != stream(e) and
                  ("tc_wgrad_group_kernel" in x["name"] or re.search(r"tc_gemm_kernel<\d+, true, true", x["name"]))]
            if wg:
                add("conv2 filter gradient", wg[-1])
            nxt = next((x for x in ev[i + 1:] if stream(x) == stream(e)), None)
            if nxt is not None and gemm(nxt) and "im2col_row_kernel" in " ".join(x["name"] for x in ev):
                add("conv1 filter gradient", nxt)
    return out


def run_bench(tree, workload, steps, warmup):
    r = subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup), "--workload", workload,
                        "--no-cpu-baseline"], cwd=tree, capture_output=True, text=True)
    for line in reversed(r.stdout.splitlines()):
        if line.startswith("{") and "ms_per_step" in line:
            d = json.loads(line)
            return d["ms_per_step"], d.get("clocks")
    raise RuntimeError("bench.py in %s failed: %s" % (tree, r.stderr[-2000:]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="profiled eager steps")
    ap.add_argument("--compare", default="", metavar="DIR", help="another built checkout to compare whole steps against")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--workloads", default="cfg2")
    ap.add_argument("--bench-steps", type=int, default=50)
    ap.add_argument("--bench-warmup", type=int, default=5)
    ap.add_argument("--out", default="", help="output directory (default bench_out/)")
    ap.add_argument("--graph", action="store_true", help="profile CUDA-graph replays of the step instead of eager steps")
    ap.add_argument("--keep-trace", action="store_true", help="keep the chrome trace (front_bench.trace.json) in the output directory")
    args = ap.parse_args()
    out_dir = args.out or (os.path.join(ROOT, "bench_out") if os.access(ROOT, os.W_OK) else tempfile.mkdtemp())
    os.makedirs(out_dir, exist_ok=True)
    res = {"card": card()}
    print("card:", res["card"])

    ev = profile(args.steps, out_dir, args.graph, args.keep_trace)
    res["profiled_span_ms_per_step"] = (ev[-1]["ts"] + ev[-1]["dur"] - ev[0]["ts"]) / 1e3 / args.steps
    times = classify(ev)
    per_name = {}
    for e in ev:
        per_name[e["name"]] = per_name.get(e["name"], 0.0) + e["dur"] / args.steps
    res["kernels_us_per_step"] = per_name         # every kernel of the step, summed per name
    implicit = "im2col" not in times
    nbytes = launch_bytes(implicit)
    res["front_end"] = "implicit conv2 (parity-class planes)" if implicit else "explicit conv2 (column matrix)"
    res["launches"] = {}
    print("front-end: %s, %d profiled %s steps, %.3f ms per step from the first kernel's start to the last one's end" %
          (res["front_end"], args.steps, "graph" if args.graph else "eager", res["profiled_span_ms_per_step"]))
    print("%-24s %10s %10s %8s" % ("launch", "us", "MB", "GB/s"))
    for k in ("conv1 forward", "im2col", "conv2 forward", "conv2 filter gradient", "conv2 data gradient", "conv1 backward",
              "conv1 filter gradient"):
        if not times.get(k) or not sum(times[k]):
            continue
        us = statistics.mean(times[k])
        mb = nbytes[k] / 1e6
        res["launches"][k] = {"us": us, "bytes": nbytes[k], "GB/s": nbytes[k] / (us * 1e-6) / 1e9, "samples": len(times[k])}
        print("%-24s %10.1f %10.1f %8.0f" % (k, us, mb, res["launches"][k]["GB/s"]))
    if times.get("front-end backward span"):
        res["front_backward_span_us"] = statistics.mean(times["front-end backward span"])
        print("%-24s %10.1f   (LN2 backward start -> conv1 backward end, main stream)" % ("front-end bwd span", res["front_backward_span_us"]))

    if args.compare:
        res["step"] = {}
        for wl in args.workloads.split(","):
            mine, other = [], []
            for _ in range(args.rounds):
                other.append(run_bench(args.compare, wl, args.bench_steps, args.bench_warmup)[0])
                mine.append(run_bench(ROOT, wl, args.bench_steps, args.bench_warmup)[0])
            s = {"this": {"median": statistics.median(mine), "min": min(mine), "max": max(mine), "all": mine},
                 "compare": {"median": statistics.median(other), "min": min(other), "max": max(other), "all": other}}
            res["step"][wl] = s
            print("%s ms_per_step  this tree: median %.3f [%.3f, %.3f]   %s: median %.3f [%.3f, %.3f]" %
                  (wl, s["this"]["median"], s["this"]["min"], s["this"]["max"], args.compare, s["compare"]["median"],
                   s["compare"]["min"], s["compare"]["max"]))
    res["card_after"] = card()
    print("card after:", res["card_after"])
    with open(os.path.join(out_dir, "front_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
