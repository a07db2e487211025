"""Where the local BA's time goes inside bench.py's device-resident step, serial vs pipelined.

  python tools/ba_step_trace.py [--steps N] [--warmup W] [--out DIR]

Runs the bench's step (extract + match on the tracking context, reset + solve of the 50-keyframe window) N times in serial mode
(everything on the tracking stream) and N times pipelined (the solve on a high-priority mapping context driven from a second host
thread, ordered after match(k)), each under torch.profiler with CUDA activities.  Writes both traces to DIR and prints, per mode:
for every kernel of the BA's LM loop its mean duration, the mean idle gap before it on its stream (negative: a programmatic
dependent launch started it while its predecessor ran) and the mean time from its predecessor's end to its own end (what the
kernel adds to the stream), and the mean span of a solve's LM loop (first LM kernel start to the end of its last).  The card's name and power limit are printed first.
"""
from __future__ import annotations

import argparse
import json
import os
import queue
import subprocess
import sys
import tempfile
import threading
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

W, H, NKP = 1920, 1080, 2000
RING = 8
# the kernels of one solve's LM loop, in either form (the launch chain or the single cluster launch); the last one of a solve
LM_KERNELS = ("ba_linearize_kernel", "ba_schur_blocks_kernel", "ba_pcg_sparse_kernel", "ba_backsub_commit_kernel",
              "ba_install_pending_kernel", "ba_local_fused_kernel")
LM_LAST = ("ba_install_pending_kernel", "ba_local_fused_kernel")


def short(name: str) -> str:
    """'void (anonymous namespace)::k<1, 2>(args)' -> 'k<1, 2>'"""
    head = name.replace("(anonymous namespace)::", "").split("(")[0]
    return head[5:] if head.startswith("void ") else head


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:  # the trace stands without it
        return f"nvidia-smi unavailable: {e!r}"


def analyse(trace_path: str):
    ev = json.load(open(trace_path))["traceEvents"]
    kern = [e for e in ev if e.get("cat") == "kernel" and "ts" in e]
    by_stream = defaultdict(list)
    for e in kern:
        by_stream[e["args"].get("stream")].append(e)
    per = defaultdict(lambda: {"n": 0, "dur": 0.0, "gap": 0.0, "end": 0.0})
    spans = []
    for s, ks in by_stream.items():
        ks.sort(key=lambda e: e["ts"])
        prev_end = None
        solve_start = None
        for e in ks:
            name = short(e["name"])
            base = name.split("<")[0]
            if base in LM_KERNELS:
                p = per[name]
                p["n"] += 1
                p["dur"] += e["dur"]
                p["gap"] += (e["ts"] - prev_end) if prev_end is not None else 0.0
                p["end"] += (e["ts"] + e["dur"] - prev_end) if prev_end is not None else e["dur"]
                if solve_start is None:
                    solve_start = e["ts"]
                if base in LM_LAST:
                    spans.append(e["ts"] + e["dur"] - solve_start)
                    solve_start = None
            prev_end = e["ts"] + e["dur"]
    table = {k: {"count": v["n"], "mean_us": v["dur"] / v["n"], "mean_gap_before_us": v["gap"] / v["n"],
                 "mean_end_to_end_us": v["end"] / v["n"]} for k, v in per.items()}
    return table, (float(np.mean(spans)) if spans else None), len(spans)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "ba_step_trace"))
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from gslam_b200 import synth
    from gslam_b200.api import BAGraph, Context, Features, OptimzeConfig
    os.makedirs(args.out, exist_ok=True)
    print("card:", card(), flush=True)
    ctx = Context(0)
    ctx_m = Context(0, high_priority=True)
    cfg = ctx.orb_cfg(nfeatures=NKP)
    ba_cfg = OptimzeConfig(maxIterations=10, functionTolerance=0.0, pcgMaxIterations=50, pcgTolerance=1e-10)
    pb = synth.synth_ba(50, 2000, 5, seed=42, n_fixed=2)
    base = synth.synth_stream(W, H, RING, seed=7)
    ring = torch.from_numpy(base).cuda()
    feats = [Features(ctx, 2 * NKP + 256), Features(ctx, 2 * NKP + 256)]
    graph_s, graph_p = BAGraph(ctx, pb), BAGraph(ctx_m, pb)
    feats[1].extract(ring[RING - 1].data_ptr(), W, H, cfg, device_ptr=True, pitch=W)

    def track(k):
        f, fp = feats[k & 1], feats[(k + 1) & 1]
        f.extract(ring[k % RING].data_ptr(), W, H, cfg, device_ptr=True, pitch=W)
        f.match(fp)

    def serial(n):
        for k in range(n):
            track(k)
            graph_s.reset(); graph_s.solve(ba_cfg)

    def pipelined(n):
        qq: queue.Queue = queue.Queue(maxsize=2)

        def mapper():
            while qq.get() is not None:
                graph_p.reset(); graph_p.solve(ba_cfg)
        th = threading.Thread(target=mapper)
        th.start()
        for k in range(n):
            track(k)
            ctx_m.wait_for(ctx)
            qq.put(k)
        qq.put(None)
        th.join()
        ctx.wait_for(ctx_m)

    report = {"card": card()}
    for mode, run in (("serial", serial), ("pipelined", pipelined)):
        run(args.warmup)
        torch.cuda.synchronize()
        l0 = ctx.launch_count() + ctx_m.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run(args.steps)
            torch.cuda.synchronize()
        launches = ctx.launch_count() + ctx_m.launch_count() - l0
        path = os.path.join(args.out, f"{mode}.pt.trace.json")
        prof.export_chrome_trace(path)
        table, span, nsolves = analyse(path)
        report[mode] = {"lm_kernels": table, "solve_lm_span_us": span, "solves": nsolves, "launches_per_step": launches / args.steps}
        print(f"\n== {mode}: {nsolves} solves, LM-loop span {span:.1f} us per solve, {launches / args.steps:.1f} launches per step")
        print(f"{'kernel':40s} {'count':>6s} {'mean us':>9s} {'gap before us':>14s} {'end-to-end us':>14s}")
        for k, v in sorted(table.items(), key=lambda kv: -kv[1]["mean_end_to_end_us"] * kv[1]["count"]):
            print(f"{k:40s} {v['count']:6d} {v['mean_us']:9.2f} {v['mean_gap_before_us']:14.2f} {v['mean_end_to_end_us']:14.2f}")
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump(report, f, indent=1)
    ctx_m.close(); ctx.close()


if __name__ == "__main__":
    main()
