#!/usr/bin/env python
"""Per-kernel timeline of one captured training step of the single-GPU engine (torch.profiler / CUPTI; Nsight is not
needed).  Same workload as bench.py's headline: XSimGCL at yelp2018 shape, resident batches, CUDA-graph replay.

    python tools/step_trace.py [--steps 20] [--out DIR]

Prints the step time (CUDA events over 500 graph replays, profiler off), then for one profiled step a table of its GPU
operations in stream order: name, duration, start offset from the step's first operation, stream and the gap to the
previous operation on the same stream.  The summary line gives the kernel count, the summed kernel time of the main
stream and the step time minus that sum (launch gaps and grid drains; the side stream's BPR kernels overlap InfoNCE).
Durations are the medians over the profiled steps.  --out DIR also writes the table as DIR/step_trace.json.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def short(name):
    name = name.split("(")[0]
    for p in ("void srb::", "srb::", "void "):
        name = name.replace(p, "")
    return name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="profiled graph replays")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import random

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from selfrec_b200 import _lib, build
    from selfrec_b200.engine import TrainEngine

    build.build()
    _lib.require_device()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = bench.CFG
    data = bench.build_data()
    random.seed(1234)
    torch.manual_seed(1234)
    eng = TrainEngine("XSimGCL", data, cfg["d"], cfg["L"], cfg["B"], cfg["lr"], cfg["reg"], device=dev, philox_seed=2026,
                      **bench.xs_kwargs())
    P = 16
    pool = torch.from_numpy(np.stack([w.copy() for _, w in zip(range(P), eng.batches())])).to(dev)
    eng.batch_dev.copy_(pool[0])
    torch.cuda.synchronize()
    l0 = _lib.launch_count()
    eng.step_resident()
    torch.cuda.synchronize()
    launches = _lib.launch_count() - l0
    graph = eng.capture()

    def step(k):
        eng.batch_dev.copy_(pool[k % P], non_blocking=True)
        graph.replay()

    for k in range(20):
        step(k)
    torch.cuda.synchronize()
    R = 500
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(R):
        step(k)
    e1.record()
    torch.cuda.synchronize()
    step_us = e0.elapsed_time(e1) * 1e3 / R

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(args.steps):
            step(k)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as fh:
            trace = json.load(fh)
    ops = [e for e in trace["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    ops.sort(key=lambda e: float(e["ts"]))
    if not ops or len(ops) % args.steps:
        raise SystemExit(f"step_trace: {len(ops)} GPU operations for {args.steps} steps; cannot split them into steps")
    per = len(ops) // args.steps
    streams = [e["args"].get("stream") for e in ops[:per] if e["cat"] == "kernel"]
    main_stream = max(set(streams), key=streams.count)  # the one that carries most of the step's kernels
    # the side stream's kernels interleave with the main stream's differently from step to step: an operation is
    # identified by (stream, name, occurrence) and timed against the previous operation of its own stream
    per_step = []
    for k in range(args.steps):
        s = ops[k * per:(k + 1) * per]
        t0 = float(s[0]["ts"])
        seen, last_end, rec = {}, {}, {}
        for e in s:
            sid, name = e["args"].get("stream"), short(e["name"]) if e["cat"] == "kernel" else e["cat"]
            n = seen[(sid, name)] = seen.get((sid, name), 0) + 1
            ts, dur = float(e["ts"]), float(e["dur"])
            rec[(sid == main_stream, name, n)] = (dur, ts - t0, ts - last_end[sid] if sid in last_end else 0.0, e["cat"])
            last_end[sid] = max(last_end.get(sid, 0.0), ts + dur)
        per_step.append(rec)
    if any(set(r) != set(per_step[0]) for r in per_step):
        raise SystemExit("step_trace: the profiled steps do not run the same sequence")
    rows = []
    for key in per_step[0]:
        vals = [r[key] for r in per_step]
        rows.append({"name": key[1], "kind": vals[0][3], "stream": "main" if key[0] else "side",
                     "us": statistics.median(v[0] for v in vals), "start_us": statistics.median(v[1] for v in vals),
                     "gap_us": statistics.median(v[2] for v in vals)})
    rows.sort(key=lambda r: r["start_us"])
    kern = [r for r in rows if r["kind"] == "kernel"]
    main_k = [r for r in kern if r["stream"] == "main"]
    main_ops = [r for r in rows if r["stream"] == "main"]
    summary = {"gpu": torch.cuda.get_device_name(dev), "step_us": step_us, "launches_per_step": launches,
               "kernels_per_step": len(kern), "memsets_per_step": sum(r["kind"] == "gpu_memset" for r in rows),
               "main_kernel_us": sum(r["us"] for r in main_k), "side_kernel_us": sum(r["us"] for r in kern if r["stream"] == "side"),
               "main_gap_us": sum(r["gap_us"] for r in main_ops[1:])}
    summary["step_minus_main_kernels_us"] = step_us - summary["main_kernel_us"]
    print(f"{'start':>8} {'us':>8} {'gap':>7}  stream  name")
    for r in rows:
        print(f"{r['start_us']:8.1f} {r['us']:8.1f} {r['gap_us']:7.1f}  {r['stream']:6}  {r['name'] if r['kind'] == 'kernel' else r['kind']}")
    print(json.dumps(summary))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "step_trace.json"), "w") as fh:
            json.dump({"summary": summary, "ops": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
