#!/usr/bin/env python
"""bench_phases.py -- where the time of a boosting round goes on one H100: a per-kernel table.

    python bench_phases.py [--steps K] [--warmup W] [--rows N] [--cols F] [--depth D] [--out DIR]

Grows the C3 model of bench.py (same generator and parameters) and measures W warm-up rounds, then K rounds twice:
  1. `phase_ms_per_step`: the engine's per-phase CUDA-event timers (profile=2; this switches the per-tree CUDA graph
     off, so these rounds run with direct launches).
  2. a torch.profiler trace (CUDA activities) of K `Booster.update` calls as bench.py runs them (profile=1, the per-tree
     CUDA graph replayed).  From it: per kernel name the launches per round, the device time per round, the mean time
     per launch, and the device idle time between consecutive GPU activities (launch / dependency gaps).
Bytes per launch are what the algorithm has to move, computed from the shapes (kernel_bytes); "GB/s" is those bytes over
kernel time, algorithmic, not a measured DRAM figure.  Prints one JSON line; with --out, also writes the table as
markdown and the JSON into DIR.  Writes nothing into the tree unless DIR points there.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def kernel_bytes(name, n, F, depth):
    """Algorithmic bytes of one round's launches of a kernel (summed over the round), or None when not modelled.
    Rows move as: row id 4 B, bin byte 1 B, gradient pair 8 B (fp32 g,h), leaf index 2 B, margin 4 B.  A histogram
    node is n_groups * 32 slots * 256 bins * 16 B (int64 g,h; a group has 32 feature slots, padding included)."""
    node = ((F + 31) // 32) * 32 * 256 * 16
    splits = depth - 1                       # levels partitioned through the ordered row lists
    if "partition_kernel" in name:
        return n * splits * (4 + 1 + 4) if splits > 0 else None
    if "final_assign_kernel" in name:
        # final_assign_kernel<kCat, kRoot, kSums>: kSums = true also gathers the row's gradient pair
        gathers_gh = name.split("(", 1)[0].replace(" ", "").endswith(",true>")
        return n * (4 + 1 + 2) + (n * 8 if gathers_gh else 0)
    if "leaf_accumulate_kernel" in name:
        return n * (2 + 8)
    if "margin_update_kernel" in name:
        return n * (2 + 4 + 4)
    if "hist_subtract_kernel" in name:
        # levels 1..depth-1: 2^(d-1) sibling pairs read parent + built, write sibling
        return sum(3 * (1 << (d - 1)) * node for d in range(1, depth))
    if "quantize_kernel" in name:
        return n * (8 + 8)
    return None


def profile_table(prof_events, rounds, n, F, depth):
    kern = [e for e in prof_events if e["kind"] == "kernel"]
    rows = {}
    for e in kern:
        r = rows.setdefault(e["name"], {"launches": 0, "us": 0.0})
        r["launches"] += 1
        r["us"] += e["dur"]
    table = []
    for name, r in sorted(rows.items(), key=lambda kv: -kv[1]["us"]):
        b = kernel_bytes(name, n, F, depth)
        us = r["us"] / rounds
        table.append({"kernel": name, "launches_per_round": r["launches"] / rounds, "us_per_round": us,
                      "us_per_launch": r["us"] / r["launches"],
                      "alg_bytes_per_round": b, "alg_GBps": (b / (us * 1e-6) / 1e9) if (b and us > 0) else None})
    gpu = sorted((e for e in prof_events if e["kind"] in ("kernel", "memcpy", "memset")), key=lambda e: e["ts"])
    gaps, end = 0.0, None
    for e in gpu:
        if end is not None and e["ts"] > end:
            gaps += e["ts"] - end
        end = e["ts"] + e["dur"] if end is None else max(end, e["ts"] + e["dur"])
    other = {}
    for e in gpu:
        if e["kind"] != "kernel":
            o = other.setdefault(e["kind"], {"count": 0, "us": 0.0})
            o["count"] += 1
            o["us"] += e["dur"]
    span = (end - gpu[0]["ts"]) if gpu else 0.0
    return table, {"span_us_per_round": span / rounds, "idle_gap_us_per_round": gaps / rounds,
                   "kernel_us_per_round": sum(t["us_per_round"] for t in table),
                   "memcpy_memset": {k: {"per_round": v["count"] / rounds, "us_per_round": v["us"] / rounds} for k, v in other.items()}}


def trace_events(prof):
    out = []
    for e in prof.events():
        dt = getattr(e, "device_type", None)
        if dt is None or "CUDA" not in str(dt):
            continue
        name = e.name
        low = name.lower()
        kind = "memcpy" if "memcpy" in low else ("memset" if "memset" in low else "kernel")
        tr = e.time_range
        out.append({"name": name, "kind": kind, "ts": float(tr.start), "dur": float(tr.end - tr.start)})
    return out


def markdown(table, summary, meta):
    lines = ["%s, %s" % (meta["gpu"], meta["power_limit"]), "",
             "| kernel | launches / round | µs / round | µs / launch | alg. MB / round | alg. GB/s |",
             "|---|---:|---:|---:|---:|---:|"]
    for t in table:
        mb = "%.0f" % (t["alg_bytes_per_round"] / 1e6) if t["alg_bytes_per_round"] else "–"
        gb = "%.0f" % t["alg_GBps"] if t["alg_GBps"] else "–"
        lines.append("| `%s` | %.1f | %.1f | %.1f | %s | %s |" % (t["kernel"][:80], t["launches_per_round"], t["us_per_round"],
                                                                 t["us_per_launch"], mb, gb))
    lines.append("")
    lines.append("span %.0f µs / round, kernels %.0f µs, idle gaps %.0f µs; copies/memsets %s" % (
        summary["span_us_per_round"], summary["kernel_us_per_round"], summary["idle_gap_us_per_round"],
        json.dumps(summary["memcpy_memset"])))
    return "\n".join(lines)


def gpu_meta():
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": pl}
    except Exception:   # noqa: BLE001 -- the table is still useful without the card's name
        return {"gpu": "unknown", "power_limit": "unknown"}


def main():
    import bench
    import torch
    from xgboost_ray_b200 import engine as E

    w = bench.WORKLOADS["C3"]
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", type=int, default=w["rows"])
    ap.add_argument("--cols", type=int, default=w["cols"])
    ap.add_argument("--depth", type=int, default=w["depth"])
    ap.add_argument("--out", default=None, help="directory for phases.md / phases.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_phases.py measures on a CUDA device"

    X, y = bench.synth_shard(args.rows, args.cols, 0, 1, workload="C3")
    dm = E.DMatrix(X, label=y)
    dm._ensure_quantized(256)
    result = {"config": "C3 synthetic %dx%d reg:squarederror depth %d 256 bins" % (args.rows, args.cols, args.depth), **gpu_meta()}

    # 1. per-phase event timers (direct launches)
    bst = E.Booster(dict(bench.PARAMS, max_depth=args.depth, profile=2), cache=[dm])
    for r in range(args.warmup):
        bst.update(dm, r)
    bst.get_timers(reset=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for r in range(args.steps):
        bst.update(dm, args.warmup + r)
    torch.cuda.synchronize()
    wall2 = time.perf_counter() - t0
    tm = bst.get_timers(reset=True)
    result["profile2"] = {"ms_per_step": 1e3 * wall2 / args.steps,
                          "phase_ms_per_step": {k: v / args.steps for k, v in tm.get("phase_ms", {}).items()},
                          "round_ms_per_step": tm.get("round_ms", 0.0) / args.steps}
    del bst

    # 2. torch.profiler trace of the graph-replayed rounds bench.py times
    bst = E.Booster(dict(bench.PARAMS, max_depth=args.depth, profile=1), cache=[dm])
    for r in range(args.warmup):
        bst.update(dm, r)
    bst.get_timers(reset=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for r in range(args.steps):
        bst.update(dm, args.warmup + r)
    torch.cuda.synchronize()
    wall1 = time.perf_counter() - t0
    tm = bst.get_timers(reset=True)
    result["profile1"] = {"ms_per_step": 1e3 * wall1 / args.steps, "kernel_launches_per_step": tm["kernel_launches"] / args.steps}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        for r in range(args.steps):
            bst.update(dm, args.warmup + args.steps + r)
        torch.cuda.synchronize()
    table, summary = profile_table(trace_events(prof), args.steps, args.rows, args.cols, args.depth)
    result["kernels"] = table
    result["summary"] = summary
    print(json.dumps(result), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "phases.json"), "w") as f:
            json.dump(result, f, indent=1)
        with open(os.path.join(args.out, "phases.md"), "w") as f:
            f.write(markdown(table, summary, result) + "\n")


if __name__ == "__main__":
    main()
