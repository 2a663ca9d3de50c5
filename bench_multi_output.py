#!/usr/bin/env python
"""bench_multi_output.py -- boosting rounds/sec of the C3 workload of bench.py with a label of T = 4 columns, one tree
per target and round against one vector-leaf tree per round (multi_strategy="multi_output_tree"), one GPU, and the time
of the vector split scan.

    python bench_multi_output.py --steps K --warmup W [--rows N] [--repeats R]

Same synthetic matrix (bench.py's generator, 10M x 100), parameters and depth as bench.py's C3 headline, quantised once
and resident in HBM, and the 4-column labels of bench_multi_target.py.  Three arms: reg:squarederror with
one_output_per_tree; reg:squarederror with multi_output_tree; binary:logistic with multi_output_tree.  The arms
alternate R times (W untimed rounds, then K timed rounds each time).  Each arm reports rounds/s and ms per round.
eval_splits_vector_kernel is then timed with torch.profiler over two rounds of the vector regression arm; its bytes come
from shapes: every level reads each node's T histograms once, 2^d nodes x T x (feature slots x 256 bins x 16 bytes) at
depth d < max_depth.  The card's name and power limit are read in the same run.  Writes nothing to the tree."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

T_MULTI = 4
ARMS = {"squarederror_per_tree": ("reg:squarederror", "one_output_per_tree"),
        "squarederror_vector": ("reg:squarederror", "multi_output_tree"),
        "logistic_vector": ("binary:logistic", "multi_output_tree")}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers are still worth printing, marked as unattributed
        return "unknown (%s)" % e


def labels(X, y):
    """bench.py's label and a T_MULTI-column label derived from it (regression, and 0/1 for classification)."""
    Y = np.empty((len(y), T_MULTI), np.float32)
    for k in range(T_MULTI):
        Y[:, k] = y + np.float32(k) * np.sin(np.nan_to_num(X[:, k], nan=0.0))
    return {"reg:squarederror": {1: y, T_MULTI: Y},
            "binary:logistic": {T_MULTI: (Y > np.median(Y, axis=0)).astype(np.float32)}}


def scan_profile(E, params, dm, rounds=2):
    import torch
    from torch.profiler import ProfilerActivity, profile
    bst = E.Booster(dict(params, objective="reg:squarederror", multi_strategy="multi_output_tree", profile=0), cache=[dm])
    bst.update(dm, 0)
    bst.get_trees()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for r in range(rounds):
            bst.update(dm, 1 + r)
        bst.get_trees()
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if "eval_splits_vector_kernel" in e.name]
    slots = ((dm.num_col() + 31) // 32) * 32
    depth = int(params["max_depth"])
    nbytes = sum((1 << d) * T_MULTI * slots * 256 * 16 for d in range(depth)) * rounds   # upper bound: every node splits
    total_s = float(np.sum(times)) / 1e6 if times else float("nan")
    return {"launches": len(times), "ms_per_round": total_s * 1e3 / rounds, "ms_per_launch": total_s * 1e3 / max(len(times), 1),
            "histogram_bytes_per_round_upper_bound": nbytes // rounds,
            "achieved_GBps_upper_bound": nbytes / total_s / 1e9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import bench
    from xgboost_ray_b200 import engine as E
    cols, depth = bench.WORKLOADS["C3"]["cols"], bench.WORKLOADS["C3"]["depth"]
    X, y = bench.synth_shard(args.rows, cols, 0, 1, workload="C3")
    L = labels(X, y)
    params = dict(bench.PARAMS, max_depth=depth, base_score=0.5)
    params.pop("objective", None)
    dm = E.DMatrix(X, label=y, multi_target=True)
    dm._ensure_quantized(256)
    out = {k: {"rounds_per_s": [], "ms_per_round": [], "model_sha256": None} for k in ARMS}
    for _ in range(args.repeats):
        for name, (obj, strategy) in ARMS.items():
            dm.set_info(label=L[obj][T_MULTI])    # the bins stay: only the label changes between arms
            bst = E.Booster(dict(params, objective=obj, multi_strategy=strategy), cache=[dm])
            for r in range(args.warmup):
                bst.update(dm, r)
            bst.get_trees()                       # the warm-up rounds are finished
            t0 = time.perf_counter()
            for r in range(args.steps):
                bst.update(dm, args.warmup + r)
            n_trees = len(bst.get_trees())        # waits for the last enqueued round
            wall = time.perf_counter() - t0
            per_round = 1 if strategy == "multi_output_tree" else T_MULTI
            assert bst.num_class == T_MULTI and n_trees == (args.warmup + args.steps) * per_round
            out[name]["rounds_per_s"].append(args.steps / wall)
            out[name]["ms_per_round"].append(wall / args.steps * 1e3)
            dump = "\n".join(bst.get_dump(dump_format="json", with_stats=True)).encode()
            out[name]["model_sha256"] = hashlib.sha256(dump).hexdigest()
            del bst
    for e in out.values():
        e["median_rounds_per_s"] = float(np.median(e["rounds_per_s"]))
        e["median_ms_per_round"] = float(np.median(e["ms_per_round"]))
    dm.set_info(label=L["reg:squarederror"][T_MULTI])
    res = {"metric": "boosting rounds/sec with a label of T columns, per-target vs vector-leaf trees", "card": card(),
           "config": "C3 synthetic %dx%d depth %d 256 bins, 1 GPU, T = %d" % (args.rows, cols, depth, T_MULTI),
           "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats, "arms": out,
           "eval_splits_vector_kernel": scan_profile(E, params, dm)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
