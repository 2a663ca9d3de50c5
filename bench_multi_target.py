#!/usr/bin/env python
"""bench_multi_target.py -- boosting rounds/sec of the C3 workload of bench.py with a label of T columns (multi-target
regression, multi-label classification), one GPU, and the time of the multi-target gradient kernel.

    python bench_multi_target.py --steps K --warmup W [--rows N] [--repeats R]

Same synthetic matrix (bench.py's generator, 10M x 100), parameters and depth as bench.py's C3 headline, quantised once
and resident in HBM.  Three arms: reg:squarederror with T = 1 (bench.py's label); reg:squarederror with T = 4;
binary:logistic with T = 4.  Column k of the 4-column label is bench.py's label plus k times a feature-dependent shift
(thresholded at its median for binary:logistic), so the columns grow different trees.  The arms alternate R times (W
untimed rounds, then K timed rounds each time), so that drift of the shared host touches every arm alike.  Each arm
reports rounds/s and ms per tree (round time / T).  gradient_multi_target_kernel is then timed with torch.profiler over
two rounds of the T = 4 regression arm; its bytes come from shapes: n T (4 label + 4 margin + 8 gradient pair) + 4 n
weight, over the data sheet's 3.35 TB/s.  The card's name and power limit are read in the same run.  Writes nothing to
the tree."""
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
ARMS = {"squarederror_T1": ("reg:squarederror", 1), "squarederror_T4": ("reg:squarederror", T_MULTI),
        "logistic_T4": ("binary:logistic", T_MULTI)}
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


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


def gradient_profile(E, params, dm, rounds=2):
    import torch
    from torch.profiler import ProfilerActivity, profile
    bst = E.Booster(dict(params, objective="reg:squarederror", profile=0), cache=[dm])
    bst.update(dm, 0)
    bst.get_trees()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for r in range(rounds):
            bst.update(dm, 1 + r)
        bst.get_trees()
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if "gradient_multi_target_kernel" in e.name]
    n = dm.num_row()
    nbytes = n * T_MULTI * (4 + 4 + 8) + 4 * n
    mean_s = float(np.mean(times)) / 1e6 if times else float("nan")
    return {"launches": len(times), "ms_per_launch": mean_s * 1e3, "bytes_per_launch": nbytes,
            "achieved_GBps": nbytes / mean_s / 1e9, "share_of_3_35_TBps": nbytes / mean_s / HBM_BYTES_PER_S}


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
    out = {k: {"rounds_per_s": [], "ms_per_tree": [], "model_sha256": None} for k in ARMS}
    for _ in range(args.repeats):
        for name, (obj, T) in ARMS.items():
            dm.set_info(label=L[obj][T])          # the bins stay: only the label changes between arms
            bst = E.Booster(dict(params, objective=obj), cache=[dm])
            for r in range(args.warmup):
                bst.update(dm, r)
            bst.get_trees()                       # the warm-up rounds are finished
            t0 = time.perf_counter()
            for r in range(args.steps):
                bst.update(dm, args.warmup + r)
            n_trees = len(bst.get_trees())        # waits for the last enqueued round
            wall = time.perf_counter() - t0
            assert bst.num_class == T and n_trees == (args.warmup + args.steps) * T
            out[name]["rounds_per_s"].append(args.steps / wall)
            out[name]["ms_per_tree"].append(wall / args.steps / T * 1e3)
            dump = "\n".join(bst.get_dump(dump_format="json", with_stats=True)).encode()
            out[name]["model_sha256"] = hashlib.sha256(dump).hexdigest()
            del bst
    for e in out.values():
        e["median_rounds_per_s"] = float(np.median(e["rounds_per_s"]))
        e["median_ms_per_tree"] = float(np.median(e["ms_per_tree"]))
    dm.set_info(label=L["reg:squarederror"][T_MULTI])
    res = {"metric": "boosting rounds/sec with a label of T columns", "card": card(),
           "config": "C3 synthetic %dx%d depth %d 256 bins, 1 GPU, T = 1 and %d" % (args.rows, cols, depth, T_MULTI),
           "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats, "arms": out,
           "gradient_kernel": gradient_profile(E, params, dm)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
