#!/usr/bin/env python
"""bench_quantile.py -- boosting rounds/sec of the C3 workload of bench.py with reg:quantileerror, one GPU, and the time
of the leaf refresh kernels (quantile_count_kernel, quantile_scan_kernel).

    python bench_quantile.py --steps K --warmup W [--rows N] [--repeats R]

Same synthetic matrix (bench.py's generator, 10M x 100), parameters and depth as bench.py's C3 headline, quantised once
and resident in HBM.  Three arms: reg:squarederror; reg:quantileerror with one alpha (0.5); with three alphas (0.05,
0.5, 0.95), three trees per round.  The arms alternate R times (W untimed rounds, then K timed rounds each time), so that
drift of the shared host touches every arm alike.  The refresh kernels are then timed with torch.profiler over two
rounds of the one-alpha arm.  Bytes per count pass come from shapes: every row reads its leaf index (2 B), label (4 B),
margin (4 B) and gradient pair (8 B); the scans read and zero 2 x 256 x 8 B per leaf.  The card's name and power limit
are read in the same run.  Writes nothing to the tree."""
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

ARMS = {"squarederror": {"objective": "reg:squarederror"},
        "quantile_1": {"objective": "reg:quantileerror", "quantile_alpha": 0.5},
        "quantile_3": {"objective": "reg:quantileerror", "quantile_alpha": [0.05, 0.5, 0.95]}}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers are still worth printing, marked as unattributed
        return "unknown (%s)" % e


def refresh_profile(E, params, dm, depth, rounds=2):
    import torch
    from torch.profiler import ProfilerActivity, profile
    bst = E.Booster(dict(params, **ARMS["quantile_1"], profile=0), cache=[dm])
    bst.update(dm, 0)
    bst.get_trees()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for r in range(rounds):
            bst.update(dm, 1 + r)
        bst.get_trees()
        torch.cuda.synchronize()
    count = [e.device_time for e in prof.events() if "quantile_count_kernel" in e.name]
    scan = [e.device_time for e in prof.events() if "quantile_scan_kernel" in e.name]
    n, leaves = dm.num_row(), 1 << depth
    count_bytes = n * (2 + 4 + 4 + 8)
    per_tree_ms = (sum(count) + sum(scan)) / 1e3 / rounds
    return {"trees": rounds, "count_launches": len(count), "scan_launches": len(scan),
            "count_ms_per_pass": float(np.mean(count)) / 1e3, "scan_ms_per_pass": float(np.mean(scan)) / 1e3,
            "refresh_ms_per_tree": per_tree_ms, "count_bytes_per_pass": count_bytes,
            "count_achieved_GBps": count_bytes / (np.mean(count) / 1e6) / 1e9,
            "scan_bytes_per_pass": leaves * 2 * 256 * 8 * 2}


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
    params = dict(bench.PARAMS, max_depth=depth, base_score=0.5)
    params.pop("objective", None)
    dm = E.DMatrix(X, label=y)
    dm._ensure_quantized(256)
    out = {k: {"rounds_per_s": [], "model_sha256": None} for k in ARMS}
    for _ in range(args.repeats):
        for name, extra in ARMS.items():
            bst = E.Booster(dict(params, **extra), cache=[dm])
            for r in range(args.warmup):
                bst.update(dm, r)
            bst.get_trees()                       # the warm-up rounds are finished
            t0 = time.perf_counter()
            for r in range(args.steps):
                bst.update(dm, args.warmup + r)
            n_trees = len(bst.get_trees())        # waits for the last enqueued round
            wall = time.perf_counter() - t0
            assert n_trees == (args.warmup + args.steps) * bst.num_class
            out[name]["rounds_per_s"].append(args.steps / wall)
            dump = "\n".join(bst.get_dump(dump_format="json", with_stats=True)).encode()
            out[name]["model_sha256"] = hashlib.sha256(dump).hexdigest()
            del bst
    for e in out.values():
        e["median_rounds_per_s"] = float(np.median(e["rounds_per_s"]))
    res = {"metric": "boosting rounds/sec with reg:quantileerror", "card": card(),
           "config": "C3 synthetic %dx%d depth %d 256 bins, 1 GPU" % (args.rows, cols, depth),
           "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats, "arms": out,
           "leaf_refresh": refresh_profile(E, params, dm, depth)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
