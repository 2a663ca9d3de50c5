#!/usr/bin/env python
"""bench_refresh.py -- the refresh updater (process_type="update", updater="refresh") against growing, one GPU.

    python bench_refresh.py [--rounds R] [--rows N] [--repeats K]

Same synthetic matrix (bench.py's generator, C3: 10M x 100), parameters and depth (8) as bench.py's C3 headline,
quantised once and resident in HBM with its raw floats.  Each repeat trains R rounds (grow), then refreshes those R
rounds on the same matrix (refresh), both through engine.train, timed by wall clock including the calls' setup.  The
refresh_kernel time comes from the engine's CUDA events around every launch (get_timers' refresh_ms and
refresh_launches; one launch per round here).  Its algorithmic bytes per launch: n x (4 x (depth + 1) path floats + 8
gradient-pair bytes + 2 pos bytes); a scattered path float can cost a whole 32-byte sector, which gives the upper
bound.  The card's name and power limit are read in the same run.  Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers are still worth printing, marked as unattributed
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=50)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import bench
    from xgboost_ray_b200 import engine as E
    cols, depth = bench.WORKLOADS["C3"]["cols"], bench.WORKLOADS["C3"]["depth"]
    X, y = bench.synth_shard(args.rows, cols, 0, 1, workload="C3")
    params = dict(bench.PARAMS, max_depth=depth, base_score=0.5)
    dm = E.DMatrix(X, label=y)
    dm._ensure_quantized(256)
    dm._ensure_raw()
    grow, refresh, kernel_ms = [], [], []
    for _ in range(args.repeats):
        t0 = time.perf_counter()
        bst = E.train(params, dm, args.rounds, verbose_eval=False)
        assert len(bst.get_trees()) == args.rounds
        grow.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        upd = E.train(dict(params, process_type="update", updater="refresh"), dm, args.rounds, xgb_model=bst)
        assert len(upd.get_trees()) == args.rounds
        refresh.append(time.perf_counter() - t0)
        timers = upd.get_timers()
        assert timers["refresh_launches"] == args.rounds
        kernel_ms.append(timers["refresh_ms"] / timers["refresh_launches"])
        del bst, upd
    n = args.rows
    lo = n * (4 * (depth + 1) + 8 + 2)
    hi = n * (32 * (depth + 1) + 8 + 2)
    km = float(np.median(kernel_ms))
    res = {"metric": "refresh rounds/s against grow rounds/s", "card": card(),
           "config": "C3 synthetic %dx%d depth %d 256 bins, 1 GPU, %d rounds" % (n, cols, depth, args.rounds),
           "repeats": args.repeats,
           "grow_rounds_per_s": float(np.median([args.rounds / t for t in grow])),
           "refresh_rounds_per_s": float(np.median([args.rounds / t for t in refresh])),
           "grow_ms_per_round": float(np.median(grow)) * 1e3 / args.rounds,
           "refresh_ms_per_round": float(np.median(refresh)) * 1e3 / args.rounds,
           "refresh_kernel": {"ms_per_launch": km, "bytes_per_launch_4B_per_float": lo,
                              "bytes_per_launch_32B_per_float": hi,
                              "GBps_at_4B_per_float": lo / (km * 1e-3) / 1e9 if km > 0 else None,
                              "GBps_at_32B_per_float": hi / (km * 1e-3) / 1e9 if km > 0 else None}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
