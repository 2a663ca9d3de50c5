#!/usr/bin/env python
"""bench_auc.py -- milliseconds per B2_BoosterEvalSet call of `auc` and `aucpr`, one GPU, next to the boosting
rounds/sec of training on the same matrix.

    python bench_auc.py --steps K --warmup W [--rows N] [--mc-rows M] [--calls C]

Two matrices, both from bench.py's C3 generator (x ~ U[0, 10), 100 columns):
- binary: N rows (default 10M, the C3 matrix) with label [y > median(y)], binary:logistic at C3's depth 8;
- multi-class: M rows (default 2M) with y cut into 10 classes at its deciles, multi:softprob with num_class = 10.
Each is trained for W + K rounds (K timed), then each metric is evaluated on the train matrix 2 times untimed and C
times timed (every call ends in a device synchronise).  The values are also checked against tests/auc_reference.py on
a 200k-row subsample (the engine's B2_BoosterEvalSet on a matrix of those rows against the reference on the engine's
predictions of it, tolerance 1e-9).  The card's name and power limit are read in the same run.  Writes nothing to
the tree."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRICS = ("auc", "aucpr")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers are still worth printing, marked as unattributed
        return "unknown (%s)" % e


def eval_once(E, bst, dm, metric):
    v = C.c_double(0)
    E._check(E.lib().B2_BoosterEvalSet(bst.handle, dm.handle, metric.encode(), C.byref(v)))
    return v.value


def run_arm(E, R, X, y, params, args, sub_rows=200_000):
    dm = E.DMatrix(X, label=y)
    dm._ensure_quantized(256)
    bst = E.Booster(dict(params, eval_metric=list(METRICS)), cache=[dm])
    for r in range(args.warmup):
        bst.update(dm, r)
    bst.get_trees()
    t0 = time.perf_counter()
    for r in range(args.steps):
        bst.update(dm, args.warmup + r)
    bst.get_trees()                               # waits for the last enqueued round
    rounds_per_s = args.steps / (time.perf_counter() - t0)
    out = {"rows": len(y), "rounds_per_s": rounds_per_s, "round_ms": 1e3 / rounds_per_s}
    for metric in METRICS:
        for _ in range(2):
            eval_once(E, bst, dm, metric)
        ms = []
        for _ in range(args.calls):
            t = time.perf_counter()
            v = eval_once(E, bst, dm, metric)
            ms.append((time.perf_counter() - t) * 1e3)
        out[metric] = {"value": v, "ms_per_call": float(np.median(ms)), "ms_min": float(np.min(ms)),
                       "ms_max": float(np.max(ms))}
    ds = E.DMatrix(X[:sub_rows], label=y[:sub_rows])
    p = bst.predict(ds)
    diffs = {m: abs(eval_once(E, bst, ds, m) - R.value(m, p, y[:sub_rows])) for m in METRICS}
    out["reference_check"] = {"rows": min(sub_rows, len(y)), "max_abs_diff": max(diffs.values()),
                              "match": all(d < 1e-9 for d in diffs.values())}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--mc-rows", type=int, default=2_000_000)
    ap.add_argument("--calls", type=int, default=10)
    args = ap.parse_args()
    import bench
    from tests import auc_reference as R
    from xgboost_ray_b200 import engine as E
    cols, depth = bench.WORKLOADS["C3"]["cols"], bench.WORKLOADS["C3"]["depth"]
    params = dict(bench.PARAMS, max_depth=depth, base_score=0.5)
    res = {"metric": "ms per B2_BoosterEvalSet call of auc / aucpr", "card": card(), "steps": args.steps,
           "warmup": args.warmup, "calls": args.calls}
    X, y = bench.synth_shard(args.rows, cols, 0, 1, workload="C3")
    yb = (y > np.median(y)).astype(np.float32)
    res["binary"] = dict(config="C3 synthetic %dx%d binary:logistic depth %d, 1 GPU" % (args.rows, cols, depth),
                         **run_arm(E, R, X, yb, dict(params, objective="binary:logistic"), args))
    del X, y, yb
    X, y = bench.synth_shard(args.mc_rows, cols, 0, 1, workload="C3")
    yk = np.digitize(y, np.quantile(y, np.linspace(0.1, 0.9, 9))).astype(np.float32)
    mc = dict(params, objective="multi:softprob", num_class=10)
    mc.pop("base_score")
    res["multiclass"] = dict(config="C3 generator %dx%d, 10 classes, multi:softprob depth %d, 1 GPU"
                             % (args.mc_rows, cols, depth), **run_arm(E, R, X, yk, mc, args))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
