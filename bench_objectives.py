#!/usr/bin/env python
"""bench_objectives.py -- boosting rounds/sec of the C3 workload of bench.py under several objectives, one H100.

    python bench_objectives.py --steps K --warmup W [--objectives reg:squarederror,count:poisson,...] [--rows N]

Same synthetic matrix (bench.py's generator, 10M x 100), parameters and depth as bench.py's C3 headline, trained once
per objective with the matrix quantised and resident in HBM (the `value` arm of bench.py: W untimed rounds, then K
timed rounds).  Labels are a fixed map of the C3 label y, with no new randomness:
  float32(log1p(exp(y/10)) + 1e-3)  for count:poisson, reg:gamma, reg:tweedie, reg:squaredlogerror, reg:pseudohubererror;
  float32(sigmoid(y/10))            for reg:logistic, binary:logistic, binary:logitraw;
  y itself                          for reg:squarederror;
  survival:aft reads bounds built from the positive map t by row index: row mod 4 = 0 -> [t, t], 1 -> [t, +inf),
  2 -> [0, t], 3 -> [t, 2t];
  rank:pairwise and rank:ndcg read the relevance digitize(y, quantiles of y at 20/40/60/80 %) in 0..4 and the query
  groups qid = row // 100 (the C3 matrix has 100k groups of 100 rows; the oracle sub-problem 2,000).
For every objective a 200k-row, 3-round sub-problem is also compared tree for tree with the CPU oracle grown from the
gradients of tests/objective_reference.py (split feature / bin / default direction exact, leaf values within 1e-5).
Prints one JSON line with one entry per objective.  Writes nothing to the tree.
"""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

RANK = ("rank:pairwise", "rank:ndcg")
POSITIVE = ("count:poisson", "reg:gamma", "reg:tweedie", "reg:squaredlogerror", "reg:pseudohubererror", "survival:aft")
UNIT = ("reg:logistic", "binary:logistic", "binary:logitraw")


def objective_labels(objective, y):
    """The C3 label mapped into the domain of `objective` (see the module docstring)."""
    t = y.astype(np.float64) / 10.0
    if objective in POSITIVE:
        return (np.logaddexp(0.0, t) + 1e-3).astype(np.float32)     # log1p(exp(t)) without overflow
    if objective in UNIT:
        return (1.0 / (1.0 + np.exp(-t))).astype(np.float32)
    if objective in RANK:
        return np.digitize(y, np.quantile(y, [0.2, 0.4, 0.6, 0.8])).astype(np.float32)
    return y


def aft_bounds(t):
    """survival:aft bounds of the positive label map t (see the module docstring)."""
    k = np.arange(len(t)) % 4
    lo = np.where(k == 2, np.float32(0.0), t).astype(np.float32)
    hi = np.where(k == 1, np.float32(np.inf), np.where(k == 3, t * np.float32(2.0), t)).astype(np.float32)
    return lo, hi


def make_matrix(E, objective, X, y):
    if objective == "survival:aft":
        lo, hi = aft_bounds(y)
        return E.DMatrix(X, label=y, label_lower_bound=lo, label_upper_bound=hi)
    if objective in RANK:
        return E.DMatrix(X, label=y, qid=np.arange(len(y)) // 100)
    return E.DMatrix(X, label=y)


def oracle_match(E, params, X, y):
    from oracle import oracle as O
    from tests import objective_reference as R
    d = make_matrix(E, params["objective"], X, y)
    b = E.train(params, d, num_boost_round=3, verbose_eval=False)
    if params["objective"] == "survival:aft":
        from tests import survival_reference as S
        ob = S.train(O, params, X, *aft_bounds(y), 3)
    elif params["objective"] in RANK:
        from tests import ranking_reference as RR
        ob = RR.train(O, params, X, y, np.arange(len(y)) // 100, 3)
    elif params["objective"] in R.OBJECTIVES:
        ob = R.train(O, params, X, y, 3)
    else:
        ob, _ = O.train(params, X, y, 3)
    worst = 0.0
    for i, t in enumerate(b.get_trees()):
        o = ob.tree(i)
        if not (np.array_equal(t["split_feature"], o.split_feature) and np.array_equal(t["split_bin"], o.split_bin)
                and np.array_equal(t["default_left"], o.default_left)):
            return False, None
        leaf = o.split_feature < 0
        worst = max(worst, float(np.max(np.abs(t["value"][leaf] - o.value[leaf]))))
    return worst <= 1e-5 and len(b.get_trees()) == ob.num_trees, worst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--objectives", default="reg:squarederror,count:poisson,reg:tweedie,reg:gamma")
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()
    import bench
    from xgboost_ray_b200 import engine as E
    cols, depth = bench.WORKLOADS["C3"]["cols"], bench.WORKLOADS["C3"]["depth"]
    X, y0 = bench.synth_shard(args.rows, cols, 0, 1, workload="C3")
    n_sub = min(200_000, args.rows)
    Xs, ys0 = bench.synth_shard(n_sub, cols, 0, 1, workload="C3")
    out = {}
    for obj in args.objectives.split(","):
        params = dict(bench.PARAMS, max_depth=depth, objective=obj)
        dm = make_matrix(E, obj, X, objective_labels(obj, y0))
        dm._ensure_quantized(256)
        bst = E.Booster(params, cache=[dm])
        for r in range(args.warmup):
            bst.update(dm, r)
        bst.get_timers(reset=True)
        t0 = time.perf_counter()
        for r in range(args.steps):
            bst.update(dm, args.warmup + r)
        wall = time.perf_counter() - t0
        timers = bst.get_timers(reset=True)
        dump = "\n".join(bst.get_dump(dump_format="json", with_stats=True)).encode()
        entry = {"value": args.steps / wall, "unit": "rounds/s", "ms_per_step": 1e3 * wall / args.steps,
                 "device_ms_per_step": timers["round_ms"] / args.steps,
                 "model_sha256": hashlib.sha256(dump).hexdigest(),
                 "final_train_metric": bst.eval_set([(dm, "train")], 0).split("\t", 1)[-1]}
        del bst, dm
        if not args.no_parity:
            sub = dict(params, max_depth=min(depth, 8), profile=0)
            entry["oracle_match"], entry["max_leaf_diff"] = oracle_match(E, sub, Xs, objective_labels(obj, ys0))
        out[obj] = entry
    print(json.dumps({"metric": "boosting rounds/sec per objective", "config": "C3 synthetic %dx%d depth %d 256 bins, 1 GPU"
                      % (args.rows, cols, depth), "steps": args.steps, "warmup": args.warmup, "objectives": out}))


if __name__ == "__main__":
    main()
