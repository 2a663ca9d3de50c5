#!/usr/bin/env python
"""bench_constraints.py -- boosting rounds/sec of the C3 workload of bench.py with and without interaction constraints,
one GPU.

    python bench_constraints.py --steps K --warmup W [--rows N] [--repeats R]

Same synthetic matrix (bench.py's generator, 10M x 100), parameters and depth as bench.py's C3 headline, quantised once
and resident in HBM.  Three arms: no constraints; two sets [[0..49], [50..99]]; twenty sets of five consecutive
features.  The arms alternate R times (W untimed rounds, then K timed rounds each time), so that drift of the shared
host touches every arm alike; the JSON line reports every repeat.  The card's name and power limit are read in the
same run.
Parity, on a 200k-row, 3-round sub-problem per arm: every tree obeys the constraints, and for the arms whose root
features all lie in one set (the C3 signal is in features 0..10, so the two-set arm) the model equals the CPU oracle's
on the matrix with the other features held constant (split feature / bin / default direction exact, leaves within
1e-5).  Writes nothing to the tree.
"""
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

ARMS = {"none": None,
        "2x50": [list(range(0, 50)), list(range(50, 100))],
        "20x5": [list(range(5 * k, 5 * k + 5)) for k in range(20)]}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers are still worth printing, marked as unattributed
        return "unknown (%s)" % e


def violations(trees, sets, F):
    bad = 0
    for t in trees:
        stack = [(0, frozenset())]
        while stack:
            nid, path = stack.pop()
            f = int(t["split_feature"][nid])
            if f < 0:
                continue
            if path and not any(path | {f} <= set(s) for s in sets):
                bad += 1
            stack += [(int(t["left"][nid]), path | {f}), (int(t["right"][nid]), path | {f})]
    return bad


def parity(E, params, sets, X, y):
    from oracle import oracle as O
    p = dict(params) if sets is None else dict(params, interaction_constraints=sets)
    bst = E.train(p, E.DMatrix(X, label=y), num_boost_round=3, verbose_eval=False)
    trees = bst.get_trees()
    out = {"rule_violations": violations(trees, sets, X.shape[1]) if sets else 0}
    roots = {int(t["split_feature"][0]) for t in trees}
    keep = None if sets is None else next((s for s in sets if roots <= set(s)), None)
    if sets is None or keep is not None:
        Xm = X.copy()
        if keep is not None:
            Xm[:, [j for j in range(X.shape[1]) if j not in keep]] = 0.0
        ob, _ = O.train(params, Xm, y, 3)
        same, leaf = True, 0.0
        for i, t in enumerate(trees):
            o = ob.tree(i)
            same &= bool(np.array_equal(t["split_feature"], o.split_feature) and np.array_equal(t["split_bin"], o.split_bin)
                         and np.array_equal(t["default_left"], o.default_left))
            lf = o.split_feature < 0
            leaf = max(leaf, float(np.max(np.abs(t["value"][lf] - o.value[lf]))))
        out["oracle_match"], out["max_leaf_diff"] = same and leaf <= 1e-5, leaf
    else:
        out["oracle_match"] = "not comparable: roots in %d sets" % len({i for i, s in enumerate(sets) if roots & set(s)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()
    import bench
    from xgboost_ray_b200 import engine as E
    cols, depth = bench.WORKLOADS["C3"]["cols"], bench.WORKLOADS["C3"]["depth"]
    X, y = bench.synth_shard(args.rows, cols, 0, 1, workload="C3")
    params = dict(bench.PARAMS, max_depth=depth, objective="reg:squarederror")
    dm = E.DMatrix(X, label=y)
    dm._ensure_quantized(256)
    out = {k: {"rounds_per_s": [], "model_sha256": None} for k in ARMS}
    for _ in range(args.repeats):
        for name, sets in ARMS.items():
            p = dict(params) if sets is None else dict(params, interaction_constraints=sets)
            bst = E.Booster(p, cache=[dm])
            for r in range(args.warmup):
                bst.update(dm, r)
            bst.get_trees()                       # the warm-up rounds are finished
            t0 = time.perf_counter()
            for r in range(args.steps):
                bst.update(dm, args.warmup + r)
            n_trees = len(bst.get_trees())        # waits for the last enqueued round
            wall = time.perf_counter() - t0
            assert n_trees == args.warmup + args.steps
            out[name]["rounds_per_s"].append(args.steps / wall)
            dump = "\n".join(bst.get_dump(dump_format="json", with_stats=True)).encode()
            out[name]["model_sha256"] = hashlib.sha256(dump).hexdigest()
            del bst
    for e in out.values():
        e["median_rounds_per_s"] = float(np.median(e["rounds_per_s"]))
    if not args.no_parity:
        Xs, ys = bench.synth_shard(min(200_000, args.rows), cols, 0, 1, workload="C3")
        for name, sets in ARMS.items():
            out[name]["parity"] = parity(E, dict(params, profile=0), sets, Xs, ys)
    print(json.dumps({"metric": "boosting rounds/sec with interaction constraints", "card": card(),
                      "config": "C3 synthetic %dx%d depth %d 256 bins, 1 GPU" % (args.rows, cols, depth),
                      "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats, "arms": out}))


if __name__ == "__main__":
    main()
