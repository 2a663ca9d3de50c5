#!/usr/bin/env python
"""bench_depth.py -- boosting rounds/sec of the C3 workload of bench.py at max_depth 14, 15 and 16, one GPU, and
TreeSHAP throughput on the depth-16 model.

    python bench_depth.py --steps K --warmup W [--rows N] [--repeats R] [--shap-rows S]

Same synthetic matrix (bench.py's generator, 10M x 100), parameters and 256 bins as bench.py's C3 headline, quantised
once and resident in HBM; only max_depth changes.  The three arms alternate R times (W untimed rounds, then K timed
rounds each time), so that drift of the shared host touches every arm alike.  At F = 100 (4 feature groups) the two
level buffers take 2 x 2^(D-1) x 4 x 128 KiB: 8 GiB at depth 14, 16 GiB at 15 and 32 GiB at 16.

TreeSHAP: pred_contribs of the last depth-16 model on S raw rows of the same generator, timed with the engine's
`shap_ms` CUDA-event timer and host wall time around the synchronised call.  A depth-16 tree has tens of thousands of
leaves whose paths cost L^2 steps each, so a row costs far more than at depth 8 and S is small.  The card's name,
power limit and maximum SM clock are read in the same run.  Parity, on a 200k-row sub-problem at depth 16: the trees
equal the CPU oracle's (splits exactly, leaf values within 1e-5), and the contributions of a few rows sum to the
margin.  Writes nothing to the tree.
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

DEPTHS = (14, 15, 16)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers are still worth printing, marked as unattributed
        return "unknown (%s)" % e


def path_steps(trees):
    """TreeSHAP work of one row: sum over leaves of L^2, L = 1 + distinct features on the leaf's path"""
    total, leaves, longest = 0, 0, 0
    for t in trees:
        left, right, feat = t["left"], t["right"], t["split_feature"]
        stack = [(0, frozenset())]
        while stack:
            nid, fs = stack.pop()
            if feat[nid] < 0:
                L = 1 + len(fs)
                total += L * L
                leaves += 1
                longest = max(longest, L)
                continue
            nfs = fs | {int(feat[nid])}
            stack.append((int(left[nid]), nfs))
            stack.append((int(right[nid]), nfs))
    return {"leaves": leaves, "longest_path": longest, "path_steps_per_row": total}


def tree_shape(trees):
    def depth(t):
        d = np.zeros(len(t["left"]), np.int32)
        for nid in range(1, len(d)):
            d[nid] = d[t["parent"][nid]] + 1
        return int(d.max())
    return {"max_depth_reached": max(depth(t) for t in trees),
            "max_leaves": max(int((t["split_feature"] < 0).sum()) for t in trees)}


def parity(E, params, X, y, rounds=2):
    from oracle import oracle as O
    O.build()
    ob, _ = O.train(params, X, y, rounds)
    bst = E.train(params, E.DMatrix(X, label=y), num_boost_round=rounds, verbose_eval=False)
    same, leaf_err = True, 0.0
    for i, t in enumerate(bst.get_trees()):
        o = ob.tree(i)
        same &= len(t["left"]) == o.n_nodes and bool(np.array_equal(t["split_feature"], o.split_feature)) \
            and bool(np.array_equal(t["split_bin"], o.split_bin)) and bool(np.array_equal(t["left"], o.left))
        leaf = o.split_feature < 0
        if len(t["left"]) == o.n_nodes:
            leaf_err = max(leaf_err, float(np.max(np.abs(t["value"][leaf] - o.value[leaf]))))
    xs = X[:2000]
    phi = bst.predict(E.DMatrix(xs), pred_contribs=True)
    margin = bst.predict(E.DMatrix(xs), output_margin=True)
    return {"rows": int(X.shape[0]), "rounds": rounds, "trees_identical": bool(same), "leaf_max_abs_err": leaf_err,
            "shape": tree_shape(bst.get_trees()),
            "contribs_local_accuracy_max_err": float(np.max(np.abs(phi.astype(np.float64).sum(axis=1) - margin)))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--shap-rows", type=int, default=2000)
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()
    import bench
    from xgboost_ray_b200 import engine as E
    cols = bench.WORKLOADS["C3"]["cols"]
    X, y = bench.synth_shard(args.rows, cols, 0, 1, workload="C3")
    params = dict(bench.PARAMS, objective="reg:squarederror", base_score=0.5)
    dm = E.DMatrix(X, label=y)
    dm._ensure_quantized(256)
    del X, y
    out = {d: {"rounds_per_s": [], "model_sha256": None} for d in DEPTHS}
    last = None
    for _ in range(args.repeats):
        for d in DEPTHS:
            last = None
            bst = E.Booster(dict(params, max_depth=d), cache=[dm])
            for r in range(args.warmup):
                bst.update(dm, r)
            bst.get_trees()                       # the warm-up rounds are finished
            t0 = time.perf_counter()
            for r in range(args.steps):
                bst.update(dm, args.warmup + r)
            trees = bst.get_trees()               # waits for the last enqueued round
            wall = time.perf_counter() - t0
            assert len(trees) == args.warmup + args.steps
            out[d]["rounds_per_s"].append(args.steps / wall)
            dump = "\n".join(bst.get_dump(dump_format="json", with_stats=True)).encode()
            out[d]["model_sha256"] = hashlib.sha256(dump).hexdigest()
            out[d].update(tree_shape(trees))
            if d == DEPTHS[-1]:
                last = bst
            else:
                del bst
    for e in out.values():
        e["median_rounds_per_s"] = float(np.median(e["rounds_per_s"]))

    Xp, _ = bench.synth_block(7, args.shap_rows, cols, seed=4321, workload="C3")
    dp = E.DMatrix(Xp)
    last.predict(E.DMatrix(Xp[:16]), pred_contribs=True)     # path table + first launch outside the timing
    last.get_timers(reset=True)
    t0 = time.perf_counter()
    phi = last.predict(dp, pred_contribs=True)
    wall = time.perf_counter() - t0
    kernel_ms = last.get_timers(reset=True)["shap_ms"]
    margin = last.predict(dp, output_margin=True)
    work = path_steps(last.get_trees())
    shap = {"rows": args.shap_rows, "trees": len(last.get_trees()), **work, "rows_per_s": args.shap_rows / wall,
            "wall_s": wall, "kernel_ms": kernel_ms,
            "path_steps_per_s": work["path_steps_per_row"] * args.shap_rows / (kernel_ms * 1e-3) if kernel_ms > 0 else None,
            "local_accuracy_max_err": float(np.max(np.abs(phi.astype(np.float64).sum(axis=1) - margin)))}
    del last, dm
    res = {"metric": "boosting rounds/sec by max_depth", "card": card(),
           "config": "C3 synthetic %dx%d 256 bins, 1 GPU" % (args.rows, cols),
           "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats,
           "arms": {"max_depth_%d" % d: v for d, v in out.items()}, "shap_depth16": shap}
    if not args.no_parity:
        Xs, ys = bench.synth_shard(min(200_000, args.rows), cols, 0, 1, workload="C3")
        res["parity_depth16"] = parity(E, dict(params, max_depth=16, min_child_weight=0.0), Xs, ys)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
