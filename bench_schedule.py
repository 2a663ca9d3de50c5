#!/usr/bin/env python
"""bench_schedule.py -- boosting rounds/sec of bench.py's C3 workload when the learning rate changes between rounds
(Booster.set_param, DESIGN.md 2 item 22), one GPU.

    python bench_schedule.py --steps K --warmup W [--rows N] [--repeats R]

Same synthetic matrix (bench.py's generator, 10M x 100), parameters and depth as bench.py's C3 headline, quantised once
and resident in HBM.  Three arms: eta constant; eta changed every 10 rounds; eta changed every round.  A change makes
the captured tree graphs stale, so the next tree of each round parity is captured again and applied to its graph with
cudaGraphExecUpdate; the engine timers report how many trees paid that and the host time it took (graph_update_ms).
The arms alternate R times (W untimed rounds, then K timed rounds each time) and report rounds/s, ms per round and the
cost per change.  The card's name and power limit are read in the same run.  Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

ARMS = {"constant": 0, "every_10_rounds": 10, "every_round": 1}   # rounds between two changes (0: never)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers are still worth printing, marked as unattributed
        return "unknown (%s)" % e


def eta_at(r, every):
    """The schedule's eta for round r: alternates between 0.3 and 0.2 every `every` rounds (0: always 0.3)."""
    return 0.3 if every == 0 or (r // every) % 2 == 0 else 0.2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=3)
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
    out = {k: {"rounds_per_s": [], "ms_per_round": [], "changes": 0, "graph_updates": 0, "graph_reinstantiations": 0,
               "graph_update_ms": 0.0} for k in ARMS}
    for _ in range(args.repeats):
        for name, every in ARMS.items():
            bst = E.Booster(params, cache=[dm])
            for r in range(args.warmup):
                bst.update(dm, r)
            bst.get_trees()                       # the warm-up rounds are finished
            bst.get_timers(reset=True)
            changes = 0
            t0 = time.perf_counter()
            for i in range(args.steps):
                r = args.warmup + i
                if eta_at(r, every) != eta_at(r - 1, every):
                    bst.set_param("learning_rate", eta_at(r, every))
                    changes += 1
                bst.update(dm, r)
            n_trees = len(bst.get_trees())        # waits for the last enqueued round
            wall = time.perf_counter() - t0
            assert n_trees == args.warmup + args.steps
            t = bst.get_timers()
            e = out[name]
            e["rounds_per_s"].append(args.steps / wall)
            e["ms_per_round"].append(wall / args.steps * 1e3)
            e["changes"] += changes
            for k in ("graph_updates", "graph_reinstantiations", "graph_update_ms"):
                e[k] += t[k]
            del bst
    base = float(np.median(out["constant"]["ms_per_round"]))
    for e in out.values():
        e["median_rounds_per_s"] = float(np.median(e["rounds_per_s"]))
        e["median_ms_per_round"] = float(np.median(e["ms_per_round"]))
        trees = e["graph_updates"] + e["graph_reinstantiations"]
        # host time of one re-captured tree, and the wall time a change adds over the constant arm
        e["graph_update_ms_per_tree"] = e["graph_update_ms"] / trees if trees else 0.0
        e["wall_ms_per_change"] = ((e["median_ms_per_round"] - base) * args.steps * args.repeats / e["changes"]
                                   if e["changes"] else 0.0)
    res = {"metric": "boosting rounds/sec with eta changed between rounds (Booster.set_param)", "card": card(),
           "config": "C3 synthetic %dx%d depth %d 256 bins, 1 GPU" % (args.rows, cols, depth),
           "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats, "arms": out}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
