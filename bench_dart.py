#!/usr/bin/env python
"""bench_dart.py -- boosting rounds/sec of the C3 workload of bench.py with booster=dart, one GPU, and the time of the
DART margin rebuild (dart_margins_kernel) per dropping round.

    python bench_dart.py --steps K --warmup W [--rows N] [--repeats R]

Same synthetic matrix (bench.py's generator, 10M x 100), parameters and depth as bench.py's C3 headline, quantised once
and resident in HBM.  Three arms: gbtree; dart rate_drop=0 (nothing is ever dropped: only a host decision per round);
dart rate_drop=0.1 uniform.  The arms alternate R times (W untimed rounds, then K timed rounds each time), so that
drift of the shared host touches every arm alike.  The rebuild is then timed with torch.profiler on models of 100 / 200
/ 400 trees (grown with rate_drop=0, continued for one round with rate_drop=1 so that the round drops and the kernel
walks every tree), reported as kernel milliseconds and as node steps per second, counting rows x trees x depth steps
(an upper bound: a row that reaches a leaf early takes fewer).  The card's name and power limit are read in the same
run.  Parity, on a 200k-row sub-problem: the dart arm's weights equal tests/dart_reference.py's replay and its train
margins equal the reference's ordered weighted sums over the model's trees, bit for bit.  Writes nothing to the tree.
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

ARMS = {"gbtree": {}, "dart_rate0": {"booster": "dart", "rate_drop": 0.0},
        "dart_rate0.1": {"booster": "dart", "rate_drop": 0.1, "sample_type": "uniform"}}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers are still worth printing, marked as unattributed
        return "unknown (%s)" % e


def rebuild_ms(E, params, dm, n_trees, depth):
    """Kernel time of one dropping round's margin rebuild over n_trees trees."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    src = E.train(dict(params, booster="dart", rate_drop=0.0), dm, num_boost_round=n_trees, verbose_eval=False)
    bst = E.train(dict(params, booster="dart", rate_drop=1.0), dm, num_boost_round=0, xgb_model=src, verbose_eval=False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        bst.update(dm, 0)
        bst.get_trees()
        torch.cuda.synchronize()
    us = [e.device_time for e in prof.events() if "dart_margins_kernel" in e.name]
    if len(us) != 1:
        raise RuntimeError("expected one dart_margins_kernel launch, profiler saw %d" % len(us))
    ms = us[0] / 1e3
    steps = dm.num_row() * n_trees * depth
    return {"trees": n_trees, "kernel_ms": ms, "node_steps_per_s": steps / (ms / 1e3)}


def parity(E, params, X, y, rounds=12):
    from tests import dart_reference as R
    p = dict(params, **ARMS["dart_rate0.1"])
    d = E.DMatrix(X, label=y)
    bst = E.train(p, d, num_boost_round=rounds, verbose_eval=False)
    w_ref, drops = R.replay_weights(rounds, float(p["eta"]), 1, seed=int(p.get("seed", 0)), rate_drop=0.1)
    w = bst.get_tree_weights()
    full = R.margins(bst.get_trees(), w, d.get_bins(), d.get_cuts()[3],
                     np.full((X.shape[0], 1), float(bst.params["base_score"]), np.float32))
    got = bst.predict(d, output_margin=True)
    return {"weights_match": bool(w.tobytes() == w_ref.tobytes()), "rounds_with_drops": sum(1 for x in drops if x),
            "margins_match": bool(got.tobytes() == full[:, 0].tobytes())}


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
    params = dict(bench.PARAMS, max_depth=depth, objective="reg:squarederror", base_score=0.5)
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
            assert n_trees == args.warmup + args.steps
            out[name]["rounds_per_s"].append(args.steps / wall)
            dump = "\n".join(bst.get_dump(dump_format="json", with_stats=True)).encode()
            out[name]["model_sha256"] = hashlib.sha256(dump).hexdigest()
            del bst
    for e in out.values():
        e["median_rounds_per_s"] = float(np.median(e["rounds_per_s"]))
    rebuild = [rebuild_ms(E, dict(params, profile=0), dm, t, depth) for t in (100, 200, 400)]
    res = {"metric": "boosting rounds/sec with booster=dart", "card": card(),
           "config": "C3 synthetic %dx%d depth %d 256 bins, 1 GPU" % (args.rows, cols, depth),
           "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats, "arms": out,
           "margin_rebuild": rebuild}
    if not args.no_parity:
        Xs, ys = bench.synth_shard(min(200_000, args.rows), cols, 0, 1, workload="C3")
        res["parity"] = parity(E, dict(params, profile=0), Xs, ys)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
