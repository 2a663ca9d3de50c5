#!/usr/bin/env python
"""bench_cv.py -- k-fold cross-validation of bench.py's C3 workload on one GPU: cv(), whose fold matrices are gathered
on the device with DMatrix.slice, against what a user without slice() does, one train() per fold on matrices rebuilt on
the host as DMatrix(X[idx]) and uploaded.

    python bench_cv.py [--rows N] [--folds K] [--rounds R] [--repeats N]

Same synthetic matrix (bench.py's generator, 10M x 100), parameters and depth as bench.py's C3 headline.  Both arms
evaluate the train and test side of every fold in every round, with the same folds (cv_folds, seed 0).  Reported:
- slice_s: the 2K slices of the folds taken on their own (host clock; B2_MatrixSlice returns after its stream is
  synchronised), against host_rebuild_s: X[idx] on the host plus the upload of every fold matrix of the loop;
- fold_rounds_per_s: boosting rounds (with their evaluation) per second summed over the folds, timed by a callback from
  the first round's start to the last round's end, so it excludes slicing, rebuilding and quantisation;
- wall_s of each arm, from the parent matrix on the device (cv) or on the host (loop) to the results;
- agree: cv()'s means and stds equal those of the loop exactly.
A small cv() runs first so that module loading is not timed; the two arms then alternate --repeats times.  The card's
name and power limit are read in the same run.  Writes nothing to the tree."""
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
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers are still worth printing, marked as unattributed
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--folds", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    import bench
    from xgboost_ray_b200 import engine as E
    if E.device_count() < 1:
        raise SystemExit("bench_cv.py needs a CUDA device")
    cols, depth = bench.WORKLOADS["C3"]["cols"], bench.WORKLOADS["C3"]["depth"]
    X, y = bench.synth_shard(args.rows, cols, 0, 1, workload="C3")
    params = dict(bench.PARAMS, max_depth=depth, objective="reg:squarederror", base_score=0.5)
    K, R = args.folds, args.rounds

    class RoundTimer(E.TrainingCallback):
        """Time from the start of round 0 to the end of the last round (its metrics are read back by then)."""
        def __init__(self):
            self.t0 = self.t1 = None

        def before_iteration(self, model, epoch, evals_log):
            if epoch == 0:
                self.t0 = time.perf_counter()
            return False

        def after_iteration(self, model, epoch, evals_log):
            self.t1 = time.perf_counter()
            return False

    small = E.DMatrix(X[:100_000], label=y[:100_000])
    E.cv(params, small, num_boost_round=2, nfold=K, as_pandas=False)
    del small
    folds = E.cv_folds(args.rows, K, seed=0)

    def run_cv():
        """(a) cv() on a matrix uploaded once; then the 2K slices of its folds timed on their own"""
        t_wall = time.perf_counter()
        dm = E.DMatrix(X, label=y)
        upload_s = time.perf_counter() - t_wall
        timer = RoundTimer()
        got = E.cv(params, dm, num_boost_round=R, nfold=K, seed=0, callbacks=[timer], as_pandas=False)
        wall = time.perf_counter() - t_wall
        t = time.perf_counter()
        slices = [dm.slice(idx) for tr, te, _, _ in folds for idx in (tr, te)]
        slice_s = time.perf_counter() - t
        del slices, dm
        return got, {"wall_s": wall, "parent_upload_s": upload_s, "slice_s": slice_s,
                     "fold_rounds_per_s": K * R / (timer.t1 - timer.t0)}

    def run_loop():
        """(b) one train() per fold on matrices rebuilt on the host"""
        t_wall = time.perf_counter()
        rebuild_s, train_s, logs = 0.0, 0.0, []
        for tr, te, _, _ in folds:
            t = time.perf_counter()
            d_in, d_out = E.DMatrix(X[tr], label=y[tr]), E.DMatrix(X[te], label=y[te])
            rebuild_s += time.perf_counter() - t
            timer, log = RoundTimer(), {}
            E.train(params, d_in, R, evals=[(d_in, "train"), (d_out, "test")], evals_result=log, verbose_eval=False,
                    callbacks=[timer])
            train_s += timer.t1 - timer.t0
            logs.append(log)
            del d_in, d_out
        wall = time.perf_counter() - t_wall
        want = {}
        for data in ("train", "test"):
            for metric in logs[0][data]:
                vals = np.array([lg[data][metric] for lg in logs])
                want["%s-%s-mean" % (data, metric)] = [float(np.mean(vals[:, r])) for r in range(R)]
                want["%s-%s-std" % (data, metric)] = [float(np.std(vals[:, r])) for r in range(R)]
        return want, {"wall_s": wall, "host_rebuild_s": rebuild_s, "fold_rounds_per_s": K * R / train_s}

    arms = {"cv": [], "loop": []}
    agree = True
    for _ in range(args.repeats):   # the arms alternate, so that drift of the shared host touches both alike
        got, a = run_cv()
        want, b = run_loop()
        arms["cv"].append(a)
        arms["loop"].append(b)
        agree = agree and got == want
    res = {"metric": "k-fold cross-validation: cv() with device slices vs a train() loop on host-built folds",
           "card": card(), "config": "C3 synthetic %dx%d depth %d 256 bins, %d folds, %d rounds, 1 GPU"
           % (args.rows, cols, depth, K, R),
           "repeats": args.repeats, "cv": arms["cv"], "loop": arms["loop"], "agree": agree,
           "final_test_rmse_mean": got["test-rmse-mean"][-1]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
