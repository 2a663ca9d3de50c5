#!/usr/bin/env python
"""bench_sparse_native.py -- quantisation, evaluation and prediction of CSR matrices at the cost of their stored entries.
One JSON line.

    python bench_sparse_native.py [--rounds 20] [--skip q5k,q20k,s1,wide,big] [--profile]

q5k / q20k  20M x 5,000 at 0.1 % and 20M x 20,000 at 0.025 % density (the same 100M entries): quantisation seconds and
            the sketch's share of them, 1 - (quantisation with the cuts given, which bins only) / (with the sketch).
s1          bench.py's C3 generator (10M x 100) with 90 % and 99 % of the entries dropped (bench_sparse.py's S1), CSR
            input: rounds/s with a 1M-row CSR evaluation set evaluated every round, and predict rows/s on it.
wide        10M x 20,000 at 0.05 % with a 1M-row evaluation set (depth 6): rounds/s with evaluation, predict rows/s.
big         A model of 1,000 trees of depth 8 (trained on 200,000 rows of S1 at 10 %), predicting 1M rows of S1 at 10 %:
            the case where a walk makes the most lookups per row (8,000 node visits against 10 stored entries).
Every workload reports its model's sha256, which must not depend on the code version.  --profile adds the CUDA kernel
times of one q5k quantisation and one s1 prediction (torch.profiler, in a run of their own after the timed ones) with
the bytes the entry pass and the CSR walk must move.  The card's name and power limit are read in the same run.
Writes nothing to the tree."""
import argparse
import gc
import hashlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_sparse import card, drop_to_csr  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def bernoulli_csr(n, f, density, seed):
    """n x f CSR whose cells are stored independently with probability `density` (geometric gaps between the stored
    cells of the flattened matrix: no sort, no duplicates), values U[0, 10), label from a sparse linear model"""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    cells = n * f
    pos = np.cumsum(rng.geometric(density, size=int(cells * density * 1.05) + 1024)) - 1
    pos = pos[pos < cells]
    rows = pos // f
    indptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(rows, minlength=n), out=indptr[1:])
    X = sp.csr_matrix((rng.random(pos.size, dtype=np.float32) * np.float32(10.0), (pos % f).astype(np.int32), indptr),
                      shape=(n, f))
    a = rng.normal(size=f).astype(np.float32)
    y = (X @ a + rng.normal(scale=0.1, size=n)).astype(np.float32)
    return X, y


def sha(bst):
    return hashlib.sha256(bytes(bst.save_raw())).hexdigest()


def quantise(E, X, y):
    dm = E.DMatrix(X, label=y)
    t = time.perf_counter()
    dm._ensure_quantized(256)
    q = time.perf_counter() - t
    cuts = dm.get_cuts()
    del dm
    d2 = E.DMatrix(X, label=y)
    t = time.perf_counter()
    d2._ensure_quantized(256, cuts=cuts)
    b = time.perf_counter() - t
    del d2
    gc.collect()
    return {"nnz": int(X.nnz), "quantise_s": round(q, 3), "bin_only_s": round(b, 3), "sketch_share": round(1 - b / q, 4),
            "cuts_sha256": hashlib.sha256(b"".join(np.ascontiguousarray(c).tobytes() for c in cuts)).hexdigest()}


def train_eval_predict(E, params, X, y, Xe, ye, rounds):
    dm = E.DMatrix(X, label=y)
    dm._ensure_quantized(256)
    de = E.DMatrix(Xe, label=ye)
    E.train(params, dm, 2, evals=[(de, "eval")], verbose_eval=False)   # warm-up; quantises de
    res = {}
    t = time.perf_counter()
    bst = E.train(params, dm, rounds, evals=[(de, "eval")], evals_result=res, verbose_eval=False)
    rps = rounds / (time.perf_counter() - t)
    return bst, {"rounds_per_s_with_eval": round(rps, 3), "predict_rows_per_s": predict_rate(E, bst, Xe),
                 "model_sha256": sha(bst), "eval_log_sha256": hashlib.sha256(json.dumps(res).encode()).hexdigest()}


def predict_rate(E, bst, Xe, repeats=3):
    dp = E.DMatrix(Xe)
    bst.predict(dp)
    t = time.perf_counter()
    for _ in range(repeats):
        p = bst.predict(dp)
    return {"rows_per_s": round(repeats * Xe.shape[0] / (time.perf_counter() - t)),
            "pred_sha256": hashlib.sha256(np.ascontiguousarray(p).tobytes()).hexdigest()}


def kernel_profile(E, fn):
    """{kernel name: (calls, total ms)} of the CUDA kernels fn launches"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0)
        if t > 0:
            out[ev.key[:120]] = {"calls": ev.count, "ms": round(t / 1000.0, 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--skip", default="")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    skip = set(s for s in args.skip.split(",") if s)
    import bench
    from xgboost_ray_b200 import engine as E
    out = {"card": card()}
    if "q5k" not in skip:
        X, y = bernoulli_csr(20_000_000, 5_000, 0.001, 1)
        out["q5k"] = quantise(E, X, y)
        if args.profile:
            dm = E.DMatrix(X, label=y)
            prof = kernel_profile(E, lambda: dm._ensure_quantized(256))
            out["q5k"]["kernels"] = {k: v for k, v in prof.items() if v["ms"] >= 0.5}
            out["q5k"]["entry_pass_bytes"] = int(16 * X.nnz + 16 * X.shape[0])   # indices, values, key in / key out, indptr
            del dm
        del X, y
        gc.collect()
    if "q20k" not in skip:
        X, y = bernoulli_csr(20_000_000, 20_000, 0.00025, 2)
        out["q20k"] = quantise(E, X, y)
        del X, y
        gc.collect()
    c3 = bench.WORKLOADS["C3"]
    p3 = dict(bench.PARAMS, max_depth=c3["depth"], base_score=0.5)
    if "s1" not in skip or "big" not in skip:
        X, y = bench.synth_shard(10_000_000, c3["cols"], 0, 1, workload="C3")
        for drop in (0.9, 0.99):
            csr, _ = drop_to_csr(X, drop, seed=7)
            key = "s1_drop_%d" % round(drop * 100)
            ne = 1_000_000
            if "s1" not in skip:
                bst, r = train_eval_predict(E, p3, csr, y, csr[:ne], y[:ne], args.rounds)
                out[key] = dict(r, nnz=int(csr.nnz))
                if args.profile and drop == 0.9:
                    dp = E.DMatrix(csr[:ne])
                    bst.predict(dp)
                    prof = kernel_profile(E, lambda: bst.predict(dp))
                    out[key]["kernels"] = {k: v for k, v in prof.items() if v["ms"] >= 0.05}
                    sub = csr[:ne]
                    out[key]["walk_min_bytes"] = int(8 * sub.nnz + 8 * (ne + 1) + 4 * ne)   # entries, indptr, margins
            if "big" not in skip and drop == 0.9:
                big = E.train(dict(p3, eta=0.05), E.DMatrix(csr[:200_000], label=y[:200_000]), 1000, verbose_eval=False)
                out["big_1000x8_s1_drop_90"] = dict(predict_rate(E, big, csr[:ne]), model_sha256=sha(big))
                del big
            del csr
            gc.collect()
        del X, y
        gc.collect()
    if "wide" not in skip:
        X, y = bernoulli_csr(10_000_000, 20_000, 0.0005, 3)
        Xe, ye = bernoulli_csr(1_000_000, 20_000, 0.0005, 4)
        _, r = train_eval_predict(E, dict(p3, max_depth=6), X, y, Xe, ye, args.rounds)
        out["wide_10M_x_20k"] = dict(r, nnz=int(X.nnz))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
