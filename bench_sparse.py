#!/usr/bin/env python
"""bench_sparse.py -- scipy.sparse (CSR) input against its dense twin, and the two CSR kernels.  One JSON line.

    python bench_sparse.py [--rows 10000000] [--rounds 100] [--s2-rows 8000000] [--no-s2]

S1  bench.py's C3 generator (10M x 100) with 90 % and 99 % of the entries dropped by a seeded mask.  The CSR and its
    dense twin (NaN in every dropped cell) are each quantised, trained for --rounds rounds with C3's parameters, once
    with a CSR (or twin) evaluation set of 1M rows evaluated every round, and predicted.  Reported per input: quantise
    seconds, rounds/s without and with the evaluation set, predict rows/s, B2_MatrixDeviceBytes before and after
    quantisation (without keep_raw) and the model's sha256 (the CSR and the twin must give the same model).
S2  8M x 2,500 at 0.1 % density: the twin (80 GB) does not fit on the card, so only the CSR runs (depth 6).
Kernel time of csr_densify_kernel (one tile) from CUDA events, with the bytes the algorithm moves (4 rows F written,
8 per entry and 8 per row read) over the time against the 3.35 TB/s HBM3 bandwidth of the H100 SXM data sheet: the
kernel is memory-bound (no arithmetic).  The sketch's entry pass is measured by bench_sparse_native.py.
The card's name and power limit are read in the same run.  Writes nothing to the tree."""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers are still worth printing, marked as unattributed
        return "unknown (%s)" % e


def drop_to_csr(X, drop, seed):
    """(CSR of X without the dropped cells, dense twin with NaN there); the mask is drawn block by block."""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    parts, twin = [], np.empty_like(X)
    for r0 in range(0, X.shape[0], 1_000_000):
        blk = X[r0:r0 + 1_000_000]
        keep = rng.random(blk.shape, dtype=np.float32) >= np.float32(drop)
        counts = keep.sum(axis=1)
        indptr = np.zeros(blk.shape[0] + 1, np.int64)
        np.cumsum(counts, out=indptr[1:])
        parts.append(sp.csr_matrix((blk[keep], np.nonzero(keep)[1].astype(np.int32), indptr), shape=blk.shape))
        twin[r0:r0 + 1_000_000] = np.where(keep, blk, np.nan)
    return sp.vstack(parts, format="csr"), twin


def random_csr(n, f, density, seed):
    """n x f CSR with about density n f entries, uniform values, and a label from a sparse linear model."""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    counts = rng.binomial(f, density, size=n)
    rows = np.repeat(np.arange(n, dtype=np.int64), counts)
    cols = rng.integers(0, f, size=rows.size, dtype=np.int64)
    key = np.unique(rows * f + cols)
    rows, cols = key // f, (key % f).astype(np.int32)
    vals = rng.random(key.size, dtype=np.float32) * np.float32(10.0)
    indptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(rows, minlength=n), out=indptr[1:])
    X = sp.csr_matrix((vals, cols, indptr), shape=(n, f))
    a = rng.normal(size=f).astype(np.float32)
    y = (X @ a + rng.normal(scale=0.1, size=n)).astype(np.float32)
    return X, y


def run_input(E, params, X, y, Xe, ye, rounds):
    """quantise seconds, rounds/s without / with the evaluation set, predict rows/s, device bytes, model sha256"""
    dm = E.DMatrix(X, label=y)
    raw_bytes = dm.device_bytes()
    t = time.perf_counter()
    dm._ensure_quantized(256)
    quant_s = time.perf_counter() - t
    E.train(params, dm, 2, verbose_eval=False)                        # warm-up (graphs, pools)
    t = time.perf_counter()
    bst = E.train(params, dm, rounds, verbose_eval=False)
    rps = rounds / (time.perf_counter() - t)
    de = E.DMatrix(Xe, label=ye)
    de._ensure_quantized(256)
    res = {}
    t = time.perf_counter()
    E.train(params, dm, rounds, evals=[(de, "eval")], evals_result=res, verbose_eval=False)
    rps_eval = rounds / (time.perf_counter() - t)
    dp = E.DMatrix(Xe)
    bst.predict(dp)
    t = time.perf_counter()
    bst.predict(dp)
    pred_rps = Xe.shape[0] / (time.perf_counter() - t)
    return {"quantise_s": round(quant_s, 4), "rounds_per_s": round(rps, 3), "rounds_per_s_with_eval": round(rps_eval, 3),
            "predict_rows_per_s": round(pred_rps), "device_bytes_before_quantise": raw_bytes,
            "device_bytes_quantised": dm.device_bytes(),
            "model_sha256": hashlib.sha256(bytes(bst.save_raw())).hexdigest()}


def kernel_times(E, X, repeats=20):
    """CUDA-event time of one densified tile of the CSR X (indptr / indices / values on the device)."""
    import torch
    lib = E.lib()
    c = E.canonical_csr(X)
    n, F = c.shape
    dev = torch.device("cuda", 0)
    ip = torch.from_numpy(c.indptr).to(dev)
    ix = torch.from_numpy(c.indices).to(dev)
    vs = torch.from_numpy(c.values).to(dev)
    rows = min(E.raw_tile_rows(F), n)
    tile = torch.empty(rows * F, dtype=torch.float32, device=dev)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    vp = C.c_void_p
    lib.b2_launch_csr_densify.argtypes = [vp, vp, vp, C.c_int64, C.c_int64, C.c_int, vp, C.c_int, vp]
    lib.b2_launch_csr_densify.restype = C.c_int
    stream = torch.cuda.current_stream().cuda_stream

    def densify():
        return lib.b2_launch_csr_densify(ip.data_ptr(), ix.data_ptr(), vs.data_ptr(), 0, rows, F, tile.data_ptr(), sms, stream)

    out = {}
    for name, fn, written_rows, width in (("csr_densify_kernel", densify, rows, F),):
        assert fn() == 0
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(repeats):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / repeats
        ind = c.indices[: c.indptr[written_rows]]
        entries = int(ind.size)
        nbytes = 4 * written_rows * width + 8 * entries + 8 * written_rows
        out[name] = {"rows": int(written_rows), "nf": int(width), "entries": entries, "ms": round(ms, 4),
                     "bytes": nbytes, "GBps": round(nbytes / ms / 1e6, 1),
                     "share_of_hbm_peak": round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3), "bound": "memory"}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--eval-rows", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=100)
    ap.add_argument("--s2-rows", type=int, default=8_000_000)
    ap.add_argument("--s2-rounds", type=int, default=20)
    ap.add_argument("--no-s2", action="store_true")
    args = ap.parse_args()
    import bench
    from xgboost_ray_b200 import engine as E
    info = card()
    c3 = bench.WORKLOADS["C3"]
    params = dict(bench.PARAMS, max_depth=c3["depth"], base_score=0.5)
    X, y = bench.synth_shard(args.rows, c3["cols"], 0, 1, workload="C3")
    out = {"card": info, "S1": {}}
    kt = {}
    for drop in (0.9, 0.99):
        csr, twin = drop_to_csr(X, drop, seed=7)
        ne = min(args.eval_rows, args.rows)
        r = {"nnz": int(csr.nnz)}
        r["csr"] = run_input(E, params, csr, y, csr[:ne], y[:ne], args.rounds)
        r["twin"] = run_input(E, params, twin, y, twin[:ne], y[:ne], args.rounds)
        r["same_model"] = r["csr"]["model_sha256"] == r["twin"]["model_sha256"]
        out["S1"]["drop_%d" % round(drop * 100)] = r
        if drop == 0.99:
            kt["S1_drop_99"] = kernel_times(E, csr)
        del csr, twin
    del X, y
    if not args.no_s2:
        Xs, ys = random_csr(args.s2_rows, 2500, 0.001, seed=11)
        p2 = dict(params, max_depth=6)
        ne = min(args.eval_rows, args.s2_rows)
        out["S2"] = dict(run_input(E, p2, Xs, ys, Xs[:ne], ys[:ne], args.s2_rounds), nnz=int(Xs.nnz),
                         dense_twin_bytes=4 * args.s2_rows * 2500)
        kt["S2"] = kernel_times(E, Xs)
    out["kernels"] = kt
    print(json.dumps(out))


if __name__ == "__main__":
    main()
