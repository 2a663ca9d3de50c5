#!/usr/bin/env python
"""bench_sparse_bins.py -- the CSR bin layout (one bin byte per stored entry) against the dense one.  One JSON line.

    python bench_sparse_bins.py [--rounds 20] [--no-b]

(a) 8M x 2,500 at 0.1 % density, bin_layout "dense" and "csr": quantise seconds, rounds/s (depth 6, eta 0.3,
    hist_qbits default) and B2_MatrixDeviceBytes after quantisation without keep_raw; the two models' sha256 must match.
(b) 20M x 5,000 at 0.1 % density: its dense bins (200 GB) do not fit the card, so only "csr" runs ("auto" picks it).
    The same three numbers, and the sketch's share of quantisation: 1 - (quantisation with the cuts given, which bins
    only) / (quantisation with the sketch).
The card's name and power limit are read in the same run.  Writes nothing to the tree."""
import argparse
import gc
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_sparse import card, random_csr  # noqa: E402

PARAMS = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5}


def run(E, X, y, layout, rounds, cuts_timing=False):
    dm = E.DMatrix(X, label=y, bin_layout=layout)
    t = time.perf_counter()
    dm._ensure_quantized(256)
    quant_s = time.perf_counter() - t
    out = {"layout": layout, "quantise_s": round(quant_s, 3), "device_bytes_quantised": dm.device_bytes()}
    if cuts_timing:
        cuts = dm.get_cuts()
        d2 = E.DMatrix(X, label=y, bin_layout=layout)
        t = time.perf_counter()
        d2._ensure_quantized(256, cuts=cuts)
        bin_s = time.perf_counter() - t
        del d2
        out["bin_only_s"] = round(bin_s, 3)
        out["sketch_share_of_quantise"] = round(1.0 - bin_s / quant_s, 3)
    E.train(PARAMS, dm, 2, verbose_eval=False)                        # warm-up (graphs, pools)
    t = time.perf_counter()
    bst = E.train(PARAMS, dm, rounds, verbose_eval=False)
    out["rounds_per_s"] = round(rounds / (time.perf_counter() - t), 3)
    out["model_sha256"] = hashlib.sha256(bytes(bst.save_raw())).hexdigest()
    del bst, dm
    gc.collect()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--no-b", action="store_true")
    args = ap.parse_args()
    from xgboost_ray_b200 import engine as E
    if E.device_count() < 1:
        raise SystemExit("bench_sparse_bins.py needs a GPU")
    res = {"card": card(), "rounds": args.rounds, "params": PARAMS}
    X, y = random_csr(8_000_000, 2_500, 0.001, 1)
    res["a_8M_x_2500"] = {"nnz": int(X.nnz), "dense": run(E, X, y, "dense", args.rounds),
                          "csr": run(E, X, y, "csr", args.rounds)}
    res["a_8M_x_2500"]["same_model"] = (res["a_8M_x_2500"]["dense"]["model_sha256"] ==
                                        res["a_8M_x_2500"]["csr"]["model_sha256"])
    del X, y
    gc.collect()
    if not args.no_b:
        X, y = random_csr(20_000_000, 5_000, 0.001, 2)
        res["b_20M_x_5000"] = {"nnz": int(X.nnz), "csr": run(E, X, y, "auto", args.rounds, cuts_timing=True)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
