#!/usr/bin/env python
"""bench_model_io.py -- model file size and save / load time of the JSON and UBJSON formats for a large model.

    python bench_model_io.py [--rows N] [--depth D] [--nodes M] [--predict-rows P] [--repeats K]

Trains bench.py's C3 matrix (10M x 100) at depth 14 one round at a time until the model holds at least --nodes nodes
(1M by default), then reports for each format:
- bytes: the size of save_raw(format);
- save_s: save_raw(format) from a model whose per-tree conversion cache is empty (what the first save of a freshly
  trained or loaded model costs), and save_warm_s with the cache filled (what a later checkpoint costs);
- load_s: Booster.load_model of those bytes;
- file_predict_s: Booster(model_file=path) followed by one predict on --predict-rows rows, which ends with the
  prediction copied to the host (so the device is synchronised).
Every time is the median of --repeats repeats, with the two formats alternating.  These are host timings of host work,
except the one device predict.  `agree` says both formats loaded to the same JSON bytes and predictions.  The card's
name and power limit are read in the same run.  The model files go to a temporary directory; nothing is written to the
tree."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

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
    ap.add_argument("--depth", type=int, default=14)
    ap.add_argument("--nodes", type=int, default=1_000_000)
    ap.add_argument("--predict-rows", type=int, default=1_000_000)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import bench
    from xgboost_ray_b200 import engine as E
    if E.device_count() < 1:
        raise SystemExit("bench_model_io.py needs a CUDA device")
    cols = bench.WORKLOADS["C3"]["cols"]
    X, y = bench.synth_shard(args.rows, cols, 0, 1, workload="C3")
    params = dict(bench.PARAMS, max_depth=args.depth, objective="reg:squarederror", base_score=0.5)
    dtrain = E.DMatrix(X, label=y)
    del X
    t = time.perf_counter()
    bst = E.train(params, dtrain, 1, verbose_eval=False)
    rounds = 1
    nodes = sum(len(tr["left"]) for tr in bst.get_trees())
    while nodes < args.nodes:
        bst.update(dtrain, rounds)
        rounds += 1
        nodes = sum(len(tr["left"]) for tr in bst.get_trees())
    train_s = time.perf_counter() - t
    del dtrain
    Xp, _ = bench.synth_shard(args.predict_rows, cols, 0, 1, workload="C3")
    dpred = E.DMatrix(Xp)
    bst.predict(dpred)   # the prediction path's first launch and the raw values' upload are not timed

    fmts = ("json", "ubj")
    times = {f: {"save_s": [], "save_warm_s": [], "load_s": [], "file_predict_s": []} for f in fmts}
    raw, loaded_json, preds = {}, {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(args.repeats):
            for f in fmts:
                bst.__dict__.pop("_tree_json_cache", None)
                t = time.perf_counter()
                raw[f] = bytes(bst.save_raw(f))
                times[f]["save_s"].append(time.perf_counter() - t)
                t = time.perf_counter()
                bst.save_raw(f)
                times[f]["save_warm_s"].append(time.perf_counter() - t)
                b = E.Booster()
                t = time.perf_counter()
                b.load_model(raw[f])
                times[f]["load_s"].append(time.perf_counter() - t)
                loaded_json[f] = bytes(b.save_raw())
                path = os.path.join(tmp, "model." + f)
                with open(path, "wb") as fh:
                    fh.write(raw[f])
                t = time.perf_counter()
                preds[f] = E.Booster(model_file=path).predict(dpred)
                times[f]["file_predict_s"].append(time.perf_counter() - t)
    agree = loaded_json["json"] == loaded_json["ubj"] and \
        preds["json"].tobytes() == preds["ubj"].tobytes() == bst.predict(dpred).tobytes()
    res = {"metric": "model file size and save / load time, JSON vs UBJSON", "card": card(),
           "config": "C3 synthetic %dx%d depth %d, %d rounds, %d nodes; predict on %d rows"
           % (args.rows, cols, args.depth, rounds, nodes, args.predict_rows),
           "train_s": train_s, "repeats": args.repeats, "agree": agree}
    for f in fmts:
        res[f] = dict({k: statistics.median(v) for k, v in times[f].items()}, bytes=len(raw[f]))
    res["json_over_ubj_bytes"] = len(raw["json"]) / len(raw["ubj"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
