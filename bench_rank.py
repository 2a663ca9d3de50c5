#!/usr/bin/env python
"""bench_rank.py -- rank:map next to rank:ndcg on one GPU: boosting rounds/sec, the LambdaMART gradient kernel alone,
and a tree-for-tree check against the CPU oracle.

    python bench_rank.py [--steps K] [--warmup W] [--repeats R] [--rows N] [--launches L] [--no-parity]

Data: bench.py's C3 matrix (10M x 100, x ~ U[0, 10)) with the query groups qid = row // 100 (100k groups of 100 rows)
and the binary label [y > quantile(y, 0.8)], for both objectives (rank:ndcg reads it as relevance 0 / 1).
- rounds/s: the matrix quantised and resident in HBM, W untimed rounds, then K timed rounds ending in a device
  synchronise; the arms alternate R times.
- gradient kernel: b2_launch_lambdarank_gradient of every mode (pairwise, ndcg, map) on the same groups, the model
  order taken once from a fixed random margin; CUDA events around L back-to-back launches after 3 untimed ones.
- parity: a 200k-row, 3-round sub-problem per objective compared tree for tree with the CPU oracle grown from the
  gradients of the tests' references (split feature / bin / default direction exact, leaf values within 1e-5).
The card's name and power limit are read in the same run.  Prints one JSON line.  Writes nothing to the tree."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

ARMS = ("rank:ndcg", "rank:map")
MODES = {"pairwise": 0, "ndcg": 1, "map": 2}
GROUP = 100


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers are still worth printing, marked as unattributed
        return "unknown (%s)" % e


def labels(y):
    return (y > np.quantile(y, 0.8)).astype(np.float32)


def rounds_per_s(E, dm, params, args):
    bst = E.Booster(params, cache=[dm])
    for r in range(args.warmup):
        bst.update(dm, r)
    bst.get_trees()
    t0 = time.perf_counter()
    for r in range(args.steps):
        bst.update(dm, args.warmup + r)
    bst.get_trees()                               # waits for the last enqueued round
    rate = args.steps / (time.perf_counter() - t0)
    metric = bst.eval_set([(dm, "train")], 0).split("\t", 1)[-1]
    return rate, metric


def kernel_ms(E, y, k, launches):
    """Milliseconds per launch of the gradient kernel of each mode, CUDA events over `launches` launches."""
    import torch
    L = E.lib()
    dev = torch.device("cuda")
    n = len(y)
    ng = n // GROUP
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    stream = torch.cuda.current_stream().cuda_stream
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    gptr = torch.arange(0, n + 1, GROUP, dtype=torch.int64, device=dev)
    label = torch.from_numpy(y).to(dev)
    margin = torch.from_numpy(np.random.RandomState(5).normal(size=n).astype(np.float32)).to(dev)
    iota, rows = (torch.empty(n, dtype=torch.int32, device=dev) for _ in range(2))
    keys, skeys, lkeys, lrows = (torch.empty(n, dtype=torch.int32, device=dev) for _ in range(4))
    L.b2_rank_order_temp_bytes.restype = C.c_size_t
    tb = L.b2_rank_order_temp_bytes(C.c_int64(n), C.c_int64(ng))
    temp = torch.empty(max(int(tb), 1), dtype=torch.uint8, device=dev)
    disc = torch.empty(GROUP, dtype=torch.float64, device=dev)
    inv = torch.empty(ng, dtype=torch.float64, device=dev)
    gh = torch.empty(2 * n, dtype=torch.float32, device=dev)
    absmax = torch.zeros(2, dtype=torch.int32, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    S = C.c_void_p(stream)

    def ok(rc, what):
        if rc != 0:
            raise RuntimeError("%s failed with CUDA error %d" % (what, rc))

    ok(L.b2_launch_rank_iota(p(iota), C.c_int64(n), sms, S), "iota")
    for v, ko, ro in ((margin, skeys, rows), (label, lkeys, lrows)):
        ok(L.b2_rank_order(p(v), C.c_int64(n), p(gptr), C.c_int64(ng), p(iota), p(keys), p(ko), p(ro), p(temp),
                           C.c_size_t(tb), sms, S), "b2_rank_order")
    ok(L.b2_launch_rank_disc(p(disc), C.c_int64(GROUP), sms, S), "disc")
    ok(L.b2_launch_rank_inv_idcg(p(gptr), C.c_int64(ng), p(lkeys), p(disc), k, 1, p(inv), sms, S), "inv_idcg")
    null = C.c_void_p(0)
    out = {}
    for name, mode in MODES.items():
        def launch():
            ok(L.b2_launch_lambdarank_gradient(mode, p(gptr), C.c_int64(ng), C.c_int64(GROUP), p(skeys), p(rows),
                                               p(label), p(inv), p(disc), k, 1, null, null, null, null, null, p(gh),
                                               p(absmax), p(err), sms, S), "lambdarank gradient")
        for _ in range(3):
            launch()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            launch()
        b.record()
        torch.cuda.synchronize()
        out[name] = a.elapsed_time(b) / launches
    return out


def oracle_match(E, params, X, y):
    from oracle import oracle as O
    from tests import rank_map_reference as RM
    from tests import ranking_reference as RR
    qid = np.arange(len(y)) // GROUP
    b = E.train(params, E.DMatrix(X, label=y, qid=qid), num_boost_round=3, verbose_eval=False)
    ob = (RM if params["objective"] == RM.MAP_OBJECTIVE else RR).train(O, params, X, y, qid, 3)
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
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()
    import bench
    from xgboost_ray_b200 import engine as E
    cols, depth = bench.WORKLOADS["C3"]["cols"], bench.WORKLOADS["C3"]["depth"]
    base = dict(bench.PARAMS, max_depth=depth)
    base.pop("base_score")                       # the rank objectives' own default, 0.5
    k = 32
    res = {"metric": "rank:map vs rank:ndcg: rounds/s and gradient-kernel ms", "card": card(),
           "config": "C3 synthetic %dx%d depth %d, qid = row // %d, label [y > q80(y)], 1 GPU"
                     % (args.rows, cols, depth, GROUP),
           "steps": args.steps, "warmup": args.warmup, "repeats": args.repeats}
    X, y0 = bench.synth_shard(args.rows, cols, 0, 1, workload="C3")
    y = labels(y0)
    dm = E.DMatrix(X, label=y, qid=np.arange(len(y)) // GROUP)
    dm._ensure_quantized(256)
    rates = {a: [] for a in ARMS}
    metrics = {}
    for _ in range(args.repeats):
        for a in ARMS:
            r, m = rounds_per_s(E, dm, dict(base, objective=a), args)
            rates[a].append(r)
            metrics[a] = m
    res["rounds_per_s"] = rates
    res["final_train_metric"] = metrics
    del dm, X
    res["gradient_kernel_ms"] = dict(kernel_ms(E, y, k, args.launches), groups=len(y) // GROUP, group_rows=GROUP, k=k,
                                     launches=args.launches)
    if not args.no_parity:
        n_sub = min(200_000, args.rows)
        Xs, ys0 = bench.synth_shard(n_sub, cols, 0, 1, workload="C3")
        ys = labels(ys0)
        res["oracle"] = {}
        for a in ARMS:
            match, worst = oracle_match(E, dict(base, objective=a, profile=0), Xs, ys)
            res["oracle"][a] = {"rows": n_sub, "rounds": 3, "match": match, "max_leaf_diff": worst}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
