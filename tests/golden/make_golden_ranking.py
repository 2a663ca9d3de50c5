"""Generates tests/golden/{rank_ndcg_mixed_groups,rank_pairwise_linear_k5}.json: rank:ndcg / rank:pairwise models grown
by the CPU oracle from the gradients of tests/ranking_reference.py.  The CPU suite checks that they are still reproduced,
the GPU suite checks the CUDA path against them.  Loaded by name: the other golden tests do not see them.
Run:  python tests/golden/make_golden_ranking.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import oracle as O  # noqa: E402
from tests import ranking_reference as R  # noqa: E402

CASES = ["rank_ndcg_mixed_groups", "rank_pairwise_linear_k5"]


def case_data(name):
    """(x, label, qid, params, rounds)."""
    if name == "rank_ndcg_mixed_groups":
        # groups of 1, 2, 3 and 37 rows and one of 2500 (larger than the gradient kernel's shared-memory stage),
        # integer labels 0-4 and missing values
        rng = np.random.RandomState(21)
        sizes = [1, 2, 3, 37] * 10 + [2500]
        qid = np.repeat(np.arange(len(sizes)), sizes)
        n = len(qid)
        x = rng.uniform(0, 4, size=(n, 7)).astype(np.float32)
        y = np.clip(np.floor(x[:, 0] + 0.6 * rng.normal(size=n)), 0, 4).astype(np.float32)
        x[rng.uniform(size=x.shape) < 0.08] = np.nan
        return x, y, qid, {"objective": "rank:ndcg", "max_depth": 5, "eta": 0.3}, 4
    if name == "rank_pairwise_linear_k5":
        rng = np.random.RandomState(22)
        sizes = rng.randint(1, 60, size=80)
        qid = np.repeat(np.arange(len(sizes)), sizes)
        n = len(qid)
        x = rng.uniform(0, 4, size=(n, 6)).astype(np.float32)
        y = np.clip(np.floor(1.5 * x[:, 1] - 0.5 * x[:, 3] + rng.normal(size=n)), 0, 6).astype(np.float32)
        return x, y, qid, {"objective": "rank:pairwise", "ndcg_exp_gain": False, "lambdarank_num_pair_per_sample": 5,
                           "max_depth": 4, "eta": 0.3}, 4
    raise KeyError(name)


def run_case(name):
    x, y, qid, params, rounds = case_data(name)
    model = R.train(O, params, x, y, qid, rounds)
    cuts = model.bst.cuts
    trees = [{k: [float(v) if k in ("split_cond", "value", "loss_chg") else int(v) for v in getattr(t, k)]
              for k in ("left", "right", "split_feature", "split_bin", "default_left", "split_cond", "value", "loss_chg")}
             for t in model.bst.trees()]
    pred = model.predict(x[:64])
    return {"name": name, "params": params, "rounds": rounds, "base_score": model.base_score,
            "cut_ptrs": [int(v) for v in cuts.ptrs], "cut_vals_bits": [int(v) for v in cuts.vals.view(np.uint32)],
            "min_vals_bits": [int(v) for v in cuts.mins.view(np.uint32)], "has_missing": [int(v) for v in cuts.has_missing],
            "trees": trees, "pred_head": [float(v) for v in np.asarray(pred, np.float64).reshape(-1)]}


if __name__ == "__main__":
    for name in CASES:
        out = run_case(name)
        with open(os.path.join(HERE, name + ".json"), "w") as f:
            json.dump(out, f)
        print(name, "trees", len(out["trees"]), "nodes", [len(t["left"]) for t in out["trees"]])
