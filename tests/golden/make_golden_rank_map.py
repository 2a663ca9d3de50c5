"""Generates tests/golden/rank_map_binary_groups.json: a rank:map model grown by the CPU oracle from the gradients of
tests/rank_map_reference.py.  The CPU suite checks that it is still reproduced, the GPU suite checks the CUDA path
against it.  Loaded by name: the other golden tests do not see it.
Run:  python tests/golden/make_golden_rank_map.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import oracle as O  # noqa: E402
from tests import rank_map_reference as M  # noqa: E402
from tests import ranking_reference as R  # noqa: E402

CASES = ["rank_map_binary_groups"]


def case_data(name):
    """(x, label, qid, params, rounds)."""
    if name == "rank_map_binary_groups":
        # groups of 1, 2, 3, 37 and 90 rows and one of 2500 (larger than the gradient kernel's shared-memory stage),
        # binary labels with about a quarter hits, groups without hits and groups of hits only, missing values
        rng = np.random.RandomState(31)
        sizes = [1, 2, 3, 37, 90] * 8 + [2500]
        qid = np.repeat(np.arange(len(sizes)), sizes)
        n = len(qid)
        x = rng.uniform(0, 4, size=(n, 7)).astype(np.float32)
        y = (x[:, 0] + 0.8 * rng.normal(size=n) > 3.0).astype(np.float32)
        ptr = R.group_ptr(qid)
        y[ptr[3]:ptr[4]] = 0.0                                 # a 37-row group without hits
        y[ptr[9]:ptr[10]] = 1.0                                # a 90-row group of hits only
        x[rng.uniform(size=x.shape) < 0.08] = np.nan
        return x, y, qid, {"objective": "rank:map", "max_depth": 5, "eta": 0.3, "lambdarank_num_pair_per_sample": 16}, 4
    raise KeyError(name)


def run_case(name):
    x, y, qid, params, rounds = case_data(name)
    model = M.train(O, params, x, y, qid, rounds)
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
