"""Generates tests/golden/{aft_normal_censored,aft_extreme_scale}.json: survival:aft models grown by the CPU oracle from
the gradients of tests/survival_reference.py.  The CPU suite checks that they are still reproduced, the GPU suite checks
the CUDA path against them.  Loaded by name: the other golden tests do not see them.
Run:  python tests/golden/make_golden_survival.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import oracle as O  # noqa: E402
from tests import survival_reference as S  # noqa: E402

CASES = ["aft_normal_censored", "aft_extreme_scale"]


def case_data(name):
    """(x, lower, upper, weight, params, rounds)."""
    if name == "aft_normal_censored":
        # all four censoring kinds (row mod 4: exact, right, left, interval), weights and missing values
        rng = np.random.RandomState(11)
        n = 3000
        x = rng.uniform(0, 4, size=(n, 8)).astype(np.float32)
        t = np.exp(0.4 * x[:, 0] - 0.3 * x[:, 1] + 0.3 * rng.normal(size=n)).astype(np.float32)
        lo, hi = t.copy(), t.copy()
        k = np.arange(n) % 4
        hi[k == 1] = np.inf
        lo[k == 2] = 0.0
        hi[k == 3] = t[k == 3] * np.float32(1.5)
        x[rng.uniform(size=x.shape) < 0.08] = np.nan
        w = rng.uniform(0.5, 2.0, size=n).astype(np.float32)
        return x, lo, hi, w, {"objective": "survival:aft", "max_depth": 5, "eta": 0.3}, 4
    if name == "aft_extreme_scale":
        rng = np.random.RandomState(12)
        n = 3000
        x = rng.uniform(0, 4, size=(n, 6)).astype(np.float32)
        t = np.exp(0.5 * x[:, 0] - 0.2 * x[:, 2] + 0.5 * rng.gumbel(size=n)).astype(np.float32)
        lo, hi = t.copy(), t.copy()
        hi[::3] = np.inf
        return x, lo, hi, None, {"objective": "survival:aft", "aft_loss_distribution": "extreme",
                                 "aft_loss_distribution_scale": 0.7, "max_depth": 4, "eta": 0.3}, 4
    raise KeyError(name)


def run_case(name):
    x, lo, hi, w, params, rounds = case_data(name)
    model = S.train(O, params, x, lo, hi, rounds, weight=w)
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
