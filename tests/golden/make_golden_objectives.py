"""Generates tests/golden/{poisson_weighted_missing,tweedie_regression}.json: models of the objectives beyond squared
error / logistic / softmax, grown by the CPU oracle from the gradients of tests/objective_reference.py.  The CPU suite
checks that they are still reproduced, the GPU suite checks the CUDA path against them.
Run:  python tests/golden/make_golden_objectives.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import oracle as O  # noqa: E402
from tests import objective_reference as R  # noqa: E402

CASES = ["poisson_weighted_missing", "tweedie_regression"]


def case_data(name):
    if name == "poisson_weighted_missing":
        # counts with sample weights and missing values; base_score estimated from the labels
        rng = np.random.RandomState(5)
        n = 3000
        x = rng.uniform(0, 4, size=(n, 8)).astype(np.float32)
        y = rng.poisson(np.exp(0.4 * x[:, 0] - 0.3 * x[:, 1] + 0.2 * np.round(x[:, 2]))).astype(np.float32)
        x[rng.uniform(size=x.shape) < 0.08] = np.nan
        w = rng.uniform(0.5, 2.0, size=n).astype(np.float32)
        return x, y, w, {"objective": "count:poisson", "max_depth": 5, "eta": 0.3}, 4
    if name == "tweedie_regression":
        # compound Poisson-gamma claims: exact zeros and positive amounts
        rng = np.random.RandomState(9)
        n = 3000
        x = rng.uniform(0, 4, size=(n, 6)).astype(np.float32)
        counts = rng.poisson(np.exp(0.3 * x[:, 0] - 0.5))
        y = np.array([rng.gamma(2.0, 1.5, size=c).sum() for c in counts], np.float32)
        return x, y, None, {"objective": "reg:tweedie", "tweedie_variance_power": 1.3, "max_depth": 4, "eta": 0.3,
                            "base_score": 1.0}, 4
    raise KeyError(name)


def run_case(name):
    x, y, w, params, rounds = case_data(name)
    model = R.train(O, params, x, y, rounds, weight=w)
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
