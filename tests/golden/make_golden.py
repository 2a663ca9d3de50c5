"""Generates tests/golden/*.json from the CPU oracle (oracle/hist_oracle.c).

The reference cannot produce golden vectors for this path (its arithmetic lives in the absent
`xgboost` wheel; SURVEY.md 8c), so these fixtures pin the ORACLE's outputs: the -m "not gpu" suite
checks the oracle still reproduces them, the -m gpu suite checks the CUDA path against them without
executing the oracle.  Run:  python tests/golden/make_golden.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import oracle as O  # noqa: E402


def case_data(name):
    if name == "toy_softmax":
        x = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 1], [0, 0, 1, 0]] * 8, np.float32)
        y = np.array([0, 1, 2, 3] * 8, np.float32)
        return x, y, None, {"max_depth": 2, "objective": "multi:softmax", "num_class": 4}, 2
    if name == "breast_cancer_logistic":
        from sklearn.datasets import load_breast_cancer
        x, y = load_breast_cancer(return_X_y=True)
        return x.astype(np.float32), y.astype(np.float32), None, \
            {"objective": "binary:logistic", "max_depth": 6, "eta": 0.3, "base_score": 0.5}, 5
    if name == "synthetic_missing_regression":
        rng = np.random.RandomState(42)
        x = rng.uniform(0, 10, size=(3000, 10)).astype(np.float32)
        x[:, 3] = np.round(x[:, 3])
        x[rng.uniform(size=x.shape) < 0.1] = np.nan
        y = (np.nan_to_num(x[:, 0]) * 2 - np.nan_to_num(x[:, 3]) + rng.normal(size=3000)).astype(np.float32)
        w = rng.uniform(0.5, 1.5, size=3000).astype(np.float32)
        return x, y, w, {"objective": "reg:squarederror", "max_depth": 5, "eta": 0.3, "base_score": 0.5,
                         "min_child_weight": 2.0, "lambda": 0.5}, 4
    if name == "synthetic_categorical_softprob":
        # a miniature of BASELINE config C5: numeric + categorical columns (cardinalities 4/16/64/250), multi:softprob
        rng = np.random.RandomState(77)
        n = 4000
        xn = rng.uniform(0, 10, size=(n, 6))
        cards = (3, 4, 16, 64, 250)
        cats = np.column_stack([rng.randint(0, c, size=n) for c in cards])
        x = np.column_stack([xn, cats]).astype(np.float32)
        x[rng.uniform(size=x.shape) < 0.04] = np.nan
        score = (np.nan_to_num(x[:, 0]) > 5) * 1 + (np.nan_to_num(x[:, 6]) == 1) * 1 + (np.nan_to_num(x[:, 8]) % 3 == 0) * 1 \
            + (np.nan_to_num(x[:, 10]) % 7 < 2) * 1
        return x, score.astype(np.float32), None, \
            {"objective": "multi:softprob", "num_class": 5, "max_depth": 5, "eta": 0.3}, 3
    if name == "synthetic_softprob_k20_weighted_missing":
        # more classes than the engine's fused gradient path takes (16): unfused gradients, one absmax pass per class tree
        rng = np.random.RandomState(2020)
        x = rng.uniform(0, 10, size=(3000, 10)).astype(np.float32)
        x[rng.uniform(size=x.shape) < 0.1] = np.nan
        v = np.nan_to_num(x[:, 0]) * 2 + np.nan_to_num(x[:, 1]) * 0.7 + rng.normal(scale=0.5, size=3000)
        y = (np.floor(v) % 20).astype(np.float32)
        w = rng.uniform(0.5, 2.0, size=3000).astype(np.float32)
        return x, y, w, {"objective": "multi:softprob", "num_class": 20, "max_depth": 4, "eta": 0.3}, 2
    raise KeyError(name)


CASES = ["toy_softmax", "breast_cancer_logistic", "synthetic_missing_regression", "synthetic_categorical_softprob",
         "synthetic_softprob_k20_weighted_missing"]
# feature kinds of the cases that have categorical columns ('c'); everything else is numeric
FEATURE_TYPES = {"synthetic_categorical_softprob": ["q"] * 6 + ["c"] * 5}


def is_cat_of(name):
    ft = FEATURE_TYPES.get(name)
    return None if ft is None else [1 if t == "c" else 0 for t in ft]


def run_case(name):
    x, y, w, params, rounds = case_data(name)
    bst, bins = O.train(params, x, y, rounds, weight=w, is_cat=is_cat_of(name))
    cuts = bst.cuts
    trees = []
    for t in bst.trees():
        trees.append({k: [float(v) if k in ("split_cond", "value", "loss_chg") else int(v) for v in getattr(t, k)]
                      for k in ("left", "right", "split_feature", "split_bin", "default_left", "split_cond", "value", "loss_chg")})
        if name in FEATURE_TYPES:   # category sets (the categories that go right) of the categorical split nodes
            trees[-1]["split_type"] = [int(v) for v in t.split_type]
            trees[-1]["categories"] = {str(i): t.categories(i) for i in range(t.n_nodes) if t.split_type[i]}
    pred = bst.predict(x[:64])
    return {"name": name, "params": params, "rounds": rounds,
            "cut_ptrs": [int(v) for v in cuts.ptrs], "cut_vals_bits": [int(v) for v in cuts.vals.view(np.uint32)],
            "min_vals_bits": [int(v) for v in cuts.mins.view(np.uint32)], "has_missing": [int(v) for v in cuts.has_missing],
            "bins_sum_per_feature": [int(v) for v in bins.astype(np.int64).sum(axis=0)],
            "trees": trees, "pred_head": [float(v) for v in np.asarray(pred, np.float64).reshape(-1)]}


if __name__ == "__main__":
    for name in CASES:
        out = run_case(name)
        with open(os.path.join(HERE, name + ".json"), "w") as f:
            json.dump(out, f)
        print(name, "trees", len(out["trees"]), "nodes", [len(t["left"]) for t in out["trees"]])
