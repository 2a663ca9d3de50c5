"""XGBoost 2.x JSON model files for the slicing tests: `xgb_model_file` writes one by hand the way XGBoost writes it
(the pattern of tests/test_model_json.py's XGB_STYLE), and `keep_rounds` edits a model file to hold only some of its
boosting rounds.  `keep_rounds` is the reference a sliced Booster is compared against: it works on the file alone, from
`iteration_indptr`, and renumbers every per-tree entry (trees, tree_info, DART weight_drop and the engine's
`b2.split_bins` / `b2.split_conds` attributes)."""
import json

import numpy as np


def _tree(i, n_features, vector=0, categorical=False):
    """Stump i: split on feature i % n_features at i + 0.5 (categorical: on categories {1, 3, 200}); tagged with i."""
    left, right = -(i + 0.25), i + 0.5
    if vector:
        bw = [0.0] * vector + [left + k for k in range(vector)] + [right + k for k in range(vector)]
        cond = [i + 0.5, 0.0, 0.0]
    else:
        bw = [0.125 * i, left, right]
        cond = [0.0 if categorical else i + 0.5, left, right]
    t = {"base_weights": bw, "categories": [], "categories_nodes": [], "categories_segments": [],
         "categories_sizes": [],
         "default_left": [i % 2, 0, 0], "id": i, "left_children": [1, -1, -1], "loss_changes": [1.0 + i, 0.0, 0.0],
         "parents": [2147483647, 0, 0], "right_children": [2, -1, -1], "split_conditions": cond,
         "split_indices": [i % n_features, 0, 0], "split_type": [1 if categorical else 0, 0, 0],
         "sum_hessian": [10.0 + i, 4.0, 6.0 + i],
         "tree_param": {"num_deleted": "0", "num_feature": str(n_features), "num_nodes": "3",
                        "size_leaf_vector": str(vector) if vector else "1"}}
    if categorical:
        t.update(categories=[1, 3, 200], categories_nodes=[0], categories_segments=[0], categories_sizes=[3])
    return t


def xgb_model_file(rounds, objective="reg:squarederror", num_class=0, npt=1, alphas=None, vector=0, dart=False,
                   categorical=False, attrs=None, n_features=4):
    """A model of `rounds` boosting rounds as XGBoost 2.x writes it.  Trees per round: num_class (multi:*) or
    len(alphas) (reg:quantileerror) outputs x npt, or 1 vector-leaf tree of size `vector`.  DART weights are float32
    values whose low bits are all in use; with `categorical`, every third tree splits on a category set and tree 1 has
    the non-finite condition +inf (written by the engine as the `b2.split_conds` attribute)."""
    outputs = num_class or (len(alphas) if alphas else 1)
    per = 1 if vector else outputs * npt
    n = rounds * per
    trees = [_tree(i, n_features, vector, categorical and i % 3 == 0) for i in range(n)]
    attributes = dict(attrs or {})
    attributes["b2.split_bins"] = json.dumps([[(7 * i) % 250, -1, -1] for i in range(n)], separators=(",", ":"))
    if categorical:
        attributes["b2.split_conds"] = json.dumps([[1, 0, "inf"]], separators=(",", ":"))
    gb = {"model": {"gbtree_model_param": {"num_parallel_tree": str(npt), "num_trees": str(n)},
                    "iteration_indptr": list(range(0, n + 1, per)),
                    "tree_info": [0 if vector else (i // npt) % outputs for i in range(n)], "trees": trees},
          "name": "gbtree"}
    if dart:
        w = (np.float32(1) / (np.arange(n, dtype=np.float32) + np.float32(3))).astype(np.float32)
        gb = {"name": "dart", "gbtree": gb, "weight_drop": [float(x) for x in w]}
    if objective.startswith("multi:"):
        obj = {"name": objective, "softmax_multiclass_param": {"num_class": str(num_class)}}
    elif objective == "reg:quantileerror":
        obj = {"name": objective, "reg_quantileerror_param": {"quantile_alpha": "[%s]" % ", ".join(map(str, alphas))}}
    else:
        obj = {"name": objective, "reg_loss_param": {"scale_pos_weight": "1"}}
    targets = vector or (len(alphas) if alphas else 1)
    return json.dumps({"learner": {
        "attributes": attributes,
        "feature_names": ["f_%d" % j for j in range(n_features)],
        "feature_types": ["c" if categorical and j == 0 else "float" for j in range(n_features)],
        "gradient_booster": gb,
        "learner_model_param": {"base_score": "3.75E-1", "boost_from_average": "1",
                                "num_class": str(num_class if num_class > 1 else 0), "num_feature": str(n_features),
                                "num_target": str(targets)},
        "objective": obj}, "version": [2, 0, 3]}).encode()


def keep_rounds(raw, rounds):
    """The model file `raw` with only the boosting rounds `rounds` (ascending), as a new file."""
    d = json.loads(bytes(raw).decode())
    L = d["learner"]
    gb = L["gradient_booster"]
    m = (gb["gbtree"] if gb["name"] == "dart" else gb)["model"]
    ip = m["iteration_indptr"]
    keep = [t for r in rounds for t in range(ip[r], ip[r + 1])]
    m["trees"] = [dict(m["trees"][t], id=i) for i, t in enumerate(keep)]
    m["tree_info"] = [m["tree_info"][t] for t in keep]
    m["iteration_indptr"] = [0] + list(np.cumsum([ip[r + 1] - ip[r] for r in rounds]).tolist())
    m["gbtree_model_param"]["num_trees"] = str(len(keep))
    if gb["name"] == "dart":
        gb["weight_drop"] = [gb["weight_drop"][t] for t in keep]
    A = L["attributes"]
    if "b2.split_bins" in A:
        bins = json.loads(A["b2.split_bins"])
        A["b2.split_bins"] = json.dumps([bins[t] for t in keep], separators=(",", ":"))
    if "b2.split_conds" in A:
        new = {t: i for i, t in enumerate(keep)}
        conds = [[new[t], nid, v] for t, nid, v in json.loads(A["b2.split_conds"]) if t in new]
        A["b2.split_conds"] = json.dumps(conds, separators=(",", ":"))
        if not conds:
            del A["b2.split_conds"]
    return json.dumps(d).encode()
