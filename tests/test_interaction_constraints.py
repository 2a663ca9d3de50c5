"""interaction_constraints on the host (no GPU): the canonical form of every accepted input, the errors, the sklearn
surface, save_config, and the path rule the GPU tests check trees against (DESIGN.md §2 item 14)."""
import json

import numpy as np
import pytest

from xgboost_ray_b200 import engine as E


def allowed_features(path, sets, n_features):
    """The rule as stated: every feature at the root; elsewhere the union of the sets that contain every feature of the
    path from the root (`path`, a set of feature indices)."""
    if not path:
        return set(range(n_features))
    out = set()
    for s in sets:
        if set(path) <= set(s):
            out |= set(s)
    return out


def rule_violations(tree, sets, n_features):
    """(node, feature, path) of every split in `tree` (a dict of arrays with left / right / split_feature) that the
    rule forbids; [] when the tree obeys the constraints."""
    bad = []
    stack = [(0, frozenset())]
    while stack:
        nid, path = stack.pop()
        f = int(tree["split_feature"][nid])
        if f < 0:
            continue
        if f not in allowed_features(path, sets, n_features):
            bad.append((nid, f, sorted(path)))
        stack.append((int(tree["left"][nid]), path | {f}))
        stack.append((int(tree["right"][nid]), path | {f}))
    return bad


def test_canonical_form_is_the_same_for_every_accepted_input():
    want = [[0, 1], [2, 3, 4]]
    names = ["a", "b", "c", "d", "e", "f"]
    for v in ("[[0, 1], [2, 3, 4]]", "[[1, 0], [4, 3, 2]]", " [[0,1],[2,3,4]] ", "((0, 1), (2, 3, 4))",
              [[0, 1], [2, 3, 4]], ((0, 1), (2, 3, 4)), [(1, 0), {2, 3, 4}], [np.array([0, 1]), np.arange(2, 5)],
              [[np.int64(0), np.int32(1)], [np.uint8(2), 3, 4]], [[0, 1, 1, 0], [2, 3, 4, 4]], [[0, 1], [], [2, 3, 4]],
              [["a", "b"], ["c", "d", "e"]], '[["a", "b"], ["c", "d", "e"]]', [["a", 1], [2, "d", "e"]]):
        assert E.interaction_sets(v, 6, names) == want, v


@pytest.mark.parametrize("off", [None, "", "  ", "[]", [], (), [[]], "[[], []]"])
def test_empty_inputs_mean_no_constraints(off):
    assert E.interaction_sets(off, 6) == []


@pytest.mark.parametrize("bad,needle", [
    ("[[0, 1], [2, 9]]", "9"), ([[0, 6]], "6"), ([[-1, 2]], "-1"), ([[0, 1.5]], "1.5"), ([[0, 1.0]], "1.0"),
    ([[True, 2]], "True"), ([["zz", 1]], "zz"), ("[[0, 1], [2, 3", "does not parse"), ("0, 1", "0"),
    ("not a list", "does not parse"), ([0, 1], "0"), (5, "5"), ([[None]], "None"),
])
def test_invalid_inputs_raise_naming_the_entry(bad, needle):
    with pytest.raises(E.XGBoostError) as ei:
        E.interaction_sets(bad, 6, ["a", "b", "c", "d", "e", "f"])
    assert needle in str(ei.value)


def test_names_need_feature_names():
    with pytest.raises(E.XGBoostError, match="unknown feature name"):
        E.interaction_sets([["a", "b"]], 6, None)


@pytest.fixture(scope="module")
def built():
    """libb2hist.so: the engine checks the parameters (B2_CheckParams needs no device)."""
    from xgboost_ray_b200 import build
    return build.build()


def test_parameter_is_no_longer_rejected(built):
    E._check_supported({"interaction_constraints": "[[0, 1], [2, 3, 4]]"})
    with pytest.raises(E.XGBoostError):     # its neighbours still are
        E._check_supported({"monotone_constraints": "(1,0)"})


@pytest.mark.parametrize("value", ["[[0, 1], [2, 3, 4]]", [[0, 1], [2, 3, 4]], [[1, 0, 0], (4, 3, 2)]])
def test_save_config_reports_the_resolved_sets(value):
    b = E.Booster({"objective": "reg:squarederror", "interaction_constraints": value})
    b.n_features = 10
    cfg = json.loads(b.save_config())
    assert cfg["learner"]["gradient_booster"]["tree_train_param"]["interaction_constraints"] == "[[0, 1], [2, 3, 4]]"


@pytest.mark.parametrize("value", [None, "", "[]", []])
def test_save_config_unchanged_without_constraints(value):
    plain = E.Booster({"objective": "reg:squarederror"})
    plain.n_features = 10
    b = E.Booster({"objective": "reg:squarederror"} if value is None else
                  {"objective": "reg:squarederror", "interaction_constraints": value})
    b.n_features = 10
    cfg = json.loads(b.save_config())
    assert "tree_train_param" not in cfg["learner"]["gradient_booster"]
    if value is None:
        assert b.save_config() == plain.save_config()


def test_sklearn_forwards_and_clones_the_parameter():
    from sklearn.base import clone

    from xgboost_ray_b200.sklearn import RayXGBClassifier, RayXGBRegressor, RayXGBRFRegressor
    for cls in (RayXGBRegressor, RayXGBClassifier, RayXGBRFRegressor):
        est = cls(interaction_constraints="[[0, 1], [2, 3, 4]]")
        assert est.get_xgb_params()["interaction_constraints"] == "[[0, 1], [2, 3, 4]]"
        assert clone(est).interaction_constraints == "[[0, 1], [2, 3, 4]]"
        assert "interaction_constraints" not in cls().get_xgb_params()
    est = RayXGBRegressor(interaction_constraints=[[0, 1], [2, 3, 4]])
    assert clone(est).get_params()["interaction_constraints"] == [[0, 1], [2, 3, 4]]


# ---- the rule the GPU tests check trees against, on hand-built trees
def _tree(splits):
    """splits: {nid: feature} of a complete binary tree numbered heap-style (children 2n+1, 2n+2)."""
    n = 2 * (max(splits) + 1) + 1
    t = {"left": -np.ones(n, np.int32), "right": -np.ones(n, np.int32), "split_feature": -np.ones(n, np.int32)}
    for nid, f in splits.items():
        t["left"][nid], t["right"][nid], t["split_feature"][nid] = 2 * nid + 1, 2 * nid + 2, f
    return t


def test_rule_root_allows_every_feature_and_paths_stay_in_one_set():
    sets = [[0, 1], [1, 2]]
    assert allowed_features(set(), sets, 5) == {0, 1, 2, 3, 4}
    assert allowed_features({1}, sets, 5) == {0, 1, 2}            # overlapping sets: 1 is in both
    assert allowed_features({0}, sets, 5) == {0, 1}
    assert allowed_features({0, 1}, sets, 5) == {0, 1}
    assert allowed_features({0, 2}, sets, 5) == set()
    assert allowed_features({4}, sets, 5) == set()                # root split on a feature in no set: leaves below
    assert allowed_features({3}, [[3]], 5) == {3}                 # singleton set
    assert rule_violations(_tree({0: 1, 1: 0, 2: 2, 3: 0, 6: 1}), sets, 5) == []
    assert rule_violations(_tree({0: 4}), sets, 5) == []
    assert rule_violations(_tree({0: 4, 1: 0}), sets, 5) == [(1, 0, [4])]
    assert rule_violations(_tree({0: 1, 1: 0, 3: 2}), sets, 5) == [(3, 2, [0, 1])]
    assert rule_violations(_tree({0: 0, 2: 3}), [[0, 1], [2, 3]], 5) == [(2, 3, [0])]


@pytest.mark.parametrize("value", [[[0, 1], [2, 3, 4]], [[np.int64(1), 0], ["c", "d", "e"]]])
def test_model_json_keeps_the_resolved_sets(value):
    """list, numpy and feature-name inputs survive save_raw / load_model (and so pickles and actor hand-offs)"""
    b = E.Booster({"objective": "reg:squarederror", "interaction_constraints": value})
    b.n_features, b.feature_names = 6, list("abcdef")
    c = E.Booster()
    c.load_model(b.save_raw())
    assert c.params["interaction_constraints"] == "[[0, 1], [2, 3, 4]]"
    assert json.loads(c.save_config())["learner"]["gradient_booster"]["tree_train_param"] == {
        "interaction_constraints": "[[0, 1], [2, 3, 4]]"}


# ---- constrained trees grown on the CPU (tests/interaction_reference.py), first checked against the oracle
from tests import interaction_reference as R  # noqa: E402


def _data(n, f, seed, nan_frac=0.0):
    rng = np.random.RandomState(seed)
    X = rng.uniform(0, 10, size=(n, f)).astype(np.float32)
    if nan_frac:
        X[rng.uniform(size=X.shape) < nan_frac] = np.nan
    Z = np.nan_to_num(X, nan=5.0)
    y = (Z[:, 0] * Z[:, 1] * 0.1 + Z[:, 2] - (Z[:, 3] - 5) * (Z[:, 4] - 5) * 0.2 + Z[:, 1] * Z[:, 5] * 0.05 +
         rng.normal(scale=0.5, size=n)).astype(np.float32)
    return X, y, rng


def _same(ref, ob):
    assert ref.num_trees == ob.num_trees
    for i in range(ob.num_trees):
        a, b = ref.tree(i), ob.tree(i)
        for k in ("left", "right", "split_feature", "split_bin", "default_left"):
            assert np.array_equal(getattr(a, k), getattr(b, k)), (i, k)
        assert np.array_equal(a.split_cond.view(np.uint32), b.split_cond.view(np.uint32)), i
        assert np.array_equal(a.loss_chg, b.loss_chg), i
        leaf = b.split_feature < 0
        assert np.max(np.abs(a.value[leaf] - b.value[leaf])) <= 1e-6, i


def _violations(model, sets, f):
    return [v for t in model.trees() for v in rule_violations(vars(t), sets, f)]


@pytest.mark.parametrize("case", [
    dict(params={"objective": "reg:squarederror", "max_depth": 4}),
    dict(params={"objective": "reg:squarederror", "max_depth": 6, "alpha": 0.5, "gamma": 0.3, "min_child_weight": 3}, nan=0.08),
    dict(params={"objective": "binary:logistic", "max_depth": 5, "max_delta_step": 0.7}, nan=0.05, weight=True),
    dict(params={"objective": "multi:softprob", "num_class": 3, "max_depth": 4}, nan=0.05),
    dict(params={"objective": "reg:squarederror", "max_depth": 6, "colsample_bytree": 0.8, "colsample_bylevel": 0.8,
                 "colsample_bynode": 0.6, "seed": 7}, fw=True),
])
@pytest.mark.parametrize("sets", [None, [], "all"])
def test_reference_without_constraints_is_the_oracle(oracle, case, sets):
    """The restated growth is the oracle's, bit for bit, when no constraint (or one set of every feature) is given."""
    n, f = 3000, 8
    X, y, rng = _data(n, f, 3, case.get("nan", 0.0))
    params = dict(case["params"], base_score=0.5)
    if params["objective"] == "binary:logistic":
        y = (y > np.median(y)).astype(np.float32)
    if params["objective"] == "multi:softprob":
        y = np.digitize(y, np.quantile(y, [1 / 3, 2 / 3])).astype(np.float32)
    w = rng.uniform(0.5, 2.0, size=n).astype(np.float32) if case.get("weight") else None
    fw = rng.uniform(0.1, 3.0, size=f).astype(np.float32) if case.get("fw") else None
    ob, _ = oracle.train(params, X, y, 3, weight=w, feature_weights=fw)
    ref = R.train(params, X, y, 3, sets=[list(range(f))] if sets == "all" else sets, weight=w, feature_weights=fw)
    _same(ref, ob)


SHAPES = {
    "disjoint": [[0, 1, 2], [3, 4, 5]],
    "overlapping": [[0, 1], [1, 2], [1, 5]],
    "singletons": [[0], [3], [1, 2, 4]],
    "not in any set": [[0, 1], [3, 4]],          # 2, 5, 6, 7 in no set
}


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_reference_trees_obey_the_rule_and_differ_from_free_trees(shape, seed):
    sets = SHAPES[shape]
    n, f = 3000, 8
    X, y, _ = _data(n, f, seed, 0.05)
    params = {"objective": "reg:squarederror", "max_depth": 5, "base_score": 0.5}
    con = R.train(params, X, y, 4, sets=sets)
    assert _violations(con, sets, f) == []
    assert _violations(R.train(params, X, y, 4), sets, f) != []     # the constraint changed the choice


def test_reference_overlapping_sets_allow_the_union():
    """root on 1 with [[0, 1], [1, 2]]: both 0 and 2 are allowed below it (one per path), never together"""
    n, f = 4000, 4
    rng = np.random.RandomState(5)
    X = rng.uniform(0, 10, size=(n, f)).astype(np.float32)
    y = (10 * (X[:, 1] > 5) + np.where(X[:, 1] > 5, X[:, 0], X[:, 2]) + rng.normal(scale=0.1, size=n)).astype(np.float32)
    sets = [[0, 1], [1, 2]]
    m = R.train({"objective": "reg:squarederror", "max_depth": 3, "base_score": 0.5}, X, y, 1, sets=sets)
    t = m.tree(0)
    assert t.split_feature[0] == 1 and {int(t.split_feature[t.left[0]]), int(t.split_feature[t.right[0]])} == {0, 2}
    assert _violations(m, sets, f) == []


def test_reference_root_on_feature_in_no_set_is_a_stump(oracle):
    n, f = 3000, 4
    rng = np.random.RandomState(6)
    X = rng.uniform(0, 10, size=(n, f)).astype(np.float32)
    y = (10 * (X[:, 3] > 5) + X[:, 0] * X[:, 1] * 0.1).astype(np.float32)
    params = {"objective": "reg:squarederror", "max_depth": 4, "base_score": 0.5}
    m = R.train(params, X, y, 1, sets=[[0, 1], [1, 2]])
    assert m.tree(0).split_feature[0] == 3 and m.tree(0).n_nodes == 3
    _same(m, oracle.train(dict(params, max_depth=1), X, y, 1)[0])


def test_reference_liveness_pairs():
    """y = x0 x1 + x2 x3: the free trees cross the pairs, the constrained ones never do"""
    rng = np.random.RandomState(8)
    X = rng.uniform(0, 10, size=(4000, 4)).astype(np.float32)
    y = (X[:, 0] * X[:, 1] + X[:, 2] * X[:, 3]).astype(np.float32)
    params = {"objective": "reg:squarederror", "max_depth": 4, "base_score": 0.5}
    sets = [[0, 1], [2, 3]]
    assert _violations(R.train(params, X, y, 3), sets, 4) != []
    assert _violations(R.train(params, X, y, 3, sets=sets), sets, 4) == []


def test_reference_column_sampling_then_constraint():
    """colsample_bynode < 1: every split lies in its node's sampled set and in its allowed set"""
    n, f = 3000, 8
    X, y, rng = _data(n, f, 9, 0.03)
    fw = rng.uniform(0.2, 3.0, size=f).astype(np.float32)
    sets = SHAPES["overlapping"]
    params = {"objective": "reg:squarederror", "max_depth": 5, "base_score": 0.5, "colsample_bynode": 0.5, "seed": 4}
    m = R.train(params, X, y, 3, sets=sets, feature_weights=fw)
    fwq = np.rint(fw.astype(np.float64) * 65536.0).astype(np.uint32)
    for ti, t in enumerate(m.trees()):
        level = R._select(4, ti, R.SCOPE_LEVEL0, None, fwq, f, 1.0)   # bytree = bylevel = 1: every feature
        stack = [(0, frozenset())]
        while stack:
            nid, path = stack.pop()
            feat = int(t.split_feature[nid])
            if feat < 0:
                continue
            node = R._select(4, ti, R.SCOPE_NODE0 + nid, level, fwq, f, 0.5)
            assert node[feat] and feat in R.allowed_features(path, sets, f)
            stack += [(int(t.left[nid]), path | {feat}), (int(t.right[nid]), path | {feat})]
    assert _violations(m, sets, f) == []
