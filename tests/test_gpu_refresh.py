"""The refresh updater (process_type="update", updater="refresh"; DESIGN.md 2 item 20) on the GPU.

Self-refresh is the identity: a model grown here without sampling, refreshed on its own training matrix with the same
parameters, keeps every leaf value and every prediction bit for bit (the 40-bit leaf sums are the grow path's), and its
covers agree within 1e-5 relative (the grow path's covers come from the histogram's coarser fixed point).  On other
data the refreshed model equals tests/refresh_reference.py: structure unchanged, leaf values and base_weight within
1e-5, loss_chg and sum_hess within 1e-5 relative.  Also: a hand-written stock-format tree with 5,000 leaves at depth
above 16 (the global-memory paths of refresh_kernel), determinism, R smaller than the model, the refusals, the model
file, pickling, save_config and the public API."""
import json
import pickle

import numpy as np
import pytest

from tests import shap_reference
from tests.refresh_reference import leaf_of_rows, refresh_model
from tests.test_gpu_parity import make_cat_data, make_data, CAT_TYPES

pytestmark = pytest.mark.gpu
F32 = np.float32
UPD = {"process_type": "update", "updater": "refresh"}
STRUCT = ("left", "right", "parent", "split_feature", "split_cond", "default_left", "split_type", "cat_bits")


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def close_rel(a, b, tol=1e-5):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.all(np.abs(a - b) <= tol * np.maximum(np.abs(b), 1e-30) + 1e-12)


def assert_structure(new, old):
    assert len(new) == len(old)
    for tn, to in zip(new, old):
        for k in STRUCT:
            assert np.array_equal(np.asarray(tn[k]), np.asarray(to[k]), equal_nan=True), k


def self_case(objective, seed):
    n, f = 6000, 10
    X = make_data(n, f, seed, "uniform", nan_frac=0.03)
    rng = np.random.RandomState(seed)
    s = np.nan_to_num(X[:, 0]) + np.sin(3 * np.nan_to_num(X[:, 1]))
    params = {"objective": objective, "eta": 0.3, "base_score": 0.5}
    kw = {}
    if objective == "multi:softprob":
        y = np.clip(np.floor((s - s.min()) / (np.ptp(s) + 1e-9) * 5), 0, 4).astype(F32)
        params["num_class"] = 5
    elif objective == "binary:logistic":
        y = (s > np.median(s)).astype(F32)
    elif objective == "count:poisson":
        y = rng.poisson(np.exp(0.3 * s)).astype(F32)
    elif objective == "rank:ndcg":
        y = np.clip(np.round(s), 0, 3).astype(F32)
        kw["group"] = [50] * (n // 50)
    elif objective == "multi_target":
        params["objective"] = "reg:squarederror"
        y = np.stack([s, 0.5 * s + np.nan_to_num(X[:, 2]), np.cos(np.nan_to_num(X[:, 3]))], axis=1).astype(F32)
    else:
        y = (s + rng.normal(0, 0.3, n)).astype(F32)
    return X, y, params, kw


def dmatrix(eng, X, y, kw=None, **extra):
    if np.ndim(y) == 2:
        extra["multi_target"] = True
    dm = eng.DMatrix(X, label=y, **extra)
    if kw and "group" in kw:
        dm.set_group(kw["group"])
    return dm


@pytest.mark.parametrize("objective, depth", [
    ("reg:squarederror", 3), ("reg:squarederror", 8), ("reg:squarederror", 14), ("binary:logistic", 6),
    ("multi:softprob", 6), ("count:poisson", 6), ("rank:ndcg", 6), ("multi_target", 6)])
def test_self_refresh_is_identity(eng, objective, depth):
    X, y, params, kw = self_case(objective, 3 + depth)
    params["max_depth"] = depth
    bst = eng.train(params, dmatrix(eng, X, y, kw), 4)
    old = bst.get_trees()
    new = eng.train(dict(params, **UPD), dmatrix(eng, X, y, kw), 4, xgb_model=bst)
    trees = new.get_trees()
    assert_structure(trees, old)
    for tn, to in zip(trees, old):
        leaf = to["split_feature"] < 0
        assert np.array_equal(tn["value"][leaf].view(np.uint32), to["value"][leaf].view(np.uint32))
        assert close_rel(tn["sum_hess"], to["sum_hess"])
    dp = dmatrix(eng, X, y, kw)
    assert np.array_equal(new.predict(dp, output_margin=True).view(np.uint32),
                          bst.predict(dp, output_margin=True).view(np.uint32))


def sqerr_grad(y, w):
    def fn(margin):
        m = margin.reshape(-1)
        g = (m - y).astype(F32)
        h = np.ones_like(g)
        if w is not None:
            g, h = (g * w).astype(F32), w.astype(F32)
        return g.reshape(-1, 1), h.reshape(-1, 1)
    return fn


def assert_matches_reference(trees, ref):
    assert_structure(trees, ref)
    for tn, tr in zip(trees, ref):
        assert np.allclose(tn["value"], tr["value"], atol=1e-5, rtol=0)
        assert np.allclose(tn["base_weight"], tr["base_weight"], atol=1e-5, rtol=0)
        assert close_rel(tn["loss_chg"], tr["loss_chg"])
        assert close_rel(tn["sum_hess"], tr["sum_hess"])


@pytest.mark.parametrize("npt", [1, 3])
def test_refresh_other_data_matches_reference(eng, npt):
    n, f = 8000, 12
    X = make_data(n, f, 11, "mixed", nan_frac=0.1)
    y = (np.nan_to_num(X[:, 0]) * 2 + np.nan_to_num(X[:, 3])).astype(F32)
    bst = eng.train({"max_depth": 6, "eta": 0.3, "base_score": 0.0, "num_parallel_tree": npt, "subsample": 0.8,
                     "colsample_bynode": 0.7, "seed": 1}, eng.DMatrix(X, label=y), 3)
    X2 = make_data(n, f, 12, "mixed", nan_frac=0.15)
    rng = np.random.RandomState(13)
    y2 = (np.nan_to_num(X2[:, 0]) * 1.5 - np.nan_to_num(X2[:, 5]) + rng.normal(0, 0.5, n)).astype(F32)
    w = rng.uniform(0.2, 2.0, n).astype(F32)
    bm = rng.normal(0, 0.3, n).astype(F32)
    up = dict(UPD, max_depth=6, eta=0.1, reg_lambda=2.0, reg_alpha=0.5, max_delta_step=0.7, min_child_weight=0.5)
    new = eng.train(up, eng.DMatrix(X2, label=y2, weight=w, base_margin=bm), 3, xgb_model=bst)
    params = {"eta": 0.1, "lambda": 2.0, "alpha": 0.5, "max_delta_step": 0.7, "min_child_weight": 0.5}
    ref, margin = refresh_model(bst.get_trees(), X2, params, 1, npt, bm, sqerr_grad(y2, w))
    assert_matches_reference(new.get_trees(), ref)
    # the base margin and the refreshed trees give the engine's train margin
    got = new.predict(eng.DMatrix(X2, base_margin=bm), output_margin=True)
    assert np.allclose(got, margin.reshape(-1), atol=1e-4)
    # TreeSHAP weighs paths by the refreshed covers: pred_contribs equals the reference on the refreshed trees, and the
    # same trees with the original model's covers give different contributions
    rows = slice(0, 600)
    xs, bs = X2[rows], bm[rows]
    phi = new.predict(eng.DMatrix(xs, base_margin=bs), pred_contribs=True, strict_shape=True)
    trees = new.get_trees()
    ref_phi = shap_reference.shap_contribs(trees, xs, npt=npt, base_margin=bs)
    tol = 1e-5 * np.maximum(1.0, np.abs(got[rows]))[:, None, None]
    assert np.all(np.abs(phi - ref_phi) <= tol)
    stale = [dict(t, sum_hess=o["sum_hess"]) for t, o in zip(trees, bst.get_trees())]
    stale_phi = shap_reference.shap_contribs(stale, xs, npt=npt, base_margin=bs)
    assert np.max(np.abs(phi - stale_phi)) > 1e-3


def test_refresh_categorical_and_custom_objective(eng):
    X, score, rng = make_cat_data(12000, 41, 0.05)
    y = (score + rng.normal(0, 0.3, len(score))).astype(F32)
    bst = eng.train({"max_depth": 5, "base_score": 0.0}, eng.DMatrix(X, label=y, feature_types=CAT_TYPES,
                                                                     enable_categorical=True), 3)
    X2, score2, rng2 = make_cat_data(9000, 42, 0.05)
    y2 = (score2 * 0.5 + rng2.normal(0, 0.3, len(score2))).astype(F32)

    def obj(pred, dm):
        return (np.asarray(pred, F32) - y2).astype(F32), np.ones(len(y2), F32)
    dm2 = eng.DMatrix(X2, label=y2, feature_types=CAT_TYPES, enable_categorical=True)
    new = eng.train(dict(UPD, max_depth=5), dm2, 3, xgb_model=bst, obj=obj)
    ref, _ = refresh_model(bst.get_trees(), X2, {"eta": 0.3}, 1, 1, np.zeros(len(y2), F32), sqerr_grad(y2, None))
    assert_matches_reference(new.get_trees(), ref)


def stock_model(n_leaves=5000, chain=24, n_features=6, seed=5):
    """an irregular xgboost JSON model: one tree with a left chain of `chain` splits, then random leaf splits"""
    rng = np.random.RandomState(seed)
    left, right, parent, feat, cond, dl = [-1], [-1], [2147483647], [0], [0.0], [0]
    def split(nid):
        for _ in range(2):
            left.append(-1); right.append(-1); parent.append(nid); feat.append(0); cond.append(0.0); dl.append(0)
        left[nid], right[nid] = len(left) - 2, len(left) - 1
        feat[nid] = int(rng.randint(n_features)); cond[nid] = float(rng.uniform(-1, 1)); dl[nid] = int(rng.randint(2))
    nid = 0
    for _ in range(chain):
        split(nid)
        nid = left[nid]
    leaves = [i for i in range(len(left)) if left[i] < 0]
    while len(leaves) < n_leaves:
        i = leaves.pop(rng.randint(len(leaves)))
        split(i)
        leaves += [left[i], right[i]]
    n = len(left)
    sc = [cond[i] if left[i] >= 0 else float(rng.normal(0, 0.1)) for i in range(n)]
    tree = {"base_weights": [0.0] * n, "categories": [], "categories_nodes": [], "categories_segments": [],
            "categories_sizes": [], "default_left": dl, "id": 0, "left_children": left, "loss_changes": [0.0] * n,
            "parents": parent, "right_children": right, "split_conditions": sc,
            "split_indices": [feat[i] if left[i] >= 0 else 0 for i in range(n)], "split_type": [0] * n,
            "sum_hessian": [0.0] * n,
            "tree_param": {"num_deleted": "0", "num_feature": str(n_features), "num_nodes": str(n),
                           "size_leaf_vector": "1"}}
    return {"learner": {"attributes": {}, "feature_names": [], "feature_types": [],
                        "gradient_booster": {"model": {"gbtree_model_param": {"num_parallel_tree": "1", "num_trees": "1"},
                                                       "iteration_indptr": [0, 1], "tree_info": [0], "trees": [tree]},
                                             "name": "gbtree"},
                        "learner_model_param": {"base_score": "0.25", "boost_from_average": "1", "num_class": "0",
                                                "num_feature": str(n_features), "num_target": "1"},
                        "objective": {"name": "reg:squarederror", "reg_loss_param": {"scale_pos_weight": "1"}}},
            "version": [2, 0, 3]}


def depth_of(tree):
    d = np.zeros(len(tree["left"]), np.int64)
    for i in range(len(tree["left"])):
        if tree["split_feature"][i] >= 0:
            d[tree["left"][i]] = d[tree["right"][i]] = d[i] + 1
    return int(d.max())


@pytest.mark.parametrize("n_leaves", [2000, 5000])
def test_stock_model_with_many_leaves(eng, tmp_path, n_leaves):
    """2,000 leaves: nodes in global memory, leaf sums in shared memory; 5,000 leaves: both in global memory"""
    path = tmp_path / "stock.json"
    path.write_text(json.dumps(stock_model(n_leaves=n_leaves)))
    src = eng.Booster(model_file=str(path))
    t0 = src.get_trees()[0]
    assert int((t0["split_feature"] < 0).sum()) == n_leaves and depth_of(t0) > 16
    rng = np.random.RandomState(6)
    X = rng.uniform(-1.2, 1.2, (50000, 6)).astype(F32)
    X[rng.rand(50000) < 0.05, 2] = np.nan
    y = rng.normal(0, 1, 50000).astype(F32)
    new = eng.train(dict(UPD, eta=0.5), eng.DMatrix(X, label=y), 1, xgb_model=str(path))
    ref, _ = refresh_model(src.get_trees(), X, {"eta": 0.5}, 1, 1, np.full(50000, 0.25, F32), sqerr_grad(y, None))
    assert_matches_reference(new.get_trees(), ref)
    leaf = np.asarray(new.predict(eng.DMatrix(X), pred_leaf=True)).reshape(-1)
    assert np.array_equal(leaf, leaf_of_rows(src.get_trees()[0], X))


def test_deterministic_rounds_and_file(eng, tmp_path):
    X, y, params, _ = self_case("reg:squarederror", 21)
    params["max_depth"] = 6
    bst = eng.train(params, eng.DMatrix(X, label=y), 5)
    X2 = X[::-1].copy(); y2 = (y[::-1] * 0.5).astype(F32)
    a = eng.train(dict(params, **UPD), eng.DMatrix(X2, label=y2), 5, xgb_model=bst)
    b = eng.train(dict(params, **UPD), eng.DMatrix(X2, label=y2), 5, xgb_model=bst)
    assert bytes(a.save_raw()) == bytes(b.save_raw())
    short = eng.train(dict(params, **UPD), eng.DMatrix(X2, label=y2), 2, xgb_model=bst)
    assert short.num_boosted_rounds() == 2
    assert bytes(json.dumps(short.get_trees()[0]["value"].tolist()).encode()) == \
        bytes(json.dumps(a.get_trees()[0]["value"].tolist()).encode())
    cfg = json.loads(a.save_config())["learner"]["gradient_booster"]["gbtree_train_param"]
    assert cfg == {"process_type": "update", "updater": "refresh", "refresh_leaf": "1"}
    assert "gbtree_train_param" not in json.loads(bst.save_config())["learner"]["gradient_booster"]
    a.save_model(str(tmp_path / "m.json"))
    c = eng.Booster(model_file=str(tmp_path / "m.json"))
    d = pickle.loads(pickle.dumps(a))
    dp = eng.DMatrix(X2)
    for m in (c, d):
        assert np.array_equal(m.predict(dp), a.predict(dp))
    keep = eng.train(dict(params, refresh_leaf=0, **UPD), eng.DMatrix(X2, label=y2), 5, xgb_model=bst)
    for tk, to in zip(keep.get_trees(), bst.get_trees()):
        assert np.array_equal(tk["value"][to["split_feature"] < 0], to["value"][to["split_feature"] < 0])


def test_refusals(eng):
    X, y, params, _ = self_case("reg:squarederror", 31)
    params["max_depth"] = 3
    dm = eng.DMatrix(X, label=y)
    bst = eng.train(params, dm, 2)
    with pytest.raises(eng.XGBoostError, match="num_boost_round=3 but the model has 2 rounds"):
        eng.train(dict(params, **UPD), dm, 3, xgb_model=bst)
    with pytest.raises(eng.XGBoostError, match="xgb_model"):
        eng.train(dict(params, **UPD), dm, 1)
    with pytest.raises(eng.XGBoostError, match="prune"):
        eng.train(dict(params, process_type="update", updater="prune"), dm, 1, xgb_model=bst)
    with pytest.raises(eng.XGBoostError, match="dart"):
        eng.train(dict(params, booster="dart", **UPD), dm, 1, xgb_model=bst)
    with pytest.raises(eng.XGBoostError, match="reg:quantileerror"):
        eng.train(dict(params, objective="reg:quantileerror", **UPD), dm, 1, xgb_model=bst)
    with pytest.raises(eng.XGBoostError, match="needs process_type='update'"):
        eng.train(dict(params, updater="refresh"), dm, 1)
    # the update call's outputs must be the model's: a 5-class model refreshed as a single-output one is refused
    ys = np.clip(np.floor(np.abs(y)), 0, 4).astype(F32)
    soft = eng.train(dict(params, objective="multi:softprob", num_class=5), eng.DMatrix(X, label=ys), 2)
    with pytest.raises(eng.XGBoostError, match="5 trees per round"):
        eng.train(dict(UPD, max_depth=3), eng.DMatrix(X, label=ys), 2, xgb_model=soft)
    quant = eng.train(dict(params, objective="reg:quantileerror", quantile_alpha=0.5), dm, 2)
    with pytest.raises(eng.XGBoostError, match="reg:quantileerror"):
        eng.train(dict(UPD, max_depth=3), dm, 2, xgb_model=quant)


def assert_same_trees(a, b):
    ta, tb = a.get_trees(), b.get_trees()
    assert len(ta) == len(tb)
    for x, y in zip(ta, tb):
        for k in ("left", "right", "split_feature", "split_cond", "value", "base_weight", "loss_chg", "sum_hess"):
            assert np.array_equal(np.asarray(x[k]), np.asarray(y[k])), k


def test_public_api_and_sklearn(eng):
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    from xgboost_ray_b200.sklearn import RayXGBRegressor
    X, y, params, _ = self_case("reg:squarederror", 41)
    params["max_depth"] = 5
    bst = eng.train(params, eng.DMatrix(X, label=y), 3)
    X2 = X[: 4000].copy(); y2 = (y[: 4000] + 1).astype(F32)
    direct = eng.train(dict(params, **UPD), eng.DMatrix(X2, label=y2), 3, xgb_model=bst)
    via = train(dict(params, **UPD), RayDMatrix(X2, y2), 3, xgb_model=bst, ray_params=RayParams(num_actors=1))
    assert_same_trees(via, direct)
    reg = RayXGBRegressor(n_estimators=3, max_depth=5, learning_rate=0.3, base_score=0.5, process_type="update",
                          updater="refresh")
    reg.fit(X2, y2, xgb_model=bst)
    assert_same_trees(reg.get_booster(), direct)
    with pytest.raises(ValueError, match="elastic training"):
        train(dict(params, **UPD), RayDMatrix(X2, y2), 3, xgb_model=bst,
              ray_params=RayParams(num_actors=1, max_actor_restarts=1))


def test_one_vs_two_gpus(eng):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    X, y, params, _ = self_case("reg:squarederror", 51)
    params["max_depth"] = 6
    bst = eng.train(params, eng.DMatrix(X, label=y), 3)
    y2 = (y * 0.7).astype(F32)
    b1 = train(dict(params, **UPD), RayDMatrix(X, y2), 3, xgb_model=bst, ray_params=RayParams(num_actors=1))
    b2 = train(dict(params, **UPD), RayDMatrix(X, y2), 3, xgb_model=bst, ray_params=RayParams(num_actors=2))
    assert bytes(b1.save_raw()) == bytes(b2.save_raw())
