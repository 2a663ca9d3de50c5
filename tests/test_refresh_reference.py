"""CPU checks of the refresh reference (tests/refresh_reference.py) and of the update-mode parameter rules (DESIGN.md 2
item 20): node sums are their children's sums, refresh_leaf=0 keeps every leaf value, a node no row reaches weighs 0,
and the parameter checks name what they refuse."""
import numpy as np
import pytest

from tests.refresh_reference import leaf_of_rows, refresh_tree

F32 = np.float32


def hand_tree():
    """root: x0 < 0.5 (missing left); left: x1 < 0 -> leaves 3, 4; right: leaf 2 (categorical split on x1 in node 1
    when categorical=True: categories {1, 3} go right)"""
    t = dict(left=np.array([1, 3, -1, -1, -1], np.int32), right=np.array([2, 4, -1, -1, -1], np.int32),
             parent=np.array([-1, 0, 0, 1, 1], np.int32), split_feature=np.array([0, 1, -1, -1, -1], np.int32),
             split_bin=np.full(5, -1, np.int32), split_cond=np.array([0.5, 0.0, 0, 0, 0], F32),
             default_left=np.array([1, 0, 0, 0, 0], np.uint8), value=np.array([0, 0, 0.25, -0.5, 0.75], F32),
             base_weight=np.zeros(5, F32), loss_chg=np.array([3.0, 1.0, 0, 0, 0], F32), sum_hess=np.zeros(5),
             split_type=np.zeros(5, np.uint8), cat_bits=np.zeros((5, 8), np.uint32))
    return t


def data(n=4000, seed=0):
    rng = np.random.RandomState(seed)
    X = rng.uniform(-1, 1, (n, 2)).astype(F32)
    X[rng.rand(n) < 0.1, 0] = np.nan
    g = rng.normal(0, 1, n).astype(F32)
    h = rng.uniform(0.5, 1.5, n).astype(F32)
    return X, g, h


PARAMS = {"eta": 0.3, "lambda": 1.0, "min_child_weight": 0.0}


@pytest.fixture(scope="module")
def built():
    """libb2hist.so: the engine checks the parameters (B2_CheckParams needs no device)."""
    from xgboost_ray_b200 import build
    return build.build()


def test_traversal_rules():
    t = hand_tree()
    X = np.array([[0.0, -1.0], [0.0, 1.0], [0.9, 0.0], [np.nan, 2.0]], F32)
    assert leaf_of_rows(t, X).tolist() == [3, 4, 2, 4]
    t["split_type"][1] = 1
    t["cat_bits"][1, 0] = (1 << 1) | (1 << 3)
    X = np.array([[0.0, 1.0], [0.0, 2.0], [0.0, 3.0], [0.0, -1.0], [0.0, 300.0]], F32)
    assert leaf_of_rows(t, X).tolist() == [4, 3, 4, 3, 3]


def test_node_sums_are_children_sums():
    X, g, h = data()
    r = refresh_tree(hand_tree(), X, g, h, PARAMS)
    sg, sh = r["_sums"]
    for nid, (l, rr) in enumerate(zip(r["left"], r["right"])):
        if r["split_feature"][nid] >= 0:
            assert sg[nid] == sg[l] + sg[rr] and sh[nid] == sh[l] + sh[rr]
    assert r["sum_hess"][0] == pytest.approx(float(h.astype(np.float64).sum()), rel=1e-9)
    internal = r["split_feature"] >= 0
    assert np.array_equal(r["value"][internal], r["base_weight"][internal])


def test_refresh_leaf_off_keeps_leaves():
    X, g, h = data(seed=1)
    t = hand_tree()
    r = refresh_tree(t, X, g, h, PARAMS, refresh_leaf=False)
    leaf = t["split_feature"] < 0
    assert np.array_equal(r["value"][leaf], t["value"][leaf])
    assert not np.array_equal(r["base_weight"], t["base_weight"])
    on = refresh_tree(t, X, g, h, PARAMS, refresh_leaf=True)
    assert np.array_equal(on["value"][leaf], (on["base_weight"][leaf] * F32(0.3)).astype(F32))
    assert np.array_equal(on["loss_chg"][leaf], t["loss_chg"][leaf])   # leaves keep theirs


def test_unreached_node_weighs_zero():
    X, g, h = data(seed=2)
    X[:, 0] = 0.0   # every row goes left at the root
    r = refresh_tree(hand_tree(), X, g, h, PARAMS)
    assert r["sum_hess"][2] == 0.0 and r["base_weight"][2] == 0.0 and r["value"][2] == 0.0


def test_parallel_tree_scaling():
    X, g, h = data(seed=3)
    r = refresh_tree(hand_tree(), X, g, h, PARAMS, num_parallel_tree=3)
    leaf = r["split_feature"] < 0
    assert np.array_equal(r["value"][leaf], (r["base_weight"][leaf] * F32(F32(0.3) / F32(3))).astype(F32))


@pytest.mark.parametrize("params, match", [
    ({"process_type": "update"}, "needs updater='refresh'"),
    ({"process_type": "update", "updater": "prune"}, "updater='prune'"),
    ({"process_type": "update", "updater": "refresh,prune"}, "refresh,prune"),
    ({"process_type": "update", "updater": "grow_quantile_histmaker"}, "grow_quantile_histmaker"),
    ({"updater": "refresh"}, "needs process_type='update'"),
    ({"process_type": "update", "updater": "refresh", "booster": "dart"}, "booster='dart'"),
    ({"process_type": "update", "updater": "refresh", "objective": "reg:quantileerror"}, "reg:quantileerror"),
    ({"process_type": "update", "updater": "refresh", "multi_strategy": "multi_output_tree", "num_target": 3},
     "multi_output_tree"),
    ({"process_type": "sideways"}, "process_type='sideways'"),
    ({"process_type": "update", "updater": "refresh", "refresh_leaf": 2}, "refresh_leaf"),
    ({"updater": "prune"}, "updater='prune'"),
])
def test_parameter_checks(built, params, match):
    from xgboost_ray_b200 import engine
    with pytest.raises(engine.XGBoostError, match=match):
        engine._check_supported(params)


def test_accepted_parameters(built):
    from xgboost_ray_b200 import engine
    engine._check_supported({"process_type": "update", "updater": "refresh", "refresh_leaf": 0})
    engine._check_supported({"process_type": "default", "refresh_leaf": 1})
    engine._check_supported({"updater": "grow_gpu_hist"})


def test_update_without_model_is_refused(built):
    from xgboost_ray_b200 import engine
    with pytest.raises(engine.XGBoostError, match="xgb_model"):
        engine.train({"process_type": "update", "updater": "refresh"}, None, 1)


def test_update_refuses_restarts():
    from xgboost_ray_b200 import main
    from xgboost_ray_b200.matrix import RayDMatrix
    X = np.zeros((8, 2), F32)
    d = RayDMatrix(X, np.zeros(8, F32))
    p = {"process_type": "update", "updater": "refresh"}
    for rp in (main.RayParams(num_actors=1, max_actor_restarts=1),
               main.RayParams(num_actors=1, elastic_training=True, max_failed_actors=1, max_actor_restarts=1)):
        with pytest.raises(ValueError, match="process_type='update' does not support elastic training"):
            main.train(p, d, 1, ray_params=rp)
