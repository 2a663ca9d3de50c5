"""Vector-leaf trees (multi_strategy="multi_output_tree", DESIGN.md 2 item 19) on the GPU.

With Y = [y, y] (min_child_weight = 0, gamma = 0) every target's integer histograms are those of the single-target tree
of y, every gain term is exactly doubled and every leaf vector is (v, v): the vector model must have the single-target
model's topology and splits, loss_chg exactly twice its, and margins (m, m) bit for bit.  Row and column sampling draw
per tree and round, so they keep that equality.  Also: T = 1 ignoring the strategy, the train margin against predict,
prediction shapes, pred_leaf and iteration_range, the model file, pickling, continuation, the public API and the
refused combinations.  Distinct targets are compared with tests/multi_output_reference.py: trees and loss_chg
exactly, leaf vectors within 1e-5, train margins bit for bit."""
import json
import pickle

import numpy as np
import pytest

from tests.test_gpu_parity import make_data

pytestmark = pytest.mark.gpu
F32 = np.float32
VEC = {"multi_strategy": "multi_output_tree"}


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def dataset(obj, T, n=6000, f=12, seed=0, nan_frac=0.05):
    X = make_data(n, f, seed, "uniform", nan_frac)
    Z = np.nan_to_num(X, nan=5.0)
    rng = np.random.RandomState(seed)
    cols = [Z[:, k % f] * (0.3 + 0.1 * k) + np.sin(Z[:, (k + 1) % f]) + rng.normal(0, 0.3, n) for k in range(T)]
    Y = np.stack(cols, axis=1).astype(F32)
    if obj in ("binary:logistic", "binary:logitraw", "reg:logistic"):
        Y = (Y > np.median(Y, axis=0)).astype(F32)
    elif obj == "reg:squaredlogerror":
        Y = np.abs(Y).astype(F32)
    return X, Y


def assert_doubled(vec, ref, T):
    """vec: vector model of Y = [y] * T; ref: single-target model of y."""
    assert vec.num_trees() == ref.num_trees()
    for tv, tr in zip(vec.get_trees(), ref.get_trees()):
        for k in ("left", "right", "parent", "split_feature", "split_bin", "default_left"):
            assert np.array_equal(tv[k], tr[k]), k
        internal = tr["split_feature"] >= 0
        assert np.array_equal(tv["split_cond"][internal], tr["split_cond"][internal])
        assert np.array_equal(tv["loss_chg"][internal], F32(T) * tr["loss_chg"][internal])
        leaf = ~internal
        assert tv["leaf_vector"].shape == (len(tr["left"]), T)
        for k in range(T):
            assert np.array_equal(tv["leaf_vector"][leaf, k], tr["value"][leaf])


CASES = [
    ("reg:squarederror", {}),
    ("binary:logistic", {"max_delta_step": 0.7}),
    ("reg:pseudohubererror", {"reg_alpha": 0.5}),
    ("reg:squaredlogerror", {}),
    ("reg:logistic", {"reg_lambda": 3.0}),
    ("binary:logitraw", {}),
]


@pytest.mark.parametrize("obj,extra", CASES)
@pytest.mark.parametrize("depth", [3, 8])
def test_duplicated_targets_double_the_single_target_tree(eng, obj, extra, depth):
    X, Y = dataset(obj, 1, seed=depth)
    y = Y[:, 0]
    w = np.random.RandomState(depth).uniform(0.5, 2.0, len(y)).astype(F32)
    params = dict({"objective": obj, "max_depth": depth, "eta": 0.3, "min_child_weight": 0, "gamma": 0,
                   "base_score": 0.5}, **extra)
    ref = eng.train(params, eng.DMatrix(X, label=y, weight=w), num_boost_round=4, verbose_eval=False)
    d2 = eng.DMatrix(X, label=np.stack([y, y], 1), weight=w, multi_target=True)
    vec = eng.train(dict(params, **VEC), d2, num_boost_round=4, verbose_eval=False)
    assert vec.is_vector_leaf and vec.num_boosted_rounds() == 4
    assert_doubled(vec, ref, 2)
    m = vec.predict(d2, output_margin=True)
    assert m.shape == (len(y), 2)
    r = ref.predict(eng.DMatrix(X), output_margin=True)
    assert np.array_equal(m[:, 0], r) and np.array_equal(m[:, 1], r)
    assert vec.predict(d2, training=True, output_margin=True).tobytes() == m.tobytes()


def test_duplicated_targets_deep_and_sampled(eng):
    X, Y = dataset("reg:squarederror", 1, n=20000, f=30, seed=3)
    y = Y[:, 0]
    params = {"objective": "reg:squarederror", "max_depth": 7, "eta": 0.3, "min_child_weight": 0, "gamma": 0,
              "base_score": 0.5, "subsample": 0.7, "colsample_bytree": 0.8, "colsample_bylevel": 0.9,
              "colsample_bynode": 0.8, "seed": 7}
    ref = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=3, verbose_eval=False)
    d2 = eng.DMatrix(X, label=np.stack([y, y], 1), multi_target=True)
    vec = eng.train(dict(params, **VEC), d2, num_boost_round=3, verbose_eval=False)
    assert_doubled(vec, ref, 2)


def test_interaction_constraints_duplicated(eng):
    X, Y = dataset("reg:squarederror", 1, seed=11)
    y = Y[:, 0]
    params = {"objective": "reg:squarederror", "max_depth": 5, "min_child_weight": 0, "gamma": 0, "base_score": 0.5,
              "interaction_constraints": [[0, 1, 2], [3, 4, 5, 6]]}
    ref = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=3, verbose_eval=False)
    vec = eng.train(dict(params, **VEC), eng.DMatrix(X, label=np.stack([y, y], 1), multi_target=True), num_boost_round=3,
                    verbose_eval=False)
    assert_doubled(vec, ref, 2)


@pytest.mark.parametrize("T", [2, 5, 17])
def test_margin_matches_predict_and_shapes(eng, T):
    X, Y = dataset("reg:squarederror", T, seed=T)
    d = eng.DMatrix(X, label=Y, multi_target=True)
    bst = eng.train(dict({"objective": "reg:squarederror", "max_depth": 6}, **VEC), d, num_boost_round=5,
                    verbose_eval=False)
    assert bst.num_trees() == 5 and bst.num_class == T
    m = bst.predict(d, output_margin=True)
    assert m.shape == (len(Y), T)
    assert bst.predict(d, training=True, output_margin=True).tobytes() == m.tobytes()
    # every tree adds its leaf vector: rebuild the margin from pred_leaf and the leaf vectors
    leaves = bst.predict(d, pred_leaf=True).astype(np.int64)
    assert leaves.shape == (len(Y), 5)
    acc = np.full((len(Y), T), F32(bst.params["base_score"]), F32)
    for t, tr in enumerate(bst.get_trees()):
        acc = (acc + tr["leaf_vector"][leaves[:, t]]).astype(F32)
    assert acc.tobytes() == m.tobytes()
    m2 = bst.predict(d, output_margin=True, iteration_range=(0, 2))
    acc = np.full((len(Y), T), F32(bst.params["base_score"]), F32)
    for t, tr in enumerate(bst.get_trees()[:2]):
        acc = (acc + tr["leaf_vector"][leaves[:, t]]).astype(F32)
    assert acc.tobytes() == m2.tobytes()
    assert bst.predict(d, pred_leaf=True, iteration_range=(1, 3)).shape == (len(Y), 2)
    # the loss goes down
    r0 = float(bst.eval_set([(d, "t")]).split(":")[-1])
    assert r0 < float(np.sqrt(np.mean((Y - Y.mean(0)) ** 2)))


def test_targets_train_differently_from_one_output_per_tree(eng):
    X, Y = dataset("binary:logistic", 4, seed=2)
    d = eng.DMatrix(X, label=Y, multi_target=True)
    a = eng.train({"objective": "binary:logistic", "max_depth": 4}, d, num_boost_round=3, verbose_eval=False)
    b = eng.train(dict({"objective": "binary:logistic", "max_depth": 4}, **VEC), d, num_boost_round=3, verbose_eval=False)
    assert a.num_trees() == 12 and b.num_trees() == 3
    p = b.predict(d)
    assert p.shape == (len(Y), 4) and np.all((p > 0) & (p < 1))


def test_t1_ignores_the_strategy(eng):
    X, Y = dataset("reg:squarederror", 1, seed=5)
    d = eng.DMatrix(X, label=Y[:, 0])
    a = eng.train({"objective": "reg:squarederror", "max_depth": 6}, d, num_boost_round=4, verbose_eval=False)
    b = eng.train(dict({"objective": "reg:squarederror", "max_depth": 6}, **VEC), d, num_boost_round=4, verbose_eval=False)
    assert not b.is_vector_leaf
    for ta, tb in zip(a.get_trees(), b.get_trees()):
        for k in ta:
            assert np.array_equal(ta[k], tb[k]), k
    assert np.array_equal(a.predict(d), b.predict(d))


def test_cap_64_and_65_refused(eng):
    X, Y = dataset("reg:squarederror", 65, n=3000, seed=1)
    bst = eng.train(dict({"objective": "reg:squarederror", "max_depth": 4}, **VEC),
                    eng.DMatrix(X, label=Y[:, :64], multi_target=True), num_boost_round=2, verbose_eval=False)
    assert bst.predict(eng.DMatrix(X)).shape == (3000, 64)
    with pytest.raises(eng.XGBoostError, match="at most 64 targets.*65 columns"):
        eng.train(dict({"objective": "reg:squarederror"}, **VEC), eng.DMatrix(X, label=Y, multi_target=True),
                  num_boost_round=1, verbose_eval=False)


def test_model_file_pickle_and_continuation(eng, tmp_path):
    X, Y = dataset("reg:squarederror", 3, seed=8)
    d = eng.DMatrix(X, label=Y, multi_target=True)
    params = dict({"objective": "reg:squarederror", "max_depth": 5}, **VEC)
    bst = eng.train(params, d, num_boost_round=4, verbose_eval=False)
    want = bst.predict(eng.DMatrix(X), output_margin=True)
    model = json.loads(bytes(bst.save_raw()))
    gb = model["learner"]["gradient_booster"]["model"]
    assert gb["tree_info"] == [0, 0, 0, 0] and gb["iteration_indptr"] == [0, 1, 2, 3, 4]
    assert model["learner"]["learner_model_param"]["num_target"] == "3"
    t0 = gb["trees"][0]
    n0 = int(t0["tree_param"]["num_nodes"])
    assert t0["tree_param"]["size_leaf_vector"] == "3" and len(t0["base_weights"]) == 3 * n0
    assert all(c == 0.0 for c, l in zip(t0["split_conditions"], t0["left_children"]) if l < 0)
    assert json.loads(bst.save_config())["learner"]["learner_train_param"]["multi_strategy"] == "multi_output_tree"
    assert "leaf=[" in bst.get_dump()[0]
    path = str(tmp_path / "m.json")
    bst.save_model(path)
    b2 = eng.Booster(model_file=path)
    assert b2.is_vector_leaf
    assert b2.predict(eng.DMatrix(X), output_margin=True).tobytes() == want.tobytes()
    b3 = pickle.loads(pickle.dumps(bst))
    assert b3.predict(eng.DMatrix(X), output_margin=True).tobytes() == want.tobytes()
    # continuation: 4 + 2 rounds equal 6 rounds
    full = eng.train(params, d, num_boost_round=6, verbose_eval=False)
    cont = eng.train(params, d, num_boost_round=2, xgb_model=b3, verbose_eval=False)
    assert cont.predict(eng.DMatrix(X), output_margin=True).tobytes() == \
        full.predict(eng.DMatrix(X), output_margin=True).tobytes()
    with pytest.raises(eng.XGBoostError, match="one_output_per_tree|multi_output_tree"):
        eng.train({"objective": "reg:squarederror", "max_depth": 5, "multi_strategy": "one_output_per_tree"}, d,
                  num_boost_round=1, xgb_model=b3, verbose_eval=False)
    scalar = eng.train({"objective": "reg:squarederror", "max_depth": 5}, d, num_boost_round=1, verbose_eval=False)
    with pytest.raises(eng.XGBoostError, match="one_output_per_tree"):
        eng.train(params, d, num_boost_round=1, xgb_model=scalar, verbose_eval=False)


def test_early_stopping_and_metrics(eng):
    X, Y = dataset("reg:squarederror", 2, seed=4)
    dt = eng.DMatrix(X[:4000], label=Y[:4000], multi_target=True)
    dv = eng.DMatrix(X[4000:], label=Y[4000:], multi_target=True)
    res = {}
    bst = eng.train(dict({"objective": "reg:squarederror", "max_depth": 6, "eval_metric": ["rmse", "mae"]}, **VEC), dt,
                    num_boost_round=200, evals=[(dv, "v")], evals_result=res, early_stopping_rounds=5, verbose_eval=False)
    assert bst.best_iteration < 199 and len(res["v"]["rmse"]) == bst.num_boosted_rounds()


def test_refused_combinations(eng):
    X, Y = dataset("reg:squarederror", 3, seed=6)
    d = eng.DMatrix(X, label=Y, multi_target=True)
    base = dict({"objective": "reg:squarederror", "max_depth": 3}, **VEC)
    with pytest.raises(eng.XGBoostError, match="multi_output_tree.*dart"):
        eng.train(dict(base, booster="dart"), d, num_boost_round=1, verbose_eval=False)
    with pytest.raises(eng.XGBoostError, match="multi_output_tree.*num_parallel_tree"):
        eng.train(dict(base, num_parallel_tree=2), d, num_boost_round=1, verbose_eval=False)
    with pytest.raises(eng.XGBoostError, match="multi_output_tree.*multi:softprob"):
        eng.train(dict(base, objective="multi:softprob", num_class=3), eng.DMatrix(X, label=Y[:, 0] > 0),
                  num_boost_round=1, verbose_eval=False)
    with pytest.raises(eng.XGBoostError, match="bogus"):
        eng.train(dict(base, multi_strategy="bogus"), d, num_boost_round=1, verbose_eval=False)
    bst = eng.train(base, d, num_boost_round=1, verbose_eval=False)
    with pytest.raises(eng.XGBoostError, match="pred_contribs.*vector-leaf"):
        bst.predict(d, pred_contribs=True)
    with pytest.raises(eng.XGBoostError, match="pred_interactions.*vector-leaf"):
        bst.predict(d, pred_interactions=True)
    Xc = X.copy()
    Xc[:, 0] = np.floor(np.abs(np.nan_to_num(Xc[:, 0])) * 3) % 5
    dc = eng.DMatrix(Xc, label=Y, multi_target=True, feature_types=["c"] + ["q"] * (X.shape[1] - 1),
                     enable_categorical=True)
    with pytest.raises(eng.XGBoostError, match="multi_output_tree.*categorical"):
        eng.train(base, dc, num_boost_round=1, verbose_eval=False)


def test_two_million_rows(eng):
    rng = np.random.RandomState(0)
    n = 2_000_000
    X = rng.rand(n, 8).astype(F32)
    Y = np.stack([X[:, 0] + X[:, 1], X[:, 2] - X[:, 3], np.sin(6 * X[:, 4])], 1).astype(F32)
    d = eng.DMatrix(X, label=Y, multi_target=True)
    bst = eng.train(dict({"objective": "reg:squarederror", "max_depth": 8}, **VEC), d, num_boost_round=5,
                    verbose_eval=False)
    m = bst.predict(d, output_margin=True)
    assert bst.predict(d, training=True, output_margin=True).tobytes() == m.tobytes()
    assert np.sqrt(np.mean((m - Y) ** 2)) < np.sqrt(np.mean((Y - Y.mean(0)) ** 2))


def test_public_api(eng):
    from xgboost_ray_b200 import RayDMatrix, RayParams, predict, train
    from xgboost_ray_b200.sklearn import RayXGBRegressor
    X, Y = dataset("reg:squarederror", 3, seed=9)
    dm = RayDMatrix(X, Y)
    bst = train(dict({"objective": "reg:squarederror", "max_depth": 4}, **VEC), dm, num_boost_round=3,
                ray_params=RayParams(num_actors=1))
    assert bst.num_trees() == 3 and bst.is_vector_leaf
    assert predict(bst, RayDMatrix(X), ray_params=RayParams(num_actors=1)).shape == (len(Y), 3)
    reg = RayXGBRegressor(n_estimators=3, max_depth=4, multi_strategy="multi_output_tree")
    reg.fit(X, Y)
    assert reg.get_booster().num_trees() == 3
    assert reg.predict(X).shape == (len(Y), 3)


# ---- distinct targets against tests/multi_output_reference.py (the rules of DESIGN.md 2 item 19 restated in NumPy)
from tests import multi_output_reference as MO  # noqa: E402


@pytest.mark.parametrize("obj", [c[0] for c in CASES])
@pytest.mark.parametrize("T,depth", [(2, 14), (5, 8), (17, 3)])
def test_matches_reference(eng, obj, T, depth):
    X, Y = dataset(obj, T, n=5000, seed=T + depth, nan_frac=0.05)
    w = np.random.RandomState(T).uniform(0.5, 2.0, len(Y)).astype(F32)
    params = dict({"objective": obj, "max_depth": depth, "eta": 0.3, "min_child_weight": 0.5}, **VEC)
    d = eng.DMatrix(X, label=Y, weight=w, multi_target=True)
    bst = eng.train(params, d, num_boost_round=3, verbose_eval=False)
    ref = MO.train(params, X, Y, 3, weight=w)
    assert F32(bst.params["base_score"]) == F32(ref.base_score)
    MO.assert_engine_matches(bst, ref)
    m = bst.predict(d, training=True, output_margin=True)
    assert m.shape == (len(Y), T) and m.tobytes() == ref.margin.tobytes()


def test_sampling_constraints_and_base_margin_match_reference(eng):
    X, Y = dataset("reg:squarederror", 3, n=6000, f=12, seed=21)
    fw = np.linspace(0.2, 3.0, X.shape[1]).astype(F32)
    bm = np.random.RandomState(3).normal(0, 0.5, Y.shape).astype(F32)
    params = dict({"objective": "reg:squarederror", "max_depth": 6, "base_score": 0.5, "colsample_bytree": 0.8,
                   "colsample_bylevel": 0.8, "colsample_bynode": 0.7, "seed": 5,
                   "interaction_constraints": [[0, 1, 2, 3], [3, 4, 5, 6, 7, 8]]}, **VEC)
    d = eng.DMatrix(X, label=Y, base_margin=bm, multi_target=True)
    d.set_info(feature_weights=fw)
    bst = eng.train(params, d, num_boost_round=3, verbose_eval=False)
    ref = MO.train(params, X, Y, 3, sets=params["interaction_constraints"], feature_weights=fw, base_margin=bm)
    MO.assert_engine_matches(bst, ref)
    assert bst.predict(d, training=True, output_margin=True).tobytes() == ref.margin.tobytes()


def test_custom_objective_and_min_child_weight_match_reference(eng):
    # target 1's hessians are 0.05 per row: with min_child_weight = 2 a child of fewer than 40 rows adds nothing for it
    X, Y = dataset("reg:squarederror", 2, n=3000, seed=13)
    scale = np.array([1.0, 0.05], F32)

    def grads(margin):
        g = ((margin - Y) * scale).astype(F32)
        return g, np.broadcast_to(scale, g.shape).astype(F32)

    params = dict({"max_depth": 8, "min_child_weight": 2.0, "base_score": 0.0}, **VEC)
    d = eng.DMatrix(X, label=Y, multi_target=True)
    bst = eng.train(params, d, num_boost_round=3, obj=lambda p, dm: grads(np.asarray(p, F32).reshape(Y.shape)),
                    verbose_eval=False)
    ref = MO.train(params, X, Y, 3, gradients=grads)
    MO.assert_engine_matches(bst, ref)
    assert any(np.any(t.leaf_vector[t.split_feature < 0, 1] == 0) for t in ref._trees)


def test_one_vs_two_gpus(eng):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    X, Y = dataset("reg:squarederror", 3, n=30001, seed=47)
    params = dict({"objective": "reg:squarederror", "max_depth": 6}, **VEC)
    b1 = train(params, RayDMatrix(X, Y), num_boost_round=4, ray_params=RayParams(num_actors=1))
    b2 = train(params, RayDMatrix(X, Y), num_boost_round=4, ray_params=RayParams(num_actors=2))
    assert b1.is_vector_leaf and bytes(b1.save_raw()) == bytes(b2.save_raw())
