"""Multi-target regression and multi-label classification (a label of T > 1 columns) on the GPU.

Models are compared with tests/multi_target_reference.py (the oracle grows every round's T trees from the per-column
gradients): the trees with assert_same_model, the intercept exactly, the metrics within 1e-9 relative.  Also the engine
against itself (tree k equals the single-target model of column k), T = 1 staying byte-identical, prediction shapes,
the model file, continuation, the public API and the refused combinations."""
import pickle

import numpy as np
import pytest

from tests import multi_target_reference as R
from tests.test_gpu_parity import IS_CAT, assert_same_model, make_cat_data, make_data

pytestmark = pytest.mark.gpu
F32 = np.float32


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def dataset(obj, T, n=5000, f=10, seed=0, nan_frac=0.0):
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


def same_as_reference(oracle, bst, params, X, Y, rounds, weight=None, is_cat=None, base_margin=None):
    ref = R.train(oracle, params, X, Y, rounds, weight=weight, is_cat=is_cat, base_margin=base_margin)
    assert_same_model(bst, ref)
    if params.get("base_score") is None:
        assert F32(bst.params["base_score"]) == F32(ref.base_score)
    return ref


@pytest.mark.parametrize("obj", R.MULTI_TARGET_OBJECTIVES)
@pytest.mark.parametrize("T", [2, 5, 17])
def test_matches_reference(eng, oracle, obj, T):
    depth = 3 if T != 5 else 8
    X, Y = dataset(obj, T, seed=T, nan_frac=0.05)
    w = np.random.RandomState(T).uniform(0.5, 2.0, len(Y)).astype(F32)
    params = {"objective": obj, "max_depth": depth, "eta": 0.3}
    d = eng.DMatrix(X, label=Y, multi_target=True, weight=w)
    bst = eng.train(params, d, num_boost_round=4, verbose_eval=False)
    assert bst.num_class == T and bst.num_trees() == 4 * T
    ref = same_as_reference(oracle, bst, params, X, Y, 4, weight=w)
    m = bst.predict(d, output_margin=True)
    assert m.shape == (len(Y), T)
    assert np.array_equal(m, ref.predict_margin(X))
    assert bst.predict(d, training=True, output_margin=True).tobytes() == ref.margin.tobytes()
    p = bst.predict(d)
    assert p.shape == (len(Y), T)
    if obj in ("binary:logistic", "reg:logistic"):
        assert np.allclose(p, 1 / (1 + np.exp(-m.astype(np.float64))), rtol=1e-6, atol=1e-7)
    else:
        assert np.array_equal(p, m)


@pytest.mark.parametrize("variant", ["categorical", "subsample", "colsample_bynode", "scale_pos_weight"])
def test_variants_match_reference(eng, oracle, variant):
    obj = "binary:logistic" if variant == "scale_pos_weight" else "reg:squarederror"
    params = {"objective": obj, "max_depth": 5, "eta": 0.3}
    is_cat = None
    if variant == "categorical":
        X = make_cat_data(4000, 1)[0]
        is_cat = IS_CAT
        _, Y = dataset(obj, 3, n=len(X), seed=7)
    else:
        X, Y = dataset(obj, 3, n=4000, seed=7)
    if variant == "subsample":
        params.update(subsample=0.7, seed=5)
    elif variant == "colsample_bynode":
        params.update(colsample_bynode=0.5, seed=6)
    elif variant == "scale_pos_weight":
        params["scale_pos_weight"] = 2.5
    ft = ["c" if c else "q" for c in is_cat] if is_cat is not None else None
    d = eng.DMatrix(X, label=Y, multi_target=True, feature_types=ft, enable_categorical=is_cat is not None)
    bst = eng.train(params, d, num_boost_round=4, verbose_eval=False)
    same_as_reference(oracle, bst, params, X, Y, 4, is_cat=is_cat)


def test_single_column_label_is_unchanged(eng):
    for obj in ("reg:squarederror", "binary:logistic", "reg:pseudohubererror"):
        X, Y = dataset(obj, 1, seed=11)
        params = {"objective": obj, "max_depth": 6}
        a = eng.train(params, eng.DMatrix(X, label=Y[:, 0]), num_boost_round=5, verbose_eval=False)
        b = eng.train(params, eng.DMatrix(X, label=Y), num_boost_round=5, verbose_eval=False)
        assert bytes(a.save_raw()) == bytes(b.save_raw())
        assert "num_target" not in b.params


@pytest.mark.parametrize("obj,npt", [("reg:squarederror", 1), ("binary:logistic", 1), ("reg:squarederror", 2)])
def test_tree_k_is_the_single_target_model_of_column_k(eng, obj, npt):
    """Without row sampling the trees of target k are the single-target model of column k; with num_parallel_tree the
    npt trees of target k sit next to each other, as for multi-class models (subsample < 1 keys each tree's sample by
    its index in the model, so it is left out here)."""
    X, Y = dataset(obj, 4, seed=13)
    params = {"objective": obj, "max_depth": 6, "base_score": 0.5, "num_parallel_tree": npt, "colsample_bynode": 1.0}
    multi = eng.train(params, eng.DMatrix(X, label=Y, multi_target=True), num_boost_round=5, verbose_eval=False).get_trees()
    for k in range(4):
        single = eng.train(params, eng.DMatrix(X, label=Y[:, k]), num_boost_round=5, verbose_eval=False).get_trees()
        for r in range(5 * npt):
            t, s = multi[(r // npt) * 4 * npt + k * npt + r % npt], single[r]
            for f in ("left", "split_feature", "split_bin", "value", "loss_chg"):
                assert t[f].tobytes() == s[f].tobytes(), (k, r, f)


def test_non_finite_round_fails(eng):
    # margins clamped near -1 give |g| ~ 1e7, |h| ~ 1e13; weights of 1e30 push the pairs past FLT_MAX
    X, Y = dataset("reg:squaredlogerror", 3, seed=17)
    d = eng.DMatrix(X, label=Y, multi_target=True, weight=np.full(len(Y), 1e30, F32), base_margin=np.full(Y.shape, -5.0, F32))
    with pytest.raises(eng.XGBoostError, match="not finite"):
        eng.train({"objective": "reg:squaredlogerror", "base_score": 0.5}, d, num_boost_round=1, verbose_eval=False)


@pytest.mark.parametrize("obj,metrics", [("reg:squarederror", ["rmse", "mae", "mape"]),
                                         ("binary:logistic", ["logloss", "error"]),
                                         ("reg:squaredlogerror", ["rmsle"]),
                                         ("reg:pseudohubererror", ["mphe"])])
def test_metrics(eng, obj, metrics):
    X, Y = dataset(obj, 3, seed=19)
    if obj == "reg:squarederror":
        Y = Y + F32(5.0)     # mape divides by the label
    w = np.random.RandomState(2).uniform(0.5, 2.0, len(Y)).astype(F32)
    d = eng.DMatrix(X, label=Y, multi_target=True, weight=w)
    bst = eng.train({"objective": obj, "max_depth": 4, "eval_metric": metrics}, d, num_boost_round=3, verbose_eval=False)
    m = bst.predict(d, output_margin=True)
    import ctypes as C
    for name in metrics:
        v = C.c_double(0)
        eng._check(eng.lib().B2_BoosterEvalSet(bst.handle, d.handle, name.encode(), C.byref(v)))
        want = R.metric(name, obj, m, Y, w, bst.params)
        assert abs(v.value - want) <= 1e-9 * max(1.0, abs(want)), (name, v.value, want)
    for name in ("auc", "aucpr"):
        with pytest.raises(eng.XGBoostError, match="multi-target"):
            eng.train({"objective": obj, "eval_metric": name}, d, num_boost_round=1, evals=[(d, "train")],
                      verbose_eval=False)


def test_prediction_shapes_and_shap(eng):
    X, Y = dataset("reg:squarederror", 3, n=2000, f=6, seed=23)
    d = eng.DMatrix(X, label=Y, multi_target=True)
    bst = eng.train({"objective": "reg:squarederror", "max_depth": 4}, d, num_boost_round=4, verbose_eval=False)
    m = bst.predict(d, output_margin=True)
    assert bst.predict(d, pred_leaf=True).shape == (len(Y), 4 * 3)
    c = bst.predict(d, pred_contribs=True)
    assert c.shape == (len(Y), 3, X.shape[1] + 1)
    assert np.max(np.abs(c.sum(axis=2) - m)) <= 1e-4
    assert bst.predict(d, pred_interactions=True).shape == (len(Y), 3, X.shape[1] + 1, X.shape[1] + 1)
    part = bst.predict(d, output_margin=True, iteration_range=(0, 2))
    full2 = eng.train({"objective": "reg:squarederror", "max_depth": 4, "base_score": bst.params["base_score"]},
                      d, num_boost_round=2, verbose_eval=False).predict(d, output_margin=True)
    assert np.array_equal(part, full2)


def test_base_margin_custom_objective_and_dart(eng, oracle):
    X, Y = dataset("reg:squarederror", 3, seed=29)
    bm = np.random.RandomState(4).normal(0, 1, Y.shape).astype(F32)
    params = {"objective": "reg:squarederror", "max_depth": 5, "base_score": 0.5}
    bst = eng.train(params, eng.DMatrix(X, label=Y, multi_target=True, base_margin=bm), num_boost_round=3, verbose_eval=False)
    same_as_reference(oracle, bst, params, X, Y, 3, base_margin=bm)

    def sq(pred, dm):
        return (pred - dm.get_label()).astype(F32), np.ones_like(pred)
    d = eng.DMatrix(X, label=Y, multi_target=True)
    builtin = eng.train(params, d, num_boost_round=3, verbose_eval=False)
    custom = eng.train(params, eng.DMatrix(X, label=Y, multi_target=True), num_boost_round=3, obj=sq, verbose_eval=False)
    for a, b in zip(builtin.get_trees(), custom.get_trees()):
        assert a["value"].tobytes() == b["value"].tobytes()
    dart = eng.train(dict(params, booster="dart", rate_drop=0.0), eng.DMatrix(X, label=Y, multi_target=True), num_boost_round=3,
                     verbose_eval=False)
    assert np.array_equal(dart.predict(d, output_margin=True), builtin.predict(d, output_margin=True))


def test_model_file_pickle_and_continuation(eng, tmp_path):
    import jsonschema
    from tests.model_schema import MODEL
    X, Y = dataset("binary:logistic", 4, seed=31)
    d = eng.DMatrix(X, label=Y, multi_target=True)
    params = {"objective": "binary:logistic", "max_depth": 5}
    full = eng.train(params, d, num_boost_round=6, verbose_eval=False)
    raw = bytes(full.save_raw())
    import json
    j = json.loads(raw)
    jsonschema.validate(j, MODEL)
    lmp = j["learner"]["learner_model_param"]
    assert lmp["num_target"] == "4" and lmp["num_class"] == "0"
    assert j["learner"]["gradient_booster"]["model"]["tree_info"] == [t % 4 for t in range(24)]
    path = str(tmp_path / "m.json")
    full.save_model(path)
    loaded = eng.Booster(model_file=path)
    assert loaded.num_class == 4 and bytes(loaded.save_raw()) == raw
    assert np.array_equal(loaded.predict(d), full.predict(d))
    assert np.array_equal(pickle.loads(pickle.dumps(full)).predict(d), full.predict(d))
    first = eng.train(params, d, num_boost_round=3, verbose_eval=False)
    cont = eng.train(params, d, num_boost_round=3, verbose_eval=False, xgb_model=first)
    assert bytes(cont.save_raw()) == raw
    with pytest.raises(eng.XGBoostError, match="targets"):
        eng.train(params, eng.DMatrix(X, label=Y[:, :2], multi_target=True), num_boost_round=1, verbose_eval=False, xgb_model=first)


def test_two_million_rows(eng, oracle):
    X, Y = dataset("reg:squarederror", 4, n=2_000_000, f=8, seed=37)
    params = {"objective": "reg:squarederror", "max_depth": 6}
    bst = eng.train(params, eng.DMatrix(X, label=Y, multi_target=True), num_boost_round=2, verbose_eval=False)
    same_as_reference(oracle, bst, params, X, Y, 2)


def test_refused_combinations(eng):
    X, Y = dataset("reg:squarederror", 2, n=500, seed=41)
    d = eng.DMatrix(X, label=Y, multi_target=True)
    for params, match in (({"objective": "count:poisson"}, "count:poisson"), ({"objective": "multi:softprob",
                          "num_class": 2}, "multi:softprob"), ({"objective": "reg:quantileerror"}, "quantileerror"),
                          ({"objective": "reg:squarederror", "num_class": 2}, "num_class")):
        with pytest.raises(eng.XGBoostError, match=match):
            eng.train(params, d, num_boost_round=1, verbose_eval=False)
    with pytest.raises(eng.XGBoostError, match="query groups"):
        eng.DMatrix(X, label=Y, multi_target=True, qid=np.repeat(np.arange(50), 10))
    with pytest.raises(eng.XGBoostError, match="4096"):
        eng.DMatrix(X[:2], label=np.zeros((2, 4097), F32), multi_target=True)
    bst = eng.train({"objective": "reg:squarederror"}, d, num_boost_round=1, verbose_eval=False)
    with pytest.raises(eng.XGBoostError, match="columns"):
        bst.eval_set([(eng.DMatrix(X, label=Y[:, 0]), "eval")])


def test_label_of_several_columns_needs_multi_target(eng):
    """A 2-D label is trained as T outputs only when asked for: without multi_target=True it is refused (a one-hot
    class label or a target passed twice is not silently fitted as independent columns); (n, 1) is a plain label."""
    X, Y = dataset("reg:squarederror", 2, n=500, seed=16)
    with pytest.raises(eng.XGBoostError, match="multi_target=True"):
        eng.DMatrix(X, label=Y)
    d = eng.DMatrix(X, label=Y[:, :1])
    with pytest.raises(eng.XGBoostError, match="multi_target=True"):
        d.set_info(label=Y)
    assert d.get_label().shape == (len(Y),)
    # reg:quantileerror's outputs are its alphas: a label of two columns is refused at training
    with pytest.raises(eng.XGBoostError, match="2 columns"):
        eng.train({"objective": "reg:quantileerror"}, eng.DMatrix(X, label=Y, multi_target=True), num_boost_round=1,
                  verbose_eval=False)


def same_trees(a, b):
    ta, tb = a.get_trees(), b.get_trees()
    assert len(ta) == len(tb)
    for x, y in zip(ta, tb):
        for f in ("left", "split_feature", "split_bin", "split_cond", "value"):
            assert x[f].tobytes() == y[f].tobytes(), f


def test_public_api_and_sklearn(eng, tmp_path):
    import pandas as pd
    from xgboost_ray_b200 import RayDMatrix, RayParams, predict, train
    from xgboost_ray_b200.sklearn import RayXGBClassifier, RayXGBRegressor
    X, Y = dataset("reg:squarederror", 3, n=6000, f=6, seed=43)
    params = {"objective": "reg:squarederror", "max_depth": 5}
    ref = eng.train(params, eng.DMatrix(X, label=Y, multi_target=True), num_boost_round=4, verbose_eval=False)
    want = ref.predict(eng.DMatrix(X), output_margin=True)
    df = pd.DataFrame(np.column_stack([X, Y]), columns=["f%d" % i for i in range(6)] + ["y0", "y1", "y2"])
    for label, data in ((Y, X), (pd.DataFrame(Y), X), (["y0", "y1", "y2"], df)):
        bst = train(params, RayDMatrix(data, label), num_boost_round=4, ray_params=RayParams(num_actors=1))
        same_trees(bst, ref)
        got = predict(bst, RayDMatrix(X), ray_params=RayParams(num_actors=1))
        assert got.shape == (len(Y), 3) and np.array_equal(got, want)
    pq = str(tmp_path / "d.parquet")
    df.to_parquet(pq)
    bst = train(params, RayDMatrix([pq], ["y0", "y1", "y2"], distributed=False), num_boost_round=4,
                ray_params=RayParams(num_actors=1))
    same_trees(bst, ref)
    reg = RayXGBRegressor(n_estimators=4, max_depth=5).fit(X, Y)
    assert reg.predict(X).shape == (len(Y), 3)
    L = (Y > np.median(Y, axis=0)).astype(np.int64)
    clf = RayXGBClassifier(n_estimators=4, max_depth=5).fit(X, L)
    assert clf.n_classes_ == 2 and list(clf.classes_) == [0, 1]
    p = clf.predict_proba(X)
    assert p.shape == L.shape
    assert np.array_equal(clf.predict(X), (p > 0.5).astype(np.int64))
    with pytest.raises(ValueError, match="0 or 1"):
        RayXGBClassifier(n_estimators=1).fit(X, L * 2)


@pytest.mark.timeout(300)
def test_two_actors_same_model(eng):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    X, Y = dataset("reg:squarederror", 3, n=30001, seed=47)
    params = {"objective": "reg:squarederror", "max_depth": 6}
    b1 = train(params, RayDMatrix(X, Y), num_boost_round=4, ray_params=RayParams(num_actors=1))
    b2 = train(params, RayDMatrix(X, Y), num_boost_round=4, ray_params=RayParams(num_actors=2))
    assert bytes(b1.save_raw()) == bytes(b2.save_raw())
