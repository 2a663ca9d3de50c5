"""GPU checks of the Poisson, Tweedie, gamma, pseudo-Huber, squared-log and logistic-variant objectives: trees identical
to the oracle grown from the gradients of tests/objective_reference.py, metrics, save / load, continuation, the public
API, SHAP, multi-GPU identity and the failure modes."""
import copy
import json

import jsonschema
import numpy as np
import pytest

from tests import objective_reference as R
from tests.golden.make_golden_objectives import CASES as OBJECTIVE_CASES, case_data
from tests.model_schema import MODEL
from tests.test_gpu_parity import assert_same_model, make_data

pytestmark = pytest.mark.gpu

NEW_OBJECTIVES = list(R.OBJECTIVES)
OBJ_PARAMS = {"reg:pseudohubererror": {"huber_slope": 1.5}, "reg:tweedie": {"tweedie_variance_power": 1.4}}
METRICS = {"reg:logistic": ["rmse", "logloss"], "binary:logitraw": ["logloss"],
           "reg:squaredlogerror": ["rmsle", "rmse"], "reg:pseudohubererror": ["mphe", "mae"],
           "count:poisson": ["poisson-nloglik", "rmse"], "reg:gamma": ["gamma-nloglik", "gamma-deviance", "mape"],
           "reg:tweedie": ["tweedie-nloglik@1.4", "rmse"]}


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def labels(obj, X, rng):
    """Labels in the objective's domain that depend on the first features (missing values count as 0)."""
    x = np.nan_to_num(X.astype(np.float64))
    s = 0.3 * x[:, 0] - 0.2 * x[:, 1] + 0.1 * x[:, 2] - 0.5
    if obj in ("reg:logistic", "binary:logitraw"):
        y = 1.0 / (1.0 + np.exp(-s))
        y[::4] = (y[::4] > 0.5)
    elif obj == "reg:squaredlogerror":
        y = np.exp(0.5 * s) - 0.2 + rng.uniform(0, 0.3, len(s))
    elif obj == "reg:pseudohubererror":
        y = 3 * s + rng.standard_t(2, len(s))
    elif obj == "reg:gamma":
        y = rng.gamma(2.0, np.exp(s) / 2.0)
        y = np.maximum(y, 1e-3)
    elif obj == "count:poisson":
        y = rng.poisson(np.exp(s))
    else:
        c = rng.poisson(np.exp(0.5 * s))
        y = np.array([rng.gamma(2.0, 1.0, size=k).sum() for k in c])
    return y.astype(np.float32)


def metric_close(a, b):
    return abs(a - b) <= 1e-6 * max(1.0, abs(b))


@pytest.mark.parametrize("obj", NEW_OBJECTIVES)
@pytest.mark.parametrize("variant", ["estimated", "missing_weights", "categorical", "subsample_given"])
def test_trees_and_metrics_identical_to_oracle(eng, oracle, obj, variant):
    rng = np.random.RandomState(NEW_OBJECTIVES.index(obj) + 7)
    n, f = 6000, 8
    X = make_data(n, f, 31, "uniform", nan_frac=0.1 if variant == "missing_weights" else 0.0)
    is_cat, kw = None, {}
    if variant == "categorical":
        X[:, 3] = rng.randint(0, 3, n)
        X[:, 4] = rng.randint(0, 20, n)
        is_cat = [0, 0, 0, 1, 1, 0, 0, 0]
        kw = {"feature_types": ["q" if c == 0 else "c" for c in is_cat], "enable_categorical": True}
    y = labels(obj, X, rng)
    if variant == "categorical":
        y = np.where(X[:, 4] % 3 == 0, y * 2 if obj not in ("reg:logistic", "binary:logitraw") else 1 - y, y).astype(np.float32)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32) if variant == "missing_weights" else None
    params = dict(OBJ_PARAMS.get(obj, {}), objective=obj, max_depth=5, eta=0.3, eval_metric=METRICS[obj])
    if variant == "subsample_given":
        params.update(subsample=0.7, seed=5, base_score={"reg:logistic": 0.4, "binary:logitraw": 0.1}.get(obj, 1.2))
    rounds = 4
    obst = R.train(oracle, params, X, y, rounds, weight=w, is_cat=is_cat)
    dm = eng.DMatrix(X, label=y, weight=w, **kw)
    res = {}
    ebst = eng.train(params, dm, num_boost_round=rounds, evals=[(dm, "train")], evals_result=res, verbose_eval=False)
    if "base_score" not in params:
        assert np.float32(ebst.params["base_score"]) == np.float32(obst.base_score)
    assert_same_model(ebst, obst)
    m = ebst.predict(dm, output_margin=True, training=True)
    assert np.max(np.abs(m - obst.margin)) <= 1e-5 * max(1.0, float(np.max(np.abs(obst.margin))))
    for name in METRICS[obj]:
        want = obst.metric(name, obst.margin, y, w)
        assert metric_close(res["train"][name][-1], want), (name, res["train"][name][-1], want)
    Xt = make_data(2000, f, 99, "uniform")
    if variant == "categorical":
        Xt[:, 3] = rng.randint(0, 3, 2000)
        Xt[:, 4] = rng.randint(0, 20, 2000)
    pe, po = ebst.predict(eng.DMatrix(Xt, **kw)), obst.predict(Xt)
    assert np.max(np.abs(pe - po) / np.maximum(1.0, np.abs(po))) <= 1e-5


def test_default_metric_and_objective_parameters(eng):
    rng = np.random.RandomState(2)
    X = make_data(3000, 5, 4, "uniform")
    for obj, want in (("count:poisson", "poisson-nloglik"), ("reg:gamma", "gamma-nloglik"),
                      ("reg:tweedie", "tweedie-nloglik@1.4"), ("reg:pseudohubererror", "mphe"),
                      ("reg:squaredlogerror", "rmsle"), ("reg:logistic", "rmse"), ("binary:logitraw", "logloss")):
        dm = eng.DMatrix(X, label=labels(obj, X, rng))
        res = {}
        eng.train(dict(OBJ_PARAMS.get(obj, {}), objective=obj), dm, 2, evals=[(dm, "t")], evals_result=res, verbose_eval=False)
        assert list(res["t"]) == [want], obj
    dm = eng.DMatrix(X, label=labels("reg:tweedie", X, rng))
    for bad in ({"objective": "reg:tweedie", "tweedie_variance_power": 2.0},
                {"objective": "reg:pseudohubererror", "huber_slope": 0.0},
                {"objective": "count:poisson", "base_score": -1.0}):
        with pytest.raises(eng.XGBoostError):
            eng.train(bad, dm, 1, verbose_eval=False)
    with pytest.raises(eng.XGBoostError, match="unsupported objective"):
        eng.train({"objective": "reg:absoluteerror"}, dm, 1, verbose_eval=False)


def test_poisson_max_delta_step_default_and_override(eng, oracle):
    rng = np.random.RandomState(3)
    X = make_data(4000, 6, 8, "uniform")
    y = labels("count:poisson", X, rng)
    for extra in ({}, {"max_delta_step": 0.2}):
        params = dict(extra, objective="count:poisson", max_depth=4, base_score=0.5)
        obst = R.train(oracle, params, X, y, 3)
        ebst = eng.train(params, eng.DMatrix(X, label=y), 3, verbose_eval=False)
        assert_same_model(ebst, obst)
        leaves = np.concatenate([t["value"][t["split_feature"] < 0] for t in ebst.get_trees()])
        assert np.max(np.abs(leaves)) <= 0.3 * extra.get("max_delta_step", 0.7) + 1e-6   # eta * clamp


@pytest.mark.parametrize("obj,bad,msg", [("count:poisson", -1.0, "label must be nonnegative for count:poisson"),
                                         ("reg:gamma", 0.0, "label must be positive for reg:gamma"),
                                         ("reg:tweedie", -2.0, "label must be nonnegative for reg:tweedie"),
                                         ("reg:logistic", 2.0, r"label must be in \[0, 1\] for reg:logistic"),
                                         ("reg:squaredlogerror", -1.0, "label must be greater than -1")])
def test_label_domain_errors(eng, obj, bad, msg):
    X = make_data(500, 3, 1, "uniform")
    y = np.full(500, 0.5, np.float32)
    y[123] = bad
    with pytest.raises(eng.XGBoostError, match=msg):
        eng.train({"objective": obj}, eng.DMatrix(X, label=y), 2, verbose_eval=False)


def test_gamma_nonfinite_gradient_fails_the_round(eng):
    """A margin of -200 underflows exp: y / exp(margin) is infinite, and the round must fail instead of growing a tree."""
    X = make_data(2000, 4, 2, "uniform")
    y = np.full(2000, 2.0, np.float32)
    dm = eng.DMatrix(X, label=y, base_margin=np.full(2000, -200.0, np.float32))
    with pytest.raises(eng.XGBoostError, match="not finite"):
        eng.train({"objective": "reg:gamma", "base_score": 1.0}, dm, 2, verbose_eval=False)
    # the same data with a sane margin trains
    ok = eng.train({"objective": "reg:gamma", "base_score": 1.0}, eng.DMatrix(X, label=y), 2, verbose_eval=False)
    assert ok.num_trees() == 2


@pytest.mark.parametrize("obj", ["count:poisson", "reg:tweedie", "reg:gamma", "reg:pseudohubererror", "reg:logistic"])
def test_save_load_predict_and_schema(eng, obj, tmp_path):
    rng = np.random.RandomState(4)
    X = make_data(3000, 6, 6, "uniform")
    y = labels(obj, X, rng)
    params = dict(OBJ_PARAMS.get(obj, {}), objective=obj, max_depth=4, scale_pos_weight=1.5)
    bst = eng.train(params, eng.DMatrix(X, label=y), 3, verbose_eval=False)
    path = str(tmp_path / "m.json")
    bst.save_model(path)
    d = json.load(open(path))
    schema = copy.deepcopy(MODEL)
    s = lambda k: {"type": "object", "properties": {k: {"type": "string"}}, "required": [k], "additionalProperties": False}  # noqa: E731
    schema["properties"]["learner"]["properties"]["objective"]["oneOf"] += [
        {"type": "object", "properties": {"name": {"const": "count:poisson"}, "poisson_regression_param": s("max_delta_step")},
         "required": ["name", "poisson_regression_param"], "additionalProperties": False},
        {"type": "object", "properties": {"name": {"const": "reg:tweedie"},
                                          "tweedie_regression_param": s("tweedie_variance_power")},
         "required": ["name", "tweedie_regression_param"], "additionalProperties": False},
        {"type": "object", "properties": {"name": {"const": "reg:pseudohubererror"}, "pseudo_huber_param": s("huber_slope")},
         "required": ["name", "pseudo_huber_param"], "additionalProperties": False},
        {"type": "object", "properties": {"name": {"const": "reg:gamma"}}, "required": ["name"], "additionalProperties": False},
        {"type": "object", "properties": {"name": {"enum": ["reg:squaredlogerror"]}, "reg_loss_param": s("scale_pos_weight")},
         "required": ["name", "reg_loss_param"], "additionalProperties": False},
    ]
    jsonschema.validate(d, schema)
    block = d["learner"]["objective"]
    if obj == "count:poisson":
        assert block["poisson_regression_param"] == {"max_delta_step": "0.7"}
    elif obj == "reg:tweedie":
        assert block["tweedie_regression_param"] == {"tweedie_variance_power": "1.4"}
    elif obj == "reg:pseudohubererror":
        assert block["pseudo_huber_param"] == {"huber_slope": "1.5"}
    elif obj == "reg:gamma":
        assert block == {"name": "reg:gamma"}
    else:
        assert block["reg_loss_param"] == {"scale_pos_weight": "1.5"}
    loaded = eng.Booster(model_file=path)
    Xt = eng.DMatrix(make_data(1000, 6, 60, "uniform"))
    assert np.array_equal(bst.predict(Xt).view(np.uint32), loaded.predict(Xt).view(np.uint32))
    assert np.array_equal(bst.predict(Xt, output_margin=True).view(np.uint32),
                          loaded.predict(Xt, output_margin=True).view(np.uint32))
    for k in ("tweedie_variance_power", "huber_slope"):
        if k in params:
            assert float(loaded.params[k]) == params[k]
    # a stock xgboost model carries only the objective block: it alone restores the parameter
    del d["learner"]["attributes"]["b2.params"]
    again = eng.Booster(model_file=bytearray(json.dumps(d).encode()))
    assert np.array_equal(bst.predict(Xt).view(np.uint32), again.predict(Xt).view(np.uint32))


@pytest.mark.parametrize("obj", ["count:poisson", "reg:tweedie"])
def test_continuation_from_saved_model_equals_uninterrupted(eng, oracle, obj, tmp_path):
    rng = np.random.RandomState(5)
    X = make_data(5000, 6, 9, "uniform")
    y = labels(obj, X, rng)
    params = dict(OBJ_PARAMS.get(obj, {}), objective=obj, max_depth=4)
    dm = eng.DMatrix(X, label=y)
    first = eng.train(params, dm, 3, verbose_eval=False)
    path = str(tmp_path / "m.json")
    first.save_model(path)
    cont = eng.train(params, eng.DMatrix(X, label=y), 2, xgb_model=path, verbose_eval=False)
    obst = R.train(oracle, params, X, y, 5)
    assert_same_model(cont, obst)


@pytest.mark.parametrize("name", OBJECTIVE_CASES)
def test_engine_reproduces_objective_golden(eng, name):
    import os
    want = json.load(open(os.path.join(os.path.dirname(__file__), "golden", name + ".json")))
    x, y, w, params, rounds = case_data(name)
    dm = eng.DMatrix(x, label=y, weight=w)
    bst = eng.train(params, dm, num_boost_round=rounds, verbose_eval=False)
    trees = bst.get_trees()
    assert len(trees) == len(want["trees"])
    for t, g in zip(trees, want["trees"]):
        for k in ("left", "right", "split_feature", "split_bin", "default_left"):
            assert [int(v) for v in t[k]] == g[k], k
        leaf = np.asarray(g["split_feature"]) < 0
        assert np.max(np.abs(t["value"][leaf] - np.asarray(g["value"], np.float32)[leaf])) <= 1e-5
    pred = np.asarray(bst.predict(eng.DMatrix(x[:64])), np.float64)
    ref = np.asarray(want["pred_head"])
    assert np.max(np.abs(pred - ref) / np.maximum(1.0, np.abs(ref))) <= 1e-5


def test_poisson_pred_contribs_sum_to_margin(eng):
    rng = np.random.RandomState(6)
    X = make_data(3000, 6, 10, "uniform", nan_frac=0.05)
    bst = eng.train({"objective": "count:poisson", "max_depth": 5}, eng.DMatrix(X, label=labels("count:poisson", X, rng)), 5,
                    verbose_eval=False)
    d = eng.DMatrix(X[:500])
    c = bst.predict(d, pred_contribs=True)
    m = bst.predict(d, output_margin=True)
    assert c.shape == (500, 7)
    assert np.max(np.abs(c.sum(axis=1) - m)) <= 1e-5 * max(1.0, float(np.max(np.abs(m))))
    assert np.allclose(np.exp(m.astype(np.float64)), bst.predict(d), rtol=1e-5)


@pytest.mark.parametrize("num_actors", [1, 2])
def test_public_train_predict_and_regressor(eng, oracle, num_actors):
    if num_actors > eng.device_count():
        pytest.skip("needs %d GPUs" % num_actors)
    from sklearn.base import clone
    from xgboost_ray_b200 import RayDMatrix, RayParams, predict, train
    from xgboost_ray_b200.sklearn import RayXGBRegressor
    rng = np.random.RandomState(7)
    X = make_data(6001, 6, 12, "uniform")
    y = labels("reg:tweedie", X, rng)
    params = {"objective": "reg:tweedie", "tweedie_variance_power": 1.4, "max_depth": 4, "eta": 0.3}
    bst = train(params, RayDMatrix(X, y), num_boost_round=4, ray_params=RayParams(num_actors=num_actors))
    ob = R.train(oracle, params, X, y, 4)
    assert_same_model(bst, ob)
    p = predict(bst, RayDMatrix(X), ray_params=RayParams(num_actors=num_actors))
    assert np.max(np.abs(p - ob.predict(X)) / np.maximum(1.0, ob.predict(X))) <= 1e-5
    reg = RayXGBRegressor(n_estimators=4, max_depth=4, objective="reg:tweedie", tweedie_variance_power=1.4, n_jobs=num_actors)
    assert reg.get_params()["tweedie_variance_power"] == 1.4
    reg2 = clone(reg)
    assert reg2.get_params()["tweedie_variance_power"] == 1.4
    reg2.fit(X, y)
    assert np.allclose(reg2.predict(X), p, rtol=1e-6)
    hub = RayXGBRegressor(n_estimators=3, objective="reg:pseudohubererror", huber_slope=2.0, n_jobs=num_actors)
    assert clone(hub).get_params()["huber_slope"] == 2.0
    yh = labels("reg:pseudohubererror", X, rng)
    hub.fit(X, yh)
    ohub = R.train(oracle, {"objective": "reg:pseudohubererror", "huber_slope": 2.0, "max_depth": 6, "eta": 0.3,
                            "max_bin": 256}, X, yh, 3)
    assert_same_model(hub.get_booster(), ohub)
    for obj in NEW_OBJECTIVES:
        r = RayXGBRegressor(n_estimators=2, max_depth=3, objective=obj, n_jobs=num_actors).fit(X, labels(obj, X, rng))
        assert np.all(np.isfinite(r.predict(X)))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("obj", ["count:poisson", "reg:tweedie"])
def test_two_gpu_models_byte_identical(eng, obj):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    rng = np.random.RandomState(8)
    X = make_data(30001, 10, 13, "uniform", nan_frac=0.05)
    y = labels(obj, X, rng)
    params = dict(OBJ_PARAMS.get(obj, {}), objective=obj, max_depth=6)
    b1 = train(params, RayDMatrix(X, y), num_boost_round=5, ray_params=RayParams(num_actors=1))
    b2 = train(params, RayDMatrix(X, y), num_boost_round=5, ray_params=RayParams(num_actors=2))
    assert bytes(b1.save_raw()) == bytes(b2.save_raw())
