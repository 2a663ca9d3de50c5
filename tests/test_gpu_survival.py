"""GPU checks of survival:aft: gradients bit-equal to tests/survival_reference.py (read back with
B2_BoosterGetGradients), trees identical to the oracle grown from them, both metrics, the default metric, input errors,
save / load / continuation, the golden fixtures, SHAP and the public train / predict on one and two GPUs."""
import copy
import json
import os

import jsonschema
import numpy as np
import pytest

from tests import survival_reference as S
from tests.golden.make_golden_survival import CASES as SURVIVAL_CASES, case_data
from tests.model_schema import MODEL
from tests.test_gpu_parity import assert_same_model, make_data

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def bounds(X, rng):
    """Times that depend on the first features, censored by row index: exact, right, left, interval."""
    x = np.nan_to_num(X.astype(np.float64))
    t = np.exp(0.2 * x[:, 0] - 0.15 * x[:, 1] + 0.3 * rng.normal(size=len(x))).astype(np.float32)
    lo, hi = t.copy(), t.copy()
    k = np.arange(len(t)) % 4
    hi[k == 1] = np.inf
    lo[k == 2] = 0.0
    hi[k == 3] = t[k == 3] * np.float32(1.8)
    return lo, hi


def get_gradients(eng, bst, n):
    import ctypes as C
    g = np.zeros(n, np.float32)
    h = np.zeros(n, np.float32)
    eng._check(eng.lib().B2_BoosterGetGradients(bst.handle, g.ctypes.data_as(C.POINTER(C.c_float)),
                                                  h.ctypes.data_as(C.POINTER(C.c_float)), n))
    return g, h


@pytest.mark.parametrize("dist", S.DISTRIBUTIONS)
@pytest.mark.parametrize("sigma", [0.3, 1.0, 2.5])
def test_gradients_bit_equal_to_reference(eng, dist, sigma):
    """Margins across +-60 (pdf underflow, cancelled CDF differences and the limit branches) for every censoring kind,
    with weights: the engine's gradient pairs equal the reference bit for bit."""
    rng = np.random.RandomState(1)
    n = 40000
    X = make_data(n, 3, 2, "uniform")
    lo, hi = bounds(X, rng)
    lo[::97] = 0.0            # a few rows left-censored at [0, +inf): F_u - F_l = 1
    hi[::97] = np.inf
    m = rng.uniform(-60, 60, n).astype(np.float32)
    m[::5] = (np.log(np.maximum(lo[::5], 1e-3)) + rng.normal(size=len(m[::5]))).astype(np.float32)
    w = rng.uniform(0.1, 3.0, n).astype(np.float32)
    params = {"objective": "survival:aft", "aft_loss_distribution": dist, "aft_loss_distribution_scale": sigma,
              "max_depth": 2}
    dm = eng.DMatrix(X, weight=w, base_margin=m, label_lower_bound=lo, label_upper_bound=hi)
    bst = eng.Booster(params, cache=[dm])
    bst.update(dm, 0)
    g, h = get_gradients(eng, bst, n)
    rg, rh, bad = S.gradients(params, m, lo, hi, w)
    assert bad == 0
    assert np.array_equal(g.view(np.uint32), rg.view(np.uint32)), np.nonzero(g != rg)[0][:10]
    assert np.array_equal(h.view(np.uint32), rh.view(np.uint32)), np.nonzero(h != rh)[0][:10]


@pytest.mark.parametrize("dist", S.DISTRIBUTIONS)
@pytest.mark.parametrize("depth", [4, 8])
def test_trees_identical_to_oracle(eng, oracle, dist, depth):
    rng = np.random.RandomState(3 + depth)
    n, f = 8000, 8
    X = make_data(n, f, 31, "uniform", nan_frac=0.1)
    lo, hi = bounds(X, rng)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32)
    params = {"objective": "survival:aft", "aft_loss_distribution": dist, "aft_loss_distribution_scale": 0.8,
              "max_depth": depth, "eta": 0.3}
    obst = S.train(oracle, params, X, lo, hi, 4, weight=w)
    dm = eng.DMatrix(X, weight=w, label_lower_bound=lo, label_upper_bound=hi)
    ebst = eng.train(params, dm, num_boost_round=4, verbose_eval=False)
    assert_same_model(ebst, obst)
    Xt = make_data(2000, f, 99, "uniform")
    pe, po = ebst.predict(eng.DMatrix(Xt)), obst.predict(Xt)
    assert np.max(np.abs(pe - po) / np.maximum(1.0, np.abs(po))) <= 1e-5


@pytest.mark.parametrize("dist", S.DISTRIBUTIONS)
def test_trees_identical_to_oracle_categorical_colsample(eng, oracle, dist):
    rng = np.random.RandomState(9)
    n, f = 8000, 8
    X = make_data(n, f, 32, "uniform", nan_frac=0.05)
    X[:, 3] = rng.randint(0, 3, n)
    X[:, 4] = rng.randint(0, 20, n)
    is_cat = [0, 0, 0, 1, 1, 0, 0, 0]
    lo, hi = bounds(X, rng)
    scale = np.where(X[:, 4] % 3 == 0, 2.0, 1.0).astype(np.float32)
    lo, hi = lo * scale, hi * scale
    w = rng.uniform(0.5, 2.0, n).astype(np.float32)
    params = {"objective": "survival:aft", "aft_loss_distribution": dist, "max_depth": 5, "eta": 0.3,
              "colsample_bynode": 0.6, "seed": 4}
    obst = S.train(oracle, params, X, lo, hi, 4, weight=w, is_cat=is_cat)
    dm = eng.DMatrix(X, weight=w, label_lower_bound=lo, label_upper_bound=hi,
                     feature_types=["q" if c == 0 else "c" for c in is_cat], enable_categorical=True)
    ebst = eng.train(params, dm, num_boost_round=4, verbose_eval=False)
    assert_same_model(ebst, obst)


@pytest.mark.parametrize("dist", S.DISTRIBUTIONS)
def test_metrics_per_round(eng, dist):
    rng = np.random.RandomState(4)
    n = 6000
    X = make_data(n, 6, 5, "uniform")
    lo, hi = bounds(X, rng)
    w = rng.uniform(0.5, 2.0, n).astype(np.float32)
    params = {"objective": "survival:aft", "aft_loss_distribution": dist, "aft_loss_distribution_scale": 1.3,
              "max_depth": 4, "eval_metric": ["aft-nloglik", "interval-regression-accuracy"]}
    dm = eng.DMatrix(X, weight=w, label_lower_bound=lo, label_upper_bound=hi)
    Xv = make_data(3000, 6, 6, "uniform")
    lov, hiv = bounds(Xv, rng)
    dv = eng.DMatrix(Xv, label_lower_bound=lov, label_upper_bound=hiv)
    bst = eng.Booster(params, cache=[dm])
    for r in range(4):
        bst.update(dm, r)
        res = dict((f"{d}-{k}", v) for d, k, v in eng._parse_eval_str(bst.eval_set([(dm, "train"), (dv, "valid")], r)))
        mt = bst.predict(dm, output_margin=True, training=True)
        mv = bst.predict(dv, output_margin=True)
        for name in ("aft-nloglik", "interval-regression-accuracy"):
            for key, (m, a, b, ww) in (("train", (mt, lo, hi, w)), ("valid", (mv, lov, hiv, None))):
                want = S.metric(name, params, m, a, b, ww)
                got = res[f"{key}-{name}"]
                assert abs(got - want) <= max(1e-9 * abs(want), 5e-7), (r, key, name, got, want)   # printed with %.6f
        v = eng.lib().B2_BoosterEvalSet
        import ctypes as C
        out = C.c_double(0)
        eng._check(v(bst.handle, dv.handle, b"aft-nloglik", C.byref(out)))
        want = S.metric("aft-nloglik", params, mv, lov, hiv)
        assert abs(out.value - want) <= 1e-9 * abs(want)


def test_default_metric_and_base_score(eng):
    rng = np.random.RandomState(5)
    X = make_data(3000, 5, 4, "uniform")
    lo, hi = bounds(X, rng)
    dm = eng.DMatrix(X, label=lo, label_lower_bound=lo, label_upper_bound=hi)
    res = {}
    bst = eng.train({"objective": "survival:aft"}, dm, 2, evals=[(dm, "t")], evals_result=res, verbose_eval=False)
    assert list(res["t"]) == ["aft-nloglik"]
    assert bst.params["base_score"] == 0.5
    # early stopping maximises the accuracy
    res = {}
    bst = eng.train({"objective": "survival:aft", "eval_metric": "interval-regression-accuracy"}, dm, 6,
                    evals=[(dm, "t")], evals_result=res, early_stopping_rounds=2, verbose_eval=False)
    acc = res["t"]["interval-regression-accuracy"]
    assert bst.best_score == max(acc[:bst.best_iteration + 1])


def test_input_errors(eng):
    rng = np.random.RandomState(6)
    X = make_data(800, 3, 1, "uniform")
    lo, hi = bounds(X, rng)
    E = eng.XGBoostError
    p = {"objective": "survival:aft"}
    with pytest.raises(E, match="survival:aft needs label_lower_bound and label_upper_bound"):
        eng.train(p, eng.DMatrix(X, label=lo), 1, verbose_eval=False)
    with pytest.raises(E, match="survival:aft needs label_lower_bound and label_upper_bound"):
        eng.train(p, eng.DMatrix(X, label=lo, label_lower_bound=lo), 1, verbose_eval=False)
    for bad_lo, bad_hi, msg in ((np.where(np.arange(800) == 7, np.nan, lo), hi, "NaN"),
                                (np.where(np.arange(800) == 7, -1.0, lo), hi, "label_lower_bound must be finite and >= 0"),
                                (lo, np.where(np.arange(800) == 4, lo / 2, hi), "label_upper_bound must be >= label_lower_bound"),
                                (np.where(np.arange(800) == 8, 0.0, lo), np.where(np.arange(800) == 8, 0.0, hi),
                                 r"uncensored row \(lower == upper\) needs a label > 0")):
        dm = eng.DMatrix(X, label_lower_bound=bad_lo.astype(np.float32), label_upper_bound=bad_hi.astype(np.float32))
        with pytest.raises(E, match=msg):
            eng.train(p, dm, 1, verbose_eval=False)
    dm = eng.DMatrix(X, label=lo, label_lower_bound=lo, label_upper_bound=hi)
    with pytest.raises(E, match="length"):
        dm.set_info(label_lower_bound=lo[:10])
    with pytest.raises(E, match="aft_loss_distribution"):
        eng.train(dict(p, aft_loss_distribution="weibull"), dm, 1, verbose_eval=False)
    for s in (0.0, -1.0):
        with pytest.raises(E, match="aft_loss_distribution_scale"):
            eng.train(dict(p, aft_loss_distribution_scale=s), dm, 1, verbose_eval=False)
    with pytest.raises(E, match="base_score"):
        eng.train(dict(p, base_score=0.0), dm, 1, verbose_eval=False)
    for metric in ("aft-nloglik", "interval-regression-accuracy"):
        with pytest.raises(E, match="does not fit"):
            eng.train({"objective": "reg:squarederror", "eval_metric": metric}, dm, 1, evals=[(dm, "t")], verbose_eval=False)
    bst = eng.train(p, dm, 1, verbose_eval=False)
    with pytest.raises(E, match="needs label_lower_bound"):
        bst.eval_set([(eng.DMatrix(X, label=lo), "v")])
    with pytest.raises(E, match="unsupported objective"):
        eng.train({"objective": "survival:cox"}, dm, 1, verbose_eval=False)
    # other objectives store and ignore the bounds
    plain = eng.train({"objective": "reg:squarederror", "max_depth": 3}, eng.DMatrix(X, label=lo), 2, verbose_eval=False)
    with_b = eng.train({"objective": "reg:squarederror", "max_depth": 3}, dm, 2, verbose_eval=False)
    assert bytes(plain.save_raw()) == bytes(with_b.save_raw())


def aft_schema():
    schema = copy.deepcopy(MODEL)
    schema["properties"]["learner"]["properties"]["objective"]["oneOf"].append(
        {"type": "object", "properties": {
            "name": {"const": "survival:aft"},
            "aft_loss_param": {"type": "object",
                               "properties": {"aft_loss_distribution": {"enum": ["normal", "logistic", "extreme"]},
                                              "aft_loss_distribution_scale": {"type": "string"}},
                               "required": ["aft_loss_distribution", "aft_loss_distribution_scale"],
                               "additionalProperties": False}},
         "required": ["name", "aft_loss_param"], "additionalProperties": False})
    return schema


@pytest.mark.parametrize("dist", S.DISTRIBUTIONS)
def test_save_load_and_continuation(eng, oracle, dist, tmp_path):
    rng = np.random.RandomState(7)
    X = make_data(5000, 6, 9, "uniform")
    lo, hi = bounds(X, rng)
    params = {"objective": "survival:aft", "aft_loss_distribution": dist, "aft_loss_distribution_scale": 0.7,
              "max_depth": 4}
    dm = eng.DMatrix(X, label=lo, label_lower_bound=lo, label_upper_bound=hi)
    bst = eng.train(params, dm, 2, verbose_eval=False)
    path = str(tmp_path / "m.json")
    bst.save_model(path)
    d = json.load(open(path))
    jsonschema.validate(d, aft_schema())
    assert d["learner"]["objective"] == {"name": "survival:aft", "aft_loss_param": {
        "aft_loss_distribution": dist, "aft_loss_distribution_scale": "0.7"}}
    Xt = eng.DMatrix(make_data(1000, 6, 60, "uniform"))
    for raw in (open(path, "rb").read(), None):
        if raw is None:      # a stock xgboost file: only the objective block carries the parameters
            del d["learner"]["attributes"]["b2.params"]
            raw = json.dumps(d).encode()
        loaded = eng.Booster(model_file=bytearray(raw))
        assert loaded.params["aft_loss_distribution"] == dist
        assert float(loaded.params["aft_loss_distribution_scale"]) == 0.7
        assert np.array_equal(bst.predict(Xt).view(np.uint32), loaded.predict(Xt).view(np.uint32))
        assert np.array_equal(bst.predict(Xt, output_margin=True).view(np.uint32),
                              loaded.predict(Xt, output_margin=True).view(np.uint32))
    cont = eng.train(params, eng.DMatrix(X, label=lo, label_lower_bound=lo, label_upper_bound=hi), 2, xgb_model=path,
                     verbose_eval=False)
    full = eng.train(params, dm, 4, verbose_eval=False)
    assert_same_model(cont, S.train(oracle, params, X, lo, hi, 4))
    assert [t["split_bin"].tolist() for t in cont.get_trees()] == [t["split_bin"].tolist() for t in full.get_trees()]
    pc, pf = cont.predict(Xt), full.predict(Xt)
    assert np.max(np.abs(pc - pf) / np.maximum(1.0, np.abs(pf))) <= 1e-5


@pytest.mark.parametrize("name", SURVIVAL_CASES)
def test_engine_reproduces_survival_golden(eng, name):
    want = json.load(open(os.path.join(os.path.dirname(__file__), "golden", name + ".json")))
    x, lo, hi, w, params, rounds = case_data(name)
    bst = eng.train(params, eng.DMatrix(x, weight=w, label_lower_bound=lo, label_upper_bound=hi),
                    num_boost_round=rounds, verbose_eval=False)
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


def test_pred_contribs_and_leaf(eng):
    rng = np.random.RandomState(8)
    X = make_data(3000, 6, 10, "uniform", nan_frac=0.05)
    lo, hi = bounds(X, rng)
    bst = eng.train({"objective": "survival:aft", "max_depth": 5},
                    eng.DMatrix(X, label_lower_bound=lo, label_upper_bound=hi), 5, verbose_eval=False)
    d = eng.DMatrix(X[:500])
    c = bst.predict(d, pred_contribs=True)
    m = bst.predict(d, output_margin=True)
    assert c.shape == (500, 7)
    assert np.all(np.abs(c.sum(axis=1) - m) <= 1e-5 * np.maximum(1.0, np.abs(m)))
    assert np.allclose(np.exp(m.astype(np.float64)), bst.predict(d), rtol=1e-5)
    assert bst.predict(d, pred_interactions=True).shape == (500, 7, 7)
    assert bst.predict(d, pred_leaf=True).shape == (500, 5)


@pytest.mark.parametrize("num_actors", [1, 2])
@pytest.mark.parametrize("source", ["numpy", "pandas"])
def test_public_train_predict(eng, oracle, num_actors, source):
    if num_actors > eng.device_count():
        pytest.skip("needs %d GPUs" % num_actors)
    import pandas as pd
    from xgboost_ray_b200 import RayDMatrix, RayParams, predict, train
    rng = np.random.RandomState(10)
    X = make_data(6001, 6, 12, "uniform")
    lo, hi = bounds(X, rng)
    params = {"objective": "survival:aft", "aft_loss_distribution": "logistic", "max_depth": 4, "eta": 0.3}
    if source == "numpy":
        dtrain = RayDMatrix(X, lo, label_lower_bound=lo, label_upper_bound=hi)
    else:
        df = pd.DataFrame(X, columns=["f%d" % i for i in range(6)])
        df["y"], df["lo"], df["hi"] = lo, lo, hi
        dtrain = RayDMatrix(df, label="y", label_lower_bound="lo", label_upper_bound="hi")
    res = {}
    bst = train(params, dtrain, num_boost_round=4, evals=[(dtrain, "train")], evals_result=res,
                ray_params=RayParams(num_actors=num_actors))
    assert list(res["train"]) == ["aft-nloglik"]
    ob = S.train(oracle, params, X, lo, hi, 4)
    assert_same_model(bst, ob)
    p = predict(bst, RayDMatrix(X), ray_params=RayParams(num_actors=num_actors))
    assert np.max(np.abs(p - ob.predict(X)) / np.maximum(1.0, ob.predict(X))) <= 1e-5


@pytest.mark.timeout(300)
def test_two_gpu_model_byte_identical(eng):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    rng = np.random.RandomState(11)
    X = make_data(30001, 10, 13, "uniform", nan_frac=0.05)
    lo, hi = bounds(X, rng)
    params = {"objective": "survival:aft", "aft_loss_distribution": "extreme", "max_depth": 6}
    b1 = train(params, RayDMatrix(X, lo, label_lower_bound=lo, label_upper_bound=hi), num_boost_round=5,
               ray_params=RayParams(num_actors=1))
    b2 = train(params, RayDMatrix(X, lo, label_lower_bound=lo, label_upper_bound=hi), num_boost_round=5,
               ray_params=RayParams(num_actors=2))
    assert bytes(b1.save_raw()) == bytes(b2.save_raw())
