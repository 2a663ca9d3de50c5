"""Booster slicing and callback.EarlyStopping(save_best=True) on the GPU (DESIGN.md 2 item 23).

A slice runs the existing prediction, TreeSHAP and leaf-index kernels on a booster built from the kept trees, so its
outputs must equal the full model's outputs over the same rounds (iteration_range) bit for bit, and a slice with step
> 1 must equal the model file edited to keep the same rounds.  Continuing from a slice, training the source on after
slicing, and save / load / pickle keep the models exact.  EarlyStopping with save_best=True returns the first
best_iteration + 1 rounds through engine.train, Ray train and the sklearn estimator."""
import pickle

import numpy as np
import pytest

from tests.model_files import keep_rounds

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def E():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


BASE = {"max_depth": 4, "eta": 0.3, "seed": 7}
CASES = {
    "gbtree": ({"objective": "reg:squarederror"}, 1),
    "dart": ({"objective": "binary:logistic", "booster": "dart", "rate_drop": 0.3}, 1),
    "softprob_k3": ({"objective": "multi:softprob", "num_class": 3}, 1),
    "parallel_3": ({"objective": "reg:squarederror", "num_parallel_tree": 3, "subsample": 0.7,
                    "colsample_bynode": 0.8}, 1),
    "targets_3": ({"objective": "reg:squarederror"}, 3),
    "vector_leaf_4": ({"objective": "reg:squarederror", "multi_strategy": "multi_output_tree"}, 4),
    "quantile_2": ({"objective": "reg:quantileerror", "quantile_alpha": [0.25, 0.75]}, 1),
    "categorical_nan": ({"objective": "reg:squarederror", "max_cat_to_onehot": 1}, 1),
}
ROUNDS = 12


def _data(case, n=3000, f=8, seed=0):
    rng = np.random.RandomState(seed)
    X = rng.uniform(0, 10, size=(n, f)).astype(np.float32)
    X[rng.uniform(size=X.shape) < 0.05] = np.nan
    kw = {}
    if case == "categorical_nan":
        X[:, 0] = rng.randint(0, 12, size=n)
        X[rng.uniform(size=n) < 0.1, 0] = np.nan
        kw = {"feature_types": ["c"] + ["q"] * (f - 1), "enable_categorical": True}
    s = np.nan_to_num(X[:, 0]) + 0.5 * np.nan_to_num(X[:, 1]) + rng.normal(size=n)
    params, targets = CASES[case]
    obj = params["objective"]
    if obj == "multi:softprob":
        y = np.digitize(s, np.quantile(s, [1 / 3, 2 / 3])).astype(np.float32)
    elif obj == "binary:logistic":
        y = (s > np.median(s)).astype(np.float32)
    elif targets > 1:
        y = np.stack([s + k * np.nan_to_num(X[:, 2 + k]) for k in range(targets)], axis=1).astype(np.float32)
        kw["multi_target"] = True
    else:
        y = s.astype(np.float32)
    return X, y, kw


_MODELS = {}


def _model(E, case):
    """(booster trained ROUNDS rounds, prediction matrix) of a case, trained once per module."""
    if case not in _MODELS:
        X, y, kw = _data(case)
        bst = E.train(dict(BASE, **CASES[case][0]), E.DMatrix(X, label=y, **kw), ROUNDS)
        Xp, _, _ = _data(case, n=700, seed=1)
        kw.pop("multi_target", None)
        _MODELS[case] = (bst, E.DMatrix(Xp, **kw))
    return _MODELS[case]


def _outputs(E, bst, dm, rounds=None):
    """Every prediction mode of bst over `rounds` (None: all); a mode the model refuses gives its error type."""
    kw = {} if rounds is None else {"iteration_range": rounds}
    out = {"margin": bst.predict(dm, output_margin=True, **kw), "transformed": bst.predict(dm, **kw),
           "leaf": bst.predict(dm, pred_leaf=True, **kw)}
    for mode in ("pred_contribs", "pred_interactions"):
        try:
            out[mode] = bst.predict(dm, **{mode: True}, **kw)
        except E.XGBoostError as e:
            out[mode] = type(e)
    return out


def _assert_same(got, want, what):
    assert set(got) == set(want)
    for k, w in want.items():
        g = got[k]
        if isinstance(w, np.ndarray):
            assert g.shape == w.shape and g.dtype == w.dtype and g.tobytes() == w.tobytes(), (what, k)
        else:
            assert g is w, (what, k)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", list(CASES))
def test_slice_equals_iteration_range(E, case):
    bst, dm = _model(E, case)
    assert bst.num_boosted_rounds() == ROUNDS
    for a, b in [(0, ROUNDS), (0, 5), (3, 9), (11, 12), (7, 8)]:
        s = bst[a:b]
        assert s.num_boosted_rounds() == b - a and s.handle == 0
        _assert_same(_outputs(E, s, dm), _outputs(E, bst, dm, (a, b)), (case, a, b))
    if case in ("gbtree", "dart", "softprob_k3", "quantile_2"):   # SHAP is compared, not only its refusal
        assert isinstance(_outputs(E, bst[0:3], dm)["pred_interactions"], np.ndarray)


@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", list(CASES))
def test_step_slice_equals_edited_model_file(E, case):
    bst, dm = _model(E, case)
    for sl, rounds in ((slice(1, ROUNDS, 3), [1, 4, 7, 10]), (slice(None, None, 5), [0, 5, 10]),
                       (slice(2, 9, 2), [2, 4, 6, 8])):
        s = bst[sl]
        ref = E.Booster(model_file=keep_rounds(bst.save_raw(), rounds))
        assert s.get_tree_weights().tobytes() == ref.get_tree_weights().tobytes()
        assert s.get_dump(with_stats=True) == ref.get_dump(with_stats=True)
        _assert_same(_outputs(E, s, dm), _outputs(E, ref, dm), (case, sl))


def _cont_data(n=6000, f=10, seed=3):
    rng = np.random.RandomState(seed)
    X = rng.uniform(0, 10, size=(n, f)).astype(np.float32)
    X[rng.uniform(size=X.shape) < 0.03] = np.nan
    y = (np.nan_to_num(X[:, 0]) * np.nan_to_num(X[:, 1]) / 10 + rng.normal(size=n) > 2.5).astype(np.float32)
    return X, y


@pytest.mark.timeout(900)
@pytest.mark.parametrize("booster", ["gbtree", "dart"])
def test_continuation_from_a_slice(E, booster):
    X, y = _cont_data()
    p = {"objective": "binary:logistic", "max_depth": 5, "eta": 0.3, "subsample": 0.8, "colsample_bynode": 0.7,
         "seed": 11}
    if booster == "dart":
        p.update(booster="dart", rate_drop=0.25)
    long = E.train(p, E.DMatrix(X, label=y), 20)
    s = long[:10]
    cont = E.train(p, E.DMatrix(X, label=y), 5, xgb_model=s)
    assert cont.num_boosted_rounds() == 15
    if booster == "gbtree":
        assert bytes(cont.save_raw()) == bytes(E.train(p, E.DMatrix(X, label=y), 15).save_raw())
    else:
        # rounds 10-19 renormalised the weights of the trees they dropped, and a slice keeps the weights it has: the
        # continuation equals continuing the model file cut to the same 10 rounds, weights included
        assert s.get_tree_weights().tobytes() == long.get_tree_weights()[:10].tobytes()
        ref = E.train(p, E.DMatrix(X, label=y), 5,
                      xgb_model=E.Booster(model_file=keep_rounds(long.save_raw(), range(10))))
        assert bytes(cont.save_raw()) == bytes(ref.save_raw())
    assert long.num_boosted_rounds() == 20


@pytest.mark.timeout(900)
@pytest.mark.parametrize("booster", ["gbtree", "dart"])
def test_source_trains_on_after_slicing(E, booster):
    X, y = _cont_data()
    p = {"objective": "binary:logistic", "max_depth": 5, "eta": 0.3, "subsample": 0.8, "seed": 2}
    if booster == "dart":
        p.update(booster="dart", rate_drop=0.25)
    dp = E.DMatrix(_cont_data(n=500, seed=9)[0])
    d1 = E.DMatrix(X, label=y)
    bst = E.train(p, d1, 10)
    s = bst[2:7]
    before = s.predict(dp, output_margin=True)
    assert before.tobytes() == bst.predict(dp, output_margin=True, iteration_range=(2, 7)).tobytes()
    for r in range(10, 15):
        bst.update(d1, r)
    d2 = E.DMatrix(X, label=y)
    ref = E.train(p, d2, 10)
    for r in range(10, 15):
        ref.update(d2, r)
    assert bytes(bst.save_raw()) == bytes(ref.save_raw())
    assert s.predict(dp, output_margin=True).tobytes() == before.tobytes()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", ["dart", "softprob_k3", "vector_leaf_4", "categorical_nan", "quantile_2"])
def test_slice_round_trips(E, case, tmp_path):
    bst, dm = _model(E, case)
    s = bst[3:11:2]
    want = _outputs(E, s, dm)
    f = str(tmp_path / "slice.json")
    s.save_model(f)
    for b in (E.Booster(model_file=f), pickle.loads(pickle.dumps(s)), s.copy()):
        # trees and weights, not file bytes: a trained model keeps quantile_alpha as a list, a loaded one as its string
        assert b.get_dump(dump_format="json", with_stats=True) == s.get_dump(dump_format="json", with_stats=True)
        assert b.get_tree_weights().tobytes() == s.get_tree_weights().tobytes()
        _assert_same(_outputs(E, b, dm), want, case)


# ----------------------------------------------------------------------------- EarlyStopping(save_best=True)
ES_PARAMS = {"max_depth": 6, "eta": 0.5, "base_score": 0.5}
ES_ROUNDS = 300


def _es_data():
    rng = np.random.RandomState(21)
    X = rng.uniform(0, 10, size=(5000, 8)).astype(np.float32)
    y = (X[:, 0] + 3 * rng.normal(size=5000)).astype(np.float32)    # noisy: the valid error turns up early
    return X[:4000], y[:4000], X[4000:], y[4000:]


def _dump(bst):
    return bst.get_dump(dump_format="json", with_stats=True)


@pytest.fixture(scope="module")
def es_engine(E):
    """(full run stopped by EarlyStopping(4), save_best run), both through engine.train."""
    X, y, Xv, yv = _es_data()
    runs = []
    for save_best in (False, True):
        dtrain = E.DMatrix(X, label=y)
        runs.append(E.train(ES_PARAMS, dtrain, ES_ROUNDS, evals=[(dtrain, "train"), (E.DMatrix(Xv, label=yv), "valid")],
                            callbacks=[E.callback.EarlyStopping(4, save_best=save_best)], verbose_eval=False))
    return runs


def _assert_best_rounds(E, best, full):
    b = full.best_iteration
    assert b is not None and full.num_boosted_rounds() == b + 5 < ES_ROUNDS      # it stopped after 4 stale rounds
    assert best.num_boosted_rounds() == b + 1
    assert (best.best_iteration, best.best_score) == (b, full.best_score)
    X, _, Xv, _ = _es_data()
    dm = E.DMatrix(np.concatenate([Xv, X[:500]]))
    for om in (True, False):
        assert best.predict(dm, output_margin=om).tobytes() == \
            full.predict(dm, output_margin=om, iteration_range=(0, b + 1)).tobytes()
    assert _dump(best) == _dump(full)[:b + 1]


@pytest.mark.timeout(900)
def test_early_stopping_save_best_engine(E, es_engine):
    full, best = es_engine
    _assert_best_rounds(E, best, full)
    p = pickle.loads(pickle.dumps(best))
    assert (p.best_iteration, p.best_score) == (best.best_iteration, best.best_score)


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("actors", [1, 2])
def test_early_stopping_save_best_ray(E, es_engine, actors):
    if E.device_count() < actors:
        pytest.skip("needs %d GPUs: each actor of the %d-actor run trains on its own GPU" % (actors, actors))
    from xgboost_ray_b200 import RayDMatrix, RayParams, predict, train
    X, y, Xv, yv = _es_data()
    runs = []
    for save_best in (False, True):
        runs.append(train(ES_PARAMS, RayDMatrix(X, y), ES_ROUNDS, evals=[(RayDMatrix(X, y), "train"),
                                                                          (RayDMatrix(Xv, yv), "valid")],
                          callbacks=[E.callback.EarlyStopping(4, save_best=save_best)], verbose_eval=False,
                          ray_params=RayParams(num_actors=actors)))
    full, best = runs
    _assert_best_rounds(E, best, full)
    pred = predict(best, RayDMatrix(Xv), ray_params=RayParams(num_actors=actors))
    assert pred.tobytes() == full.predict(E.DMatrix(Xv), iteration_range=(0, full.best_iteration + 1)).tobytes()
    if actors == 1:     # one actor trains the engine's model
        _, eng_best = es_engine
        assert _dump(best) == _dump(eng_best) and best.best_iteration == eng_best.best_iteration


@pytest.mark.timeout(900)
def test_early_stopping_save_best_sklearn(E, es_engine):
    from xgboost_ray_b200 import RayParams
    from xgboost_ray_b200.sklearn import RayXGBRegressor
    X, y, Xv, yv = _es_data()
    reg = RayXGBRegressor(n_estimators=ES_ROUNDS, max_depth=6, learning_rate=0.5, base_score=0.5,
                          callbacks=[E.callback.EarlyStopping(4, save_best=True)])
    reg.fit(X, y, eval_set=[(X, y), (Xv, yv)], ray_params=RayParams(num_actors=1))
    full, best = es_engine
    b = full.best_iteration
    assert reg.best_iteration == b and reg.get_booster().num_boosted_rounds() == b + 1
    assert _dump(reg.get_booster()) == _dump(best)
    assert reg.predict(Xv, ray_params=RayParams(num_actors=1)).tobytes() == \
        full.predict(E.DMatrix(Xv), iteration_range=(0, b + 1)).tobytes()
