"""Booster.set_param between boosting rounds on the GPU (DESIGN.md 2 item 22): schedules of eta and the regularisation
against the oracle's restatement of the same schedule (split features, bins, default directions and topology exact,
leaves within 1e-5), a schedule against a continuation with xgb_model, refusals of the keys that are fixed once training
started, the public callbacks= path and pickling in the middle of a schedule."""
import pickle

import numpy as np
import pytest

from tests import schedule_reference as S

pytestmark = pytest.mark.gpu

LEAF_TOL = 1e-5


@pytest.fixture(scope="module")
def E():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def _data(objective, n=6000, f=12, seed=1, targets=1):
    rng = np.random.RandomState(seed)
    X = rng.uniform(0, 10, size=(n, f)).astype(np.float32)
    X[rng.uniform(size=X.shape) < 0.03] = np.nan
    s = np.nan_to_num(X[:, 0]) + 0.5 * np.nan_to_num(X[:, 1]) + rng.normal(size=n)
    if objective.startswith("multi"):
        y = np.digitize(s, np.quantile(s, [1 / 3, 2 / 3])).astype(np.float32)
    elif targets > 1:
        y = np.stack([s + k * np.nan_to_num(X[:, 2 + k]) for k in range(targets)], axis=1).astype(np.float32)
    else:
        y = s.astype(np.float32)
    return X, y


def _dump(bst):
    return bst.get_dump(dump_format="json", with_stats=True)


def _train_schedule(E, params, dm, rounds, schedule):
    bst = E.Booster(params)
    for r in range(rounds):
        if r in schedule:
            bst.set_param(schedule[r])
        bst.update(dm, r)
    return bst


# eta, lambda, alpha, gamma, min_child_weight and max_delta_step, each changed at its own round
SCHEDULE = {2: {"eta": 0.1}, 3: {"lambda": 4.0}, 5: {"alpha": 0.7, "eta": 0.45}, 7: {"gamma": 0.8},
            8: {"min_child_weight": 6.0}, 10: {"max_delta_step": 0.05, "eta": 0.2}}
# the same with row and column sampling switched on and off again (graph replay <-> direct launches)
SAMPLING = dict(SCHEDULE)
SAMPLING.update({4: {"subsample": 0.8, "colsample_bynode": 0.8}, 6: {"eta": 0.25},
                 9: {"subsample": 1.0, "colsample_bynode": 1.0}})


@pytest.mark.timeout(600)
@pytest.mark.parametrize("schedule", [SCHEDULE, SAMPLING], ids=["regularisation", "sampling"])
@pytest.mark.parametrize("objective", ["reg:squarederror", "multi:softprob"])
def test_schedule_matches_oracle(E, oracle, objective, schedule):
    X, y = _data(objective)
    params = {"objective": objective, "max_depth": 5, "eta": 0.3, "base_score": 0.5, "seed": 3}
    if objective == "multi:softprob":
        params["num_class"] = 3
    K = params.get("num_class", 1)
    dm = E.DMatrix(X, label=y)
    bst = _train_schedule(E, params, dm, 12, schedule)
    ob = S.train(params, X, y, 12, schedule)
    trees = bst.get_trees()
    assert len(trees) == ob.num_trees == 12 * K
    eta = params["eta"]
    for i, t in enumerate(trees):
        r = i // K
        eta = schedule.get(r, {}).get("eta", eta)
        o = ob.tree(i)
        for k in ("left", "right", "split_feature", "split_bin", "default_left"):
            assert np.array_equal(t[k], getattr(o, k)), (objective, i, k)
        leaf = o.split_feature < 0
        assert np.max(np.abs(t["value"][leaf] - o.value[leaf])) <= LEAF_TOL, (objective, i)
        # every leaf of round r is eta_r x its weight: a tree replayed from a stale graph would carry the old eta
        assert np.allclose(t["value"][leaf], t["base_weight"][leaf] * np.float32(eta), rtol=1e-6, atol=0), (i, eta)
    timers = bst.get_timers()
    assert timers["graph_updates"] + timers["graph_reinstantiations"] > 0, timers


@pytest.mark.timeout(600)
def test_same_value_does_not_recapture(E):
    X, y = _data("reg:squarederror")
    dm = E.DMatrix(X, label=y)
    params = {"max_depth": 5, "eta": 0.3, "base_score": 0.5}
    ref = _train_schedule(E, params, dm, 8, {})
    bst = _train_schedule(E, params, dm, 8, {r: {"eta": 0.3, "lambda": 1.0, "max_depth": 5} for r in range(1, 8)})
    assert _dump(bst) == _dump(ref)
    t = bst.get_timers()
    assert t["graph_updates"] == 0 and t["graph_reinstantiations"] == 0 and t["graph_update_ms"] == 0, t


def _continuation_cases():
    return [
        ("scalar", {"objective": "reg:squarederror"}, 1),
        ("targets", {"objective": "reg:squarederror"}, 3),
        ("vector_leaf", {"objective": "reg:squarederror", "multi_strategy": "multi_output_tree"}, 3),
        ("quantile", {"objective": "reg:quantileerror", "quantile_alpha": [0.2, 0.8]}, 1),
    ]


@pytest.mark.timeout(600)
@pytest.mark.parametrize("case,extra,targets", _continuation_cases(), ids=[c[0] for c in _continuation_cases()])
def test_schedule_equals_continuation(E, case, extra, targets):
    X, y = _data("reg", targets=targets)
    params = dict({"max_depth": 4, "eta": 0.4}, **extra)
    a, b = 0.4, 0.15
    mt = {"multi_target": True} if targets > 1 else {}
    sched = E.train(params, E.DMatrix(X, label=y, **mt), 10,
                    callbacks=[E.callback.LearningRateScheduler([a] * 4 + [b] * 6)])
    first = E.train(params, E.DMatrix(X, label=y, **mt), 5)
    cont = E.train(dict(params, eta=b), E.DMatrix(X, label=y, **mt), 5, xgb_model=first)
    assert _dump(sched) == _dump(cont)
    assert sched.save_config() and float(sched.params["learning_rate"]) == b


@pytest.mark.timeout(600)
def test_fixed_keys_are_refused_atomically(E):
    X, y = _data("reg:squarederror")
    params = {"max_depth": 5, "eta": 0.3, "base_score": 0.5, "seed": 0}
    dm = E.DMatrix(X, label=y)
    ref = _train_schedule(E, params, dm, 3, {})
    bst = E.Booster(params)
    bst.update(dm, 0)
    before = dict(bst.params)
    for key, value in [("max_depth", 4), ("objective", "reg:pseudohubererror"), ("num_parallel_tree", 2),
                       ("quantile_alpha", 0.3), ("hist_qbits", 12), ("seed", 7), ("booster", "dart"),
                       ("random_state", 9)]:
        with pytest.raises(E.XGBoostError, match="parameter %s cannot change" % key):
            bst.set_param({"eta": 0.01, key: value})      # the eta of a refused call is not applied either
        assert bst.params == before
    with pytest.raises(E.XGBoostError, match=r"subsample / colsample_\* must be in \(0, 1\], got 0"):
        bst.set_param("subsample", 0)
    with pytest.raises(E.XGBoostError, match="max_cat_to_onehot must be >= 1"):
        bst.set_param({"eta": 0.01, "max_cat_to_onehot": 0})
    assert bst.params == before
    bst.set_param({"max_depth": 5, "seed": 0, "objective": "reg:squarederror", "eta": 0.3, "nthread": 4})  # same values
    bst.update(dm, 1)
    bst.update(dm, 2)
    assert _dump(bst) == _dump(ref)
    # before the first round every key is accepted, with and without a device booster attached
    ref3 = _train_schedule(E, dict(params, max_depth=3, hist_qbits=14), dm, 2, {})
    for b0 in (E.Booster(params), E.Booster(params, cache=[dm])):
        b0.set_param({"max_depth": 3, "hist_qbits": 14})
        b0.update(dm, 0)
        b0.update(dm, 1)
        assert _dump(b0) == _dump(ref3)


RATES = [0.3, 0.3, 0.1, 0.1, 0.5, 0.05]


@pytest.mark.timeout(900)
def test_public_callbacks_path(E):
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    from xgboost_ray_b200.sklearn import RayXGBRegressor
    X, y = _data("reg:squarederror", n=8000)
    params = {"max_depth": 4, "learning_rate": 0.3, "base_score": 0.5}
    ref = E.train(params, E.DMatrix(X, label=y), 6, callbacks=[E.callback.LearningRateScheduler(RATES)])
    sched = {r + 1: {"eta": RATES[r]} for r in range(5)}
    assert _dump(ref) == _dump(_train_schedule(E, {"max_depth": 4, "eta": 0.3, "base_score": 0.5}, E.DMatrix(X, label=y),
                                               6, sched))
    bst = train(params, RayDMatrix(X, y), num_boost_round=6, ray_params=RayParams(num_actors=1),
                callbacks=[E.callback.LearningRateScheduler(RATES)])
    assert _dump(bst) == _dump(ref)
    import json
    assert float(json.loads(bst.save_config())["learner"]["b2_params"]["learning_rate"]) == RATES[-1]
    reg = RayXGBRegressor(n_estimators=6, max_depth=4, learning_rate=0.3, base_score=0.5,
                          callbacks=[E.callback.LearningRateScheduler(RATES)])
    reg.fit(X, y, ray_params=RayParams(num_actors=1))
    assert _dump(reg.get_booster()) == _dump(ref)
    if E.device_count() >= 2:
        bst2 = train(params, RayDMatrix(X, y), num_boost_round=6, ray_params=RayParams(num_actors=2),
                     callbacks=[E.callback.LearningRateScheduler(RATES)])
        assert _dump(bst2) == _dump(ref)


@pytest.mark.timeout(600)
def test_pickle_in_the_middle_of_a_schedule(E):
    X, y = _data("multi:softprob")
    params = {"objective": "multi:softprob", "num_class": 3, "max_depth": 4, "eta": 0.3}
    sched = {2: {"eta": 0.1, "lambda": 2.0}, 5: {"eta": 0.5}, 7: {"gamma": 0.3, "eta": 0.2}}
    dm = E.DMatrix(X, label=y)
    whole = _train_schedule(E, params, dm, 10, sched)
    bst = _train_schedule(E, params, E.DMatrix(X, label=y), 5, sched)
    bst = pickle.loads(pickle.dumps(bst))
    dm2 = E.DMatrix(X, label=y)
    for r in range(5, 10):
        if r in sched:
            bst.set_param(sched[r])
        bst.update(dm2, r)
    assert _dump(bst) == _dump(whole)
