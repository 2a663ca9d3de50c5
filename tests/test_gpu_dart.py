"""booster="dart" on the GPU.

Every model is compared with tests/dart_reference.py's DART on top of the oracle (the oracle grows each round's trees
from gradients at the reference's drop margin): the trees with assert_same_model, the weight vector bit for bit.  The
engine's margins (the full margin used by predict and the metrics, the drop margin a custom objective sees) must be the
reference's ordered weighted sums over the engine's own trees, walked on the bin matrix, bit for bit.  rate_drop = 0
and skip_drop = 1 must give the gbtree model byte for byte."""
import pickle

import numpy as np
import pytest

from tests import dart_reference as R
from tests import shap_reference as SR
from tests.test_gpu_parity import IS_CAT, assert_same_model, make_cat_data, make_data

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def labels(objective, y):
    if objective == "binary:logistic":
        return (y > np.median(y)).astype(np.float32)
    if objective == "multi:softprob":
        return np.digitize(y, np.quantile(y, [1 / 3, 2 / 3])).astype(np.float32)
    return y.astype(np.float32)


def dataset(n=6000, f=12, seed=0, nan_frac=0.0):
    X = make_data(n, f, seed, "uniform", nan_frac)
    Z = np.nan_to_num(X, nan=5.0)
    y = Z[:, 0] * 0.4 + np.sin(Z[:, 1]) * 2 + (Z[:, 2] > 5) * 1.5 + np.random.RandomState(seed).normal(scale=0.3, size=n)
    return X, y.astype(np.float32)


def reference_replay(bst, dtrain, params, rounds, base):
    """Check the weights against the reference replay and return (bins, has_missing, trees, weights)."""
    K = int(params.get("num_class", 1)) if params.get("objective", "").startswith("multi:") else 1
    npt = int(params.get("num_parallel_tree", 1))
    kw = {k: params[k] for k in ("rate_drop", "skip_drop", "sample_type", "one_drop", "normalize_type") if k in params}
    w_ref, drops = R.replay_weights(rounds, float(params.get("eta", 0.3)), K * npt, seed=int(params.get("seed", 0)), **kw)
    w = bst.get_tree_weights()
    assert w.dtype == np.float32 and w.tobytes() == w_ref.tobytes()
    bins = dtrain.get_bins()
    hm = dtrain.get_cuts()[3]
    trees = bst.get_trees()
    full = R.margins(trees, w, bins, hm, base, K, npt)
    got = bst.predict(dtrain, output_margin=True).reshape(-1, K)
    assert got.tobytes() == full.tobytes()
    return drops, bins, hm, trees, w, K, npt


CASES = [
    ("reg:squarederror", {"rate_drop": 0.3}),
    ("binary:logistic", {"rate_drop": 0.2, "sample_type": "weighted"}),
    ("multi:softprob", {"rate_drop": 0.2, "num_class": 3, "normalize_type": "forest"}),
    ("reg:pseudohubererror", {"rate_drop": 0.25, "sample_type": "weighted", "normalize_type": "forest"}),
    ("reg:squarederror", {"rate_drop": 0.0, "one_drop": 1}),
    ("reg:squarederror", {"rate_drop": 0.5, "skip_drop": 0.5, "one_drop": 1, "sample_type": "weighted"}),
    ("reg:squarederror", {"rate_drop": 0.2, "num_parallel_tree": 2, "subsample": 0.7}),
    ("binary:logistic", {"rate_drop": 0.2, "colsample_bynode": 0.5}),
]


def same_as_reference(oracle, bst, params, X, y, rounds, weight=None, is_cat=None, base_margin=None):
    ref = R.train(oracle, params, X, y, rounds, weight=weight, is_cat=is_cat, base_margin=base_margin)
    assert_same_model(bst, ref)
    assert bst.get_tree_weights().tobytes() == ref.weights.tobytes()
    return ref


@pytest.mark.parametrize("objective,extra", CASES)
@pytest.mark.parametrize("depth", [3, 8])
def test_weights_and_margins_match_reference(eng, oracle, objective, extra, depth):
    X, y = dataset(seed=depth)
    rounds = 30
    base = np.random.RandomState(1).normal(scale=0.1, size=(X.shape[0], extra.get("num_class", 1))).astype(np.float32)
    d = eng.DMatrix(X, label=labels(objective, y), base_margin=base.reshape(-1))
    params = {"booster": "dart", "objective": objective, "max_depth": depth, "eta": 0.3, "seed": 7, "base_score": 0.5}
    params.update(extra)
    bst = eng.train(params, d, num_boost_round=rounds, verbose_eval=False)
    same_as_reference(oracle, bst, params, X, labels(objective, y), rounds, base_margin=base)
    drops, bins, hm, trees, w, K, npt = reference_replay(bst, d, params, rounds, base)
    assert sum(1 for x in drops if x) >= (1 if extra.get("rate_drop", 0) == 0 else rounds // 2)
    # the next round's drop margin is what a custom objective sees
    nxt = R.drop_set(w, rounds, seed=7, **{k: extra[k] for k in ("rate_drop", "skip_drop", "sample_type", "one_drop") if k in extra})
    dm = bst.predict(d, output_margin=True, training=True).reshape(-1, K)
    assert dm.tobytes() == R.margins(trees, w, bins, hm, base, K, npt, skip=nxt).tobytes()
    # iteration_range: the first 10 rounds with their final weights
    part = bst.predict(d, output_margin=True, iteration_range=(0, 10)).reshape(-1, K)
    per = K * npt
    assert part.tobytes() == R.margins(trees[:10 * per], w[:10 * per], bins, hm, base, K, npt).tobytes()


def test_nans_weights_and_categorical(eng, oracle):
    X, score, rng = make_cat_data(8000, 3, nan_frac=0.05)
    wt = rng.uniform(0.5, 2.0, size=X.shape[0]).astype(np.float32)
    d = eng.DMatrix(X, label=score, weight=wt, feature_types=["q", "q", "q", "c", "c", "c"], enable_categorical=True)
    params = {"booster": "dart", "objective": "reg:squarederror", "max_depth": 6, "rate_drop": 0.3, "seed": 2,
              "base_score": 0.5}
    bst = eng.train(params, d, num_boost_round=30, verbose_eval=False)
    assert any(t["split_type"].any() for t in bst.get_trees())
    same_as_reference(oracle, bst, params, X, score, 30, weight=wt, is_cat=IS_CAT)
    reference_replay(bst, d, params, 30, np.full((X.shape[0], 1), 0.5, np.float32))


def test_depth_14(eng, oracle):
    X, y = dataset(n=20000, f=20, seed=4)
    d = eng.DMatrix(X, label=y)
    params = {"booster": "dart", "objective": "reg:squarederror", "max_depth": 14, "rate_drop": 0.3, "seed": 3,
              "base_score": 0.5, "min_child_weight": 0}
    bst = eng.train(params, d, num_boost_round=30, verbose_eval=False)
    same_as_reference(oracle, bst, params, X, y, 30)
    reference_replay(bst, d, params, 30, np.full((X.shape[0], 1), 0.5, np.float32))


@pytest.mark.parametrize("extra", [{"rate_drop": 0.0}, {"rate_drop": 0.5, "skip_drop": 1.0}])
@pytest.mark.parametrize("objective", ["reg:squarederror", "multi:softprob"])
def test_no_drops_is_gbtree_byte_for_byte(eng, objective, extra):
    X, y = dataset(seed=9)
    p = {"objective": objective, "max_depth": 6, "seed": 1}
    if objective == "multi:softprob":
        p["num_class"] = 3
    d = eng.DMatrix(X, label=labels(objective, y))
    a = eng.train(p, d, num_boost_round=20, verbose_eval=False)
    b = eng.train(dict(p, booster="dart", **extra), eng.DMatrix(X, label=labels(objective, y)), num_boost_round=20,
                  verbose_eval=False)
    assert a.get_dump(with_stats=True) == b.get_dump(with_stats=True)
    assert list(b.get_tree_weights()) == [1.0] * b.num_trees()
    dx = eng.DMatrix(X)
    assert a.predict(dx).tobytes() == b.predict(dx).tobytes()


def test_custom_objective_sees_the_drop_margin(eng):
    X, y = dataset(seed=5)
    d = eng.DMatrix(X, label=y)
    params = {"booster": "dart", "objective": "reg:squarederror", "max_depth": 5, "rate_drop": 0.3, "seed": 4,
              "base_score": 0.5}
    bst = eng.Booster(params, cache=[d])
    base = np.full((X.shape[0], 1), 0.5, np.float32)
    seen = 0
    for r in range(15):
        pred = bst.predict(d, output_margin=True, training=True)
        w = bst.get_tree_weights()
        drop = R.drop_set(w, r, seed=4, rate_drop=0.3)
        want = R.margins(bst.get_trees(), w, d.get_bins(), d.get_cuts()[3], base, skip=drop)
        assert pred.tobytes() == want.reshape(-1).tobytes(), r
        seen += bool(drop)
        bst.boost(d, pred - y, np.ones_like(pred))
    assert seen >= 5
    # the same objective built in (g = m - y, h = 1 in binary32, the same expression) grows the same model
    b = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=15, verbose_eval=False)
    assert b.save_raw() == bst.save_raw()


def test_eval_sets_follow_the_weights(eng):
    X, y = dataset(n=8000, seed=6)
    Xv, yv = dataset(n=3000, seed=16)
    d, dv = eng.DMatrix(X, label=y), eng.DMatrix(Xv, label=yv)
    params = {"booster": "dart", "objective": "reg:squarederror", "max_depth": 5, "rate_drop": 0.3, "seed": 5,
              "base_score": 0.5}
    log = {}
    checks = []

    class Check(eng.TrainingCallback):
        def after_iteration(self, model, epoch, evals_log):
            for dm, yy, name in ((d, y, "train"), (dv, yv, "valid")):
                p = model.predict(dm, output_margin=True).astype(np.float64)
                rmse = float(np.sqrt(np.mean((p - yy) ** 2)))
                checks.append(abs(evals_log[name]["rmse"][-1] - rmse) < 2e-6)
            return False

    bst = eng.train(params, d, num_boost_round=20, evals=[(d, "train"), (dv, "valid")], evals_result=log,
                    callbacks=[Check()], verbose_eval=False)
    assert len(checks) == 40 and all(checks)
    # rounds drained with and without evals between them give the same model
    plain = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=20, verbose_eval=False)
    assert plain.save_raw() == bst.save_raw()


def test_shap_sums_to_the_margin(eng):
    X, y = dataset(n=3000, seed=8, nan_frac=0.02)
    d = eng.DMatrix(X, label=y)
    params = {"booster": "dart", "objective": "reg:squarederror", "max_depth": 5, "rate_drop": 0.3, "seed": 6,
              "base_score": 0.5}
    bst = eng.train(params, d, num_boost_round=20, verbose_eval=False)
    assert len(set(bst.get_tree_weights().tolist())) > 1
    m = bst.predict(d, output_margin=True).astype(np.float64)
    c = bst.predict(d, pred_contribs=True).astype(np.float64)
    assert np.all(np.abs(c.sum(axis=1) - m) <= 1e-5 * np.maximum(1.0, np.abs(m)))
    it = bst.predict(eng.DMatrix(X[:200]), pred_interactions=True).astype(np.float64)
    assert np.allclose(it.sum(axis=2), c[:200], atol=1e-4)
    # against the float64 reference TreeSHAP of the trees with their leaves scaled by the weights
    w = bst.get_tree_weights()
    scaled = [dict(t, value=t["value"].astype(np.float64) * float(wt)) for t, wt in zip(bst.get_trees(), w)]
    want = SR.shap_contribs(scaled, X, base_value=0.5)[:, 0, :]
    assert np.all(np.abs(c - want) <= 1e-5 * np.maximum(1.0, np.abs(m))[:, None])
    wi = SR.shap_contribs(scaled, X[:50], base_value=0.5, interactions=True)[:, 0]
    assert np.all(np.abs(it[:50] - wi) <= 1e-5 * np.maximum(1.0, np.abs(m[:50]))[:, None, None])


def test_pickle_continue_equals_uninterrupted(eng):
    X, y = dataset(seed=10)
    params = {"booster": "dart", "objective": "reg:squarederror", "max_depth": 5, "rate_drop": 0.3, "seed": 8,
              "base_score": 0.5, "sample_type": "weighted"}
    full = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=10, verbose_eval=False)
    half = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=5, verbose_eval=False)
    half = pickle.loads(pickle.dumps(half))
    assert half.is_dart
    cont = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=5, xgb_model=half, verbose_eval=False)
    assert cont.save_raw() == full.save_raw()


def test_model_file_round_trip_predicts_the_same(eng, tmp_path):
    X, y = dataset(seed=11)
    params = {"booster": "dart", "objective": "binary:logistic", "max_depth": 4, "rate_drop": 0.3, "seed": 9}
    bst = eng.train(params, eng.DMatrix(X, label=labels("binary:logistic", y)), num_boost_round=10, verbose_eval=False)
    f = str(tmp_path / "m.json")
    bst.save_model(f)
    b2 = eng.Booster(model_file=f)
    dx = eng.DMatrix(X)
    assert b2.is_dart and b2.predict(dx).tobytes() == bst.predict(dx).tobytes()


def test_two_million_rows(eng):
    rng = np.random.RandomState(0)
    n = 2_000_000
    X = rng.uniform(0, 10, size=(n, 8)).astype(np.float32)
    y = (X[:, 0] + np.sin(X[:, 1]) * 3 + rng.normal(size=n)).astype(np.float32)
    d = eng.DMatrix(X, label=y)
    params = {"booster": "dart", "objective": "reg:squarederror", "max_depth": 6, "rate_drop": 0.2, "seed": 1,
              "base_score": 0.5}
    bst = eng.train(params, d, num_boost_round=12, verbose_eval=False)
    reference_replay(bst, d, params, 12, np.full((n, 1), 0.5, np.float32))


def test_sklearn_dart_and_bad_parameters(eng):
    from xgboost_ray_b200.sklearn import RayXGBRegressor
    X, y = dataset(n=2000, seed=12)
    r = RayXGBRegressor(n_estimators=8, booster="dart", rate_drop=0.3, max_depth=4)
    r.fit(X, y)
    p = r.predict(X)
    assert p.shape == (2000,) and np.isfinite(p).all() and r.get_booster().is_dart
    d = eng.DMatrix(X, label=y)
    for bad, name in (({"rate_drop": 1.5}, "rate_drop"), ({"skip_drop": -0.1}, "skip_drop"),
                      ({"sample_type": "random"}, "sample_type"), ({"normalize_type": "tree2"}, "normalize_type"),
                      ({"one_drop": 2}, "one_drop")):
        with pytest.raises(eng.XGBoostError, match=name):
            eng.train(dict({"booster": "dart"}, **bad), d, num_boost_round=1, verbose_eval=False)
    # gbtree ignores them, as xgboost does
    eng.train({"rate_drop": 1.5}, d, num_boost_round=1, verbose_eval=False)
    with pytest.raises(eng.XGBoostError, match="booster"):
        eng.train({"booster": "gblinear"}, d, num_boost_round=1, verbose_eval=False)


def test_non_finite_round_leaves_trees_and_weights(eng):
    """reg:gamma with labels far below exp(margin) and no L2 term: the leaves of the first rounds push the margin where
    exp overflows, so a later round's gradients are infinite.  That round raises, and neither its trees nor its weights
    exist: the model keeps the weights of the rounds before it."""
    rng = np.random.RandomState(2)
    X = rng.uniform(0, 10, size=(4000, 6)).astype(np.float32)
    y = np.full(X.shape[0], 1e-3, np.float32)
    params = {"booster": "dart", "objective": "reg:gamma", "base_score": 1.0, "eta": 1.0, "lambda": 1e-6,
              "min_child_weight": 0, "max_depth": 2, "rate_drop": 0.5, "seed": 3}
    dm = eng.DMatrix(X, label=y)
    bst = eng.Booster(params, cache=[dm])
    done = 0
    with pytest.raises(eng.XGBoostError, match="not finite"):
        for r in range(20):
            bst.update(dm, r)
            bst.num_trees()
            done += 1
    assert done >= 1 and bst.num_trees() == done
    w_ref, _ = R.replay_weights(done, 1.0, 1, seed=3, rate_drop=0.5)
    assert bst.get_tree_weights().tobytes() == w_ref.tobytes()


@pytest.mark.timeout(600)
def test_public_api_checkpoint_restart(eng, tmp_path):
    """Kill the actor at round 7 of 10: the driver restarts it from checkpoint 5, and the DART model (trees, weights,
    drop draws keyed by the round) equals the uninterrupted run's."""
    import os
    from tests.fault_injection import DieOnceCallback
    from xgboost_ray_b200 import RayDMatrix, RayParams, predict, train
    X, y = dataset(n=12007, f=9, seed=13, nan_frac=0.03)
    params = {"booster": "dart", "objective": "reg:squarederror", "max_depth": 4, "rate_drop": 0.3, "seed": 4,
              "base_score": 0.5}
    ref = train(params, RayDMatrix(X, y), num_boost_round=10, ray_params=RayParams(num_actors=1, checkpoint_frequency=5))
    lock = str(tmp_path / "lock")
    bst = train(params, RayDMatrix(X, y), num_boost_round=10,
                ray_params=RayParams(num_actors=1, max_actor_restarts=1, checkpoint_frequency=5),
                callbacks=[DieOnceCallback(lock, rank=0, at=7)])
    assert os.path.exists(lock)
    assert bst.is_dart and bst.num_boosted_rounds() == 10
    assert bst.save_raw() == ref.save_raw()
    assert len(set(bst.get_tree_weights().tolist())) > 1
    p = predict(bst, RayDMatrix(X), ray_params=RayParams(num_actors=1))
    assert p.tobytes() == ref.predict(eng.DMatrix(X)).tobytes()


@pytest.mark.timeout(300)
def test_two_gpus_identical_to_one(eng):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    X, y = dataset(n=30001, f=12, seed=14, nan_frac=0.03)
    params = {"booster": "dart", "objective": "binary:logistic", "max_depth": 6, "rate_drop": 0.3, "seed": 5,
              "base_score": 0.5}
    yb = labels("binary:logistic", y)
    b1 = train(params, RayDMatrix(X, yb), num_boost_round=12, ray_params=RayParams(num_actors=1))
    b2 = train(params, RayDMatrix(X, yb), num_boost_round=12, ray_params=RayParams(num_actors=2))
    assert b1.save_raw() == b2.save_raw()


def test_train_feval_gets_the_full_margin_and_weights_are_checked(eng):
    X, y = dataset(n=4000, seed=15)
    d = eng.DMatrix(X, label=y)
    params = {"booster": "dart", "objective": "reg:squarederror", "max_depth": 4, "rate_drop": 0.5, "seed": 6,
              "base_score": 0.5}
    seen = []

    def fsum(pred, dm):
        seen.append(pred.copy())
        return "msum", float(np.sum(pred, dtype=np.float64))

    bst = eng.train(params, d, num_boost_round=6, evals=[(d, "train")], feval=fsum, verbose_eval=False)
    assert seen[-1].tobytes() == bst.predict(d, output_margin=True).tobytes()
    zeros = np.zeros(bst.num_trees(), np.float32)
    with pytest.raises(eng.XGBoostError, match="total weight"):
        eng._check(eng.lib().B2_BoosterSetTreeWeights(bst.handle, eng._fp(zeros), zeros.size))
