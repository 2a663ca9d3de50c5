"""reg:quantileerror on the GPU.

Every model is compared with tests/quantile_reference.py (the oracle grows each tree from the pinball gradients, the
reference refreshes its leaves with np.sort): the trees with assert_same_model and every leaf value bit for bit, the
estimated intercept exactly.  Also the quantile metric, the coverage of the fitted quantiles, the failure of a
non-finite input, continuation, several GPUs and the refused parameter combinations."""
import pickle

import numpy as np
import pytest

from tests import quantile_reference as R
from tests.test_gpu_parity import IS_CAT, assert_same_model, make_cat_data, make_data

pytestmark = pytest.mark.gpu
F32 = np.float32


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def dataset(n=6000, f=10, seed=0, nan_frac=0.0):
    X = make_data(n, f, seed, "uniform", nan_frac)
    Z = np.nan_to_num(X, nan=5.0)
    rng = np.random.RandomState(seed)
    y = Z[:, 0] * 0.5 + np.sin(Z[:, 1]) * 2 + rng.standard_t(3, size=n) * (0.3 + 0.1 * Z[:, 2])
    return X, y.astype(F32)


def same_as_reference(oracle, bst, params, X, y, rounds, weight=None, is_cat=None, base_margin=None):
    ref = R.train(oracle, params, X, y, rounds, weight=weight, is_cat=is_cat, base_margin=base_margin)
    assert_same_model(bst, ref)
    for i, t in enumerate(bst.get_trees()):
        leaf = t["split_feature"] < 0
        assert t["value"][leaf].tobytes() == ref.tree(i).value[leaf].tobytes(), "tree %d leaf values" % i
    if params.get("base_score") is None:
        assert F32(bst.params["base_score"]) == ref.base_score
    return ref


@pytest.mark.parametrize("alpha", [0.1, 0.5, 0.9, [0.05, 0.5, 0.95]])
@pytest.mark.parametrize("depth", [3, 8])
def test_matches_reference(eng, oracle, alpha, depth):
    X, y = dataset(seed=depth)
    params = {"objective": "reg:quantileerror", "quantile_alpha": alpha, "max_depth": depth, "eta": 0.3}
    d = eng.DMatrix(X, label=y)
    bst = eng.train(params, d, num_boost_round=8, verbose_eval=False)
    ref = same_as_reference(oracle, bst, params, X, y, 8)
    T = np.size(alpha)
    m = bst.predict(d, output_margin=True)
    assert m.shape == ((len(y), T) if T > 1 else (len(y),))
    assert m.reshape(len(y), T).tobytes() == ref.margin.tobytes()
    # the train margin cache and prediction agree; iteration_range counts rounds of T trees
    assert bst.predict(d, training=True).tobytes() == m.tobytes()
    assert bst.predict(d, iteration_range=(0, 3)).shape == m.shape
    assert bst.num_boosted_rounds() == 8 and bst.num_trees() == 8 * T


VARIANTS = ["int_weights", "frac_weights", "nan_categorical", "sampling"]


# depth 6 and 7 sit on either side of the weighted count pass's shared-memory limit (quantile_kernel.cu)
@pytest.mark.parametrize("variant,depth", [(v, 6) for v in VARIANTS] + [(v, 7) for v in VARIANTS],
                         ids=VARIANTS + [v + "-depth7" for v in VARIANTS])
def test_variants_match_reference(eng, oracle, variant, depth):
    rng = np.random.RandomState(3)
    params = {"objective": "reg:quantileerror", "quantile_alpha": [0.2, 0.8], "max_depth": depth, "eta": 0.4}
    is_cat, kw, w = None, {}, None
    if variant == "nan_categorical":
        X, y, rng = make_cat_data(8000, 5, nan_frac=0.05)
        y = (y + rng.normal(size=len(y))).astype(F32)
        is_cat = IS_CAT
        kw = {"feature_types": ["q", "q", "q", "c", "c", "c"], "enable_categorical": True}
    else:
        X, y = dataset(seed=4)
    if variant == "int_weights":
        w = rng.randint(0, 6, size=len(y)).astype(F32)
    elif variant == "frac_weights":
        w = rng.uniform(0.1, 3.0, size=len(y)).astype(F32)
    elif variant == "sampling":
        params.update(subsample=0.7, colsample_bytree=0.8, colsample_bynode=0.7, seed=9, base_score=0.5)
    d = eng.DMatrix(X, label=y, weight=w, **kw)
    bst = eng.train(params, d, num_boost_round=6, verbose_eval=False)
    if variant == "nan_categorical":
        assert any(t["split_type"].any() for t in bst.get_trees())
    same_as_reference(oracle, bst, params, X, y, 6, weight=w, is_cat=is_cat)


def test_depth_14(eng, oracle):
    X, y = dataset(n=30000, f=16, seed=6)
    params = {"objective": "reg:quantileerror", "quantile_alpha": [0.3, 0.7], "max_depth": 14, "min_child_weight": 0}
    bst = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=3, verbose_eval=False)
    same_as_reference(oracle, bst, params, X, y, 3)


@pytest.mark.timeout(900)
def test_two_million_rows_and_coverage(eng, oracle):
    n = 2_000_000
    X, y = dataset(n=n, f=8, seed=8)
    params = {"objective": "reg:quantileerror", "quantile_alpha": [0.1, 0.5, 0.9], "max_depth": 6, "eta": 0.5}
    d = eng.DMatrix(X, label=y)
    bst = eng.train(params, d, num_boost_round=3, verbose_eval=False)
    same_as_reference(oracle, bst, params, X, y, 3)
    # the fitted quantiles cover their share of 1M held-in rows
    bst = eng.train(params, d, num_boost_round=40, verbose_eval=False)
    p = bst.predict(eng.DMatrix(X[:1_000_000]))
    for k, a in enumerate([0.1, 0.5, 0.9]):
        assert abs(np.mean(y[:1_000_000] < p[:, k]) - a) <= 0.01


def test_metric_is_pinball_loss(eng):
    X, y = dataset(seed=11)
    w = np.random.RandomState(2).uniform(0.5, 2, size=len(y)).astype(F32)
    alphas = [0.05, 0.5, 0.95]
    d = eng.DMatrix(X, label=y, weight=w)
    res = {}
    bst = eng.train({"objective": "reg:quantileerror", "quantile_alpha": alphas, "max_depth": 4}, d, num_boost_round=5,
                    evals=[(d, "train")], evals_result=res, verbose_eval=False)
    assert list(res["train"]) == ["quantile"]
    got = float(bst.eval_set([(d, "train")]).split("train-quantile:")[1])
    want = R.pinball(bst.predict(d, output_margin=True), y, w, alphas)
    assert abs(got - want) <= 1e-6 * max(1.0, want)
    with pytest.raises(eng.XGBoostError, match="quantile"):
        eng.train({"objective": "reg:squarederror", "eval_metric": "quantile"}, d, num_boost_round=1, evals=[(d, "t")],
                  verbose_eval=False)


def test_non_finite_input_commits_nothing(eng):
    """The pinball pairs are finite for finite labels and weights, so a round can only fail on its inputs: a label
    that is NaN or infinite fails the first round before any tree exists, and an infinite weight is refused."""
    X, y = dataset(seed=12)
    for bad in (np.nan, np.inf):
        y2 = y.copy()
        y2[3] = bad
        d = eng.DMatrix(X, label=y2)
        bst = eng.Booster({"objective": "reg:quantileerror", "quantile_alpha": [0.3, 0.6]}, [d])
        with pytest.raises(eng.XGBoostError, match="label must be finite"):
            bst.update(d, 0)
        assert bst.num_trees() == 0
    w = np.ones(len(y), F32)
    w[7] = np.inf
    with pytest.raises(eng.XGBoostError, match="finite"):
        eng.train({"objective": "reg:quantileerror"}, eng.DMatrix(X, label=y, weight=w), num_boost_round=1,
                  verbose_eval=False)


def test_continuation_and_checkpoint(eng):
    X, y = dataset(seed=13)
    params = {"objective": "reg:quantileerror", "quantile_alpha": [0.25, 0.75], "max_depth": 5}
    d = eng.DMatrix(X, label=y)
    full = eng.train(params, d, num_boost_round=8, verbose_eval=False)
    first = eng.train(params, d, num_boost_round=4, verbose_eval=False)
    resumed = eng.train(params, d, num_boost_round=4, verbose_eval=False, xgb_model=pickle.loads(pickle.dumps(first)))
    assert bytes(resumed.save_raw()) == bytes(full.save_raw())
    path_model = bytearray(first.save_raw())
    resumed2 = eng.train({"objective": "reg:quantileerror", "max_depth": 5}, d, num_boost_round=4, verbose_eval=False,
                         xgb_model=path_model)
    assert bytes(resumed2.save_raw()) == bytes(full.save_raw())
    with pytest.raises(eng.XGBoostError, match="quantile_alpha"):
        eng.train(dict(params, quantile_alpha=[0.25, 0.8]), d, num_boost_round=1, verbose_eval=False, xgb_model=first)


def test_public_api_and_sklearn(eng, oracle):
    from xgboost_ray_b200 import RayDMatrix, RayParams, predict, train
    from xgboost_ray_b200.sklearn import RayXGBRegressor
    X, y = dataset(seed=14)
    params = {"objective": "reg:quantileerror", "quantile_alpha": [0.1, 0.9], "max_depth": 4}
    bst = train(params, RayDMatrix(X, y), num_boost_round=4, ray_params=RayParams(num_actors=1))
    same_as_reference(oracle, bst, params, X, y, 4)
    p = predict(bst, RayDMatrix(X), ray_params=RayParams(num_actors=1))
    assert p.shape == (len(y), 2)
    r = RayXGBRegressor(objective="reg:quantileerror", quantile_alpha=[0.1, 0.9], max_depth=4, n_estimators=4)
    r.fit(X, y)
    assert r.predict(X).tobytes() == p.tobytes()


@pytest.mark.timeout(300)
def test_two_gpus_and_two_actors_same_model(eng):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    X, y = dataset(n=30001, seed=15, nan_frac=0.05)
    w = np.random.RandomState(3).uniform(0.5, 2, size=len(y)).astype(F32)
    for depth in (6, 8):          # weighted counts in shared memory, then in global memory
        params = {"objective": "reg:quantileerror", "quantile_alpha": [0.1, 0.5, 0.9], "max_depth": depth}
        b1 = train(params, RayDMatrix(X, y, weight=w), num_boost_round=5, ray_params=RayParams(num_actors=1))
        b2 = train(params, RayDMatrix(X, y, weight=w), num_boost_round=5, ray_params=RayParams(num_actors=2))
        assert bytes(b1.save_raw()) == bytes(b2.save_raw()), "max_depth %d" % depth


@pytest.mark.parametrize("extra,match", [({"num_class": 2}, "num_class"), ({"booster": "dart"}, "dart"),
                                         ({"num_parallel_tree": 2}, "num_parallel_tree"),
                                         ({"quantile_alpha": 1.0}, "quantile_alpha")])
def test_rejected_combinations_raise(eng, extra, match):
    X, y = dataset(n=500, seed=16)
    with pytest.raises(eng.XGBoostError, match=match):
        eng.train(dict({"objective": "reg:quantileerror"}, **extra), eng.DMatrix(X, label=y), num_boost_round=1,
                  verbose_eval=False)
    with pytest.raises(eng.XGBoostError):   # one label column only
        eng.DMatrix(X, label=np.stack([y, y], axis=1))
