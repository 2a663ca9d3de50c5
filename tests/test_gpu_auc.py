"""`auc` and `aucpr` on the GPU, binary and one-vs-rest over the classes of a softmax model.

Every value is compared with tests/auc_reference.py on the engine's own predictions of the same matrix: through
`evals_result` (six printed decimals) within 2e-6, through B2_BoosterEvalSet directly within 1e-9.  Also the NaN and
error rules, repeatability, early stopping, the sklearn estimator and two GPUs against the reference's multi-worker
rule."""
import ctypes as C
import math

import numpy as np
import pytest

from tests import auc_reference as R

pytestmark = pytest.mark.gpu
F32 = np.float32


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def direct(eng, bst, dm, metric):
    """B2_BoosterEvalSet without the printed rounding."""
    dm._ensure_raw()
    v = C.c_double(0)
    eng._check(eng.lib().B2_BoosterEvalSet(bst.handle, dm.handle, metric.encode(), C.byref(v)))
    return v.value


def binary_data(n, seed, weighted):
    rng = np.random.RandomState(seed)
    X = np.round(rng.uniform(0, 10, size=(n, 6)), 0).astype(F32)          # coarse values: many tied predictions
    y = (X[:, 0] + X[:, 1] + rng.normal(scale=3.0, size=n) > 11).astype(F32)
    w = rng.gamma(2.0, 1.0, size=n).astype(F32) if weighted else None
    return X, y, w


def multiclass_data(n, K, seed, weighted=False):
    rng = np.random.RandomState(seed)
    X = np.round(rng.uniform(0, 10, size=(n, 8)), 0).astype(F32)
    y = (X[:, 0] * 11 + X[:, 1]).astype(np.int64) % K                     # every class about equally frequent
    noise = rng.uniform(size=n) < 0.3
    y = np.where(noise, rng.randint(0, K, size=n), y).astype(F32)
    w = rng.uniform(0.2, 3.0, size=n).astype(F32) if weighted else None
    return X, y, w


def check(eng, bst, res, name, dm, label, weight, metrics, pred=None, shards=None):
    p = bst.predict(dm) if pred is None else pred
    for metric in metrics:
        want = R.value(metric, p, label, weight, shards)
        assert abs(res[name][metric][-1] - want) < 2e-6, (metric, res[name][metric][-1], want)
        if shards is None:
            got = direct(eng, bst, dm, metric)
            assert abs(got - want) < 1e-9, (metric, got, want)


@pytest.mark.parametrize("weighted", [False, True])
def test_binary_aucpr_and_auc(eng, weighted):
    X, y, w = binary_data(40000, 1, weighted)
    Xv, yv, wv = X[:15000] + F32(0.25), y[:15000], None if w is None else w[:15000]
    dm = eng.DMatrix(X, label=y, weight=w)
    dv = eng.DMatrix(Xv, label=yv, weight=wv)
    params = {"objective": "binary:logistic", "max_depth": 3, "eta": 0.3, "base_score": 0.5,
              "eval_metric": ["auc", "aucpr"]}
    res = {}
    bst = eng.train(params, dm, num_boost_round=6, evals=[(dm, "train"), (dv, "valid")], evals_result=res,
                    verbose_eval=False)
    p = bst.predict(dv)
    assert len(np.unique(p)) < len(p) // 4                                  # heavy ties
    check(eng, bst, res, "valid", dv, yv, wv, ["auc", "aucpr"], pred=p)
    pt = bst.predict(eng.DMatrix(X))
    for metric in ("auc", "aucpr"):
        assert abs(res["train"][metric][-1] - R.value(metric, pt, y, w)) < 2e-6
    assert 0.5 < res["valid"]["aucpr"][-1] < 1.0


@pytest.mark.parametrize("K,weighted", [(3, True), (20, False)])
def test_multiclass_ovr(eng, K, weighted):
    X, y, w = multiclass_data(30000, K, seed=K, weighted=weighted)
    Xv, yv, wv = X[:12000] + F32(0.25), y[:12000], None if w is None else w[:12000]
    dm = eng.DMatrix(X, label=y, weight=w)
    dv = eng.DMatrix(Xv, label=yv, weight=wv)
    assert len(np.unique(yv)) == K
    base = {"num_class": K, "max_depth": 4, "eta": 0.3, "eval_metric": ["auc", "aucpr"]}
    res, res_max = {}, {}
    soft = eng.train(dict(base, objective="multi:softprob"), dm, num_boost_round=4, evals=[(dv, "valid")],
                     evals_result=res, verbose_eval=False)
    hard = eng.train(dict(base, objective="multi:softmax"), dm, num_boost_round=4, evals=[(dv, "valid")],
                     evals_result=res_max, verbose_eval=False)
    P = soft.predict(dv)
    assert P.shape == (len(yv), K)
    check(eng, soft, res, "valid", dv, yv, wv, ["auc", "aucpr"], pred=P)
    # multi:softmax grows the same trees and its metrics read the same probabilities, not the argmax
    assert np.array_equal(hard.predict(dv, output_margin=True), soft.predict(dv, output_margin=True))
    check(eng, hard, res_max, "valid", dv, yv, wv, ["auc", "aucpr"], pred=P)
    assert res_max == res


def test_absent_class_gives_nan(eng):
    X, y, _ = multiclass_data(6000, 3, seed=5)
    bst = eng.train({"objective": "multi:softprob", "num_class": 3, "max_depth": 3}, eng.DMatrix(X, label=y), 3,
                    verbose_eval=False)
    keep = y != 1
    dv = eng.DMatrix(X[keep], label=y[keep])
    for metric in ("auc", "aucpr"):
        assert math.isnan(direct(eng, bst, dv, metric))
        assert math.isnan(R.value(metric, bst.predict(dv), y[keep]))
    res = {}
    eng.train({"objective": "multi:softprob", "num_class": 3, "max_depth": 3, "eval_metric": "aucpr"},
              eng.DMatrix(X, label=y), 2, evals=[(dv, "v")], evals_result=res, verbose_eval=False)
    assert all(math.isnan(v) for v in res["v"]["aucpr"])
    # binary: one class only -> auc 0.5 (unchanged), aucpr NaN
    Xb, yb, _ = binary_data(3000, 6, False)
    bb = eng.train({"objective": "binary:logistic", "max_depth": 3}, eng.DMatrix(Xb, label=yb), 2, verbose_eval=False)
    ones = eng.DMatrix(Xb[:200], label=np.ones(200, F32))
    assert direct(eng, bb, ones, "auc") == 0.5
    assert math.isnan(direct(eng, bb, ones, "aucpr"))


@pytest.mark.parametrize("bad", [3.0, -1.0, np.nan])
def test_bad_label_fails(eng, bad):
    X, y, _ = multiclass_data(5000, 3, seed=7)
    bst = eng.train({"objective": "multi:softprob", "num_class": 3, "max_depth": 3}, eng.DMatrix(X, label=y), 2,
                    verbose_eval=False)
    yb = y.copy()
    yb[123] = bad
    dv = eng.DMatrix(X, label=yb)
    for metric in ("auc", "aucpr"):
        with pytest.raises(eng.XGBoostError, match=r"label must be in \[0, num_class\)"):
            direct(eng, bst, dv, metric)


def test_refused_combinations(eng):
    X, y, _ = binary_data(2000, 8, False)
    qid = np.repeat(np.arange(100), 20)
    bst = eng.train({"objective": "binary:logistic", "max_depth": 3}, eng.DMatrix(X, label=y), 2, verbose_eval=False)
    dq = eng.DMatrix(X, label=y, qid=qid)
    for metric in ("auc", "aucpr"):
        with pytest.raises(eng.XGBoostError, match="query groups"):
            direct(eng, bst, dq, metric)
    q = eng.train({"objective": "reg:quantileerror", "quantile_alpha": [0.2, 0.8], "max_depth": 3},
                  eng.DMatrix(X, label=y), 2, verbose_eval=False)
    for metric in ("auc", "aucpr"):
        with pytest.raises(eng.XGBoostError, match="multi:softprob"):
            direct(eng, q, eng.DMatrix(X, label=y), metric)
    with pytest.raises(eng.XGBoostError, match="aucpr"):                  # the supported list names it
        direct(eng, bst, eng.DMatrix(X, label=y), "aucroc")


def test_repeated_calls_are_identical(eng):
    X, y, w = binary_data(300000, 9, True)
    bst = eng.train({"objective": "binary:logistic", "max_depth": 6}, eng.DMatrix(X, label=y, weight=w), 4,
                    verbose_eval=False)
    dv = eng.DMatrix(X + F32(0.5), label=y, weight=w)
    Xm, ym, _ = multiclass_data(300000, 5, seed=9)
    bm = eng.train({"objective": "multi:softprob", "num_class": 5, "max_depth": 5}, eng.DMatrix(Xm, label=ym), 3,
                   verbose_eval=False)
    dmv = eng.DMatrix(Xm + F32(0.5), label=ym)
    for b, d in ((bst, dv), (bm, dmv)):
        for metric in ("auc", "aucpr"):
            vals = [direct(eng, b, d, metric) for _ in range(4)]
            assert len({v.hex() for v in vals}) == 1, vals


def test_early_stopping_on_aucpr(eng):
    X, y, w = binary_data(20000, 10, True)
    rng = np.random.RandomState(10)
    flip = rng.uniform(size=len(y)) < 0.15
    yv = np.where(flip, 1 - y, y).astype(F32)                              # a noisy validation set overfits soon
    dm = eng.DMatrix(X, label=y, weight=w)
    dv = eng.DMatrix(X + F32(0.25), label=yv)
    res = {}
    bst = eng.train({"objective": "binary:logistic", "max_depth": 8, "eta": 0.6, "eval_metric": "aucpr"}, dm, 60,
                    evals=[(dv, "valid")], evals_result=res, early_stopping_rounds=4, verbose_eval=False)
    hist = res["valid"]["aucpr"]
    assert bst.best_iteration == int(np.argmax(hist))
    assert bst.best_score == max(hist)


def test_sklearn_classifier_three_classes(eng):
    from xgboost_ray_b200.sklearn import RayXGBClassifier
    X, y, _ = multiclass_data(9000, 3, seed=11)
    Xv, yv = X[:3000] + F32(0.25), y[:3000]
    clf = RayXGBClassifier(n_estimators=4, max_depth=4, eval_metric=["auc", "aucpr"])
    clf.fit(X, y, eval_set=[(Xv, yv)])
    res = clf.evals_result()["validation_0"]
    P = clf.predict_proba(Xv)
    for metric in ("auc", "aucpr"):
        assert len(res[metric]) == 4
        assert abs(res[metric][-1] - R.value(metric, P, yv)) < 2e-6


@pytest.mark.timeout(300)
def test_two_gpus_match_the_multi_worker_rule(eng):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    shards = [slice(0, None, 2), slice(1, None, 2)]                       # RayDMatrix's default INTERLEAVED sharding
    X, y, w = binary_data(20001, 12, True)
    Xv, yv, wv = X[:8001] + F32(0.25), y[:8001], w[:8001]
    res = {}
    bst = train({"objective": "binary:logistic", "max_depth": 4, "eval_metric": ["auc", "aucpr"]},
                RayDMatrix(X, y, weight=w), num_boost_round=4, evals=[(RayDMatrix(Xv, yv, weight=wv), "valid")],
                evals_result=res, ray_params=RayParams(num_actors=2))
    check(eng, bst, res, "valid", eng.DMatrix(Xv), yv, wv, ["auc", "aucpr"], shards=shards)
    Xm, ym, _ = multiclass_data(15001, 4, seed=12)
    Xmv, ymv = Xm[:6001] + F32(0.25), ym[:6001]
    res = {}
    bm = train({"objective": "multi:softprob", "num_class": 4, "max_depth": 4, "eval_metric": ["auc", "aucpr"]},
               RayDMatrix(Xm, ym), num_boost_round=3, evals=[(RayDMatrix(Xmv, ymv), "valid")], evals_result=res,
               ray_params=RayParams(num_actors=2))
    check(eng, bm, res, "valid", eng.DMatrix(Xmv), ymv, None, ["auc", "aucpr"], shards=shards)
