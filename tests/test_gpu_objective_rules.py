"""The engine's refusals of an eval metric that does not fit the model or the matrix, and of train labels outside an
objective's domain, each matched against its whole message: the rules live in one table per objective and metric, and
these tests pin which rule fires and what it says."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N = 200
SUPPORTED = ("rmse, mae, logloss, error, auc, aucpr, mlogloss, merror, rmsle, mape, mphe, poisson-nloglik, gamma-nloglik, "
             "gamma-deviance, tweedie-nloglik@rho, aft-nloglik, interval-regression-accuracy, quantile, ndcg[@k][-], "
             "map[@k][-], pre[@k][-]")
MULTI_TARGET = "rmse, rmsle, mae, mape, mphe, logloss, error"


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def features(seed=0):
    return np.random.RandomState(seed).uniform(0, 1, size=(N, 4)).astype(np.float32)


def binary():
    return (features()[:, 0] > 0.5).astype(np.float32)


def qid():
    return np.repeat(np.arange(N // 10), 10)


def bounds():
    lo = (1.0 + features()[:, 1]).astype(np.float32)
    return lo, (lo * 2).astype(np.float32)


def matrix(eng, kind):
    X = features()
    if kind == "binary":
        return eng.DMatrix(X, label=binary())
    if kind == "class3":
        return eng.DMatrix(X, label=(X[:, 0] * 3).astype(np.int32).astype(np.float32))
    if kind == "two_targets":
        return eng.DMatrix(X, label=np.stack([binary(), 1 - binary()], axis=1), multi_target=True)
    if kind == "groups":
        return eng.DMatrix(X, label=binary(), qid=qid())
    if kind == "groups_no_label":
        return eng.DMatrix(X, qid=qid())
    if kind == "no_label":
        return eng.DMatrix(X)
    if kind == "bounds":
        lo, hi = bounds()
        return eng.DMatrix(X, label_lower_bound=lo, label_upper_bound=hi)
    raise ValueError(kind)


MODELS = {
    "squarederror": ({"objective": "reg:squarederror"}, "binary"),
    "softprob": ({"objective": "multi:softprob", "num_class": 3}, "class3"),
    "two_targets": ({"objective": "reg:squarederror"}, "two_targets"),
    "quantile2": ({"objective": "reg:quantileerror", "quantile_alpha": [0.25, 0.75]}, "binary"),
    "aft": ({"objective": "survival:aft"}, "bounds"),
    "ndcg": ({"objective": "rank:ndcg"}, "groups"),
}


def evaluate(eng, model, metric, on=None):
    """B2_BoosterEvalSet of `metric` on matrix `on` (default: the train matrix) of a one-round model."""
    params, train_kind = MODELS[model]
    bst = eng.train(dict(params, max_depth=2), matrix(eng, train_kind), 1, verbose_eval=False)
    dm = bst._train if on is None else matrix(eng, on)
    dm._ensure_raw()
    v = C.c_double(0)
    eng._check(eng.lib().B2_BoosterEvalSet(bst.handle, dm.handle, metric.encode(), C.byref(v)))
    return v.value


# (model, metric, evaluation matrix or None for the train matrix, the whole message)
EVAL_REFUSED = [
    ("squarederror", "bogus", None, "unsupported eval metric 'bogus' (supported: %s)" % SUPPORTED),
    ("squarederror", "tweedie-nloglik@2.5", None,
     "eval metric 'tweedie-nloglik@2.5': the Tweedie power must be given as tweedie-nloglik@rho with rho in [1, 2)"),
    ("squarederror", "tweedie-nloglik1.5", None,
     "eval metric 'tweedie-nloglik1.5': the Tweedie power must be given as tweedie-nloglik@rho with rho in [1, 2)"),
    ("squarederror", "ndcg@0", None, "eval metric 'ndcg@0': the cut-off must be given as ndcg@k with an integer k >= 1"),
    ("squarederror", "mapx-", None, "eval metric 'mapx-': the cut-off must be given as map@k with an integer k >= 1"),
    ("softprob", "ndcg", None, "metric 'ndcg' needs a single-output objective"),
    ("squarederror", "map@3", None, "metric 'map@3' needs query groups (qid) on the evaluation matrix"),
    ("ndcg", "pre", "groups_no_label", "evaluation matrix has no labels"),
    ("squarederror", "auc", "groups",
     "metric 'auc' on a matrix with query groups (per-group ranking AUC) is not supported; use ndcg or map"),
    ("two_targets", "auc", None,
     "metric 'auc' is not supported for a multi-target model (2 targets); use rmse, mae, logloss or error"),
    ("quantile2", "aucpr", None,
     "metric 'aucpr' needs one output per row or a multi:softprob / multi:softmax model; objective 'reg:quantileerror' "
     "has 2 outputs"),
    ("squarederror", "aft-nloglik", "bounds", "metric 'aft-nloglik' does not fit objective 'reg:squarederror'"),
    ("aft", "interval-regression-accuracy", "binary",
     "metric 'interval-regression-accuracy' needs label_lower_bound and label_upper_bound on the evaluation matrix"),
    ("two_targets", "rmse", "binary", "metric 'rmse': the evaluation matrix's label has 1 columns, the model has 2 targets"),
    ("squarederror", "rmse", "no_label", "evaluation matrix has no labels"),
    ("squarederror", "mlogloss", None, "metric 'mlogloss' does not fit objective 'reg:squarederror'"),
    ("softprob", "error", None, "metric 'error' does not fit objective 'multi:softprob'"),
    ("squarederror", "quantile", None, "metric 'quantile' needs objective reg:quantileerror (it reads quantile_alpha)"),
    ("two_targets", "poisson-nloglik", None,
     "metric 'poisson-nloglik' is not supported for a multi-target model (supported: %s)" % MULTI_TARGET),
]


@pytest.mark.parametrize("model,metric,on,msg", EVAL_REFUSED,
                         ids=["%s-%s-%s" % (m, metric, on) for m, metric, on, _ in EVAL_REFUSED])
def test_eval_refusal(eng, model, metric, on, msg):
    with pytest.raises(eng.XGBoostError) as e:
        evaluate(eng, model, metric, on)
    assert str(e.value) == msg


# (objective, bad label, the whole message of check_labels / check_rank_labels)
LABEL_REFUSED = [
    ("binary:logitraw", 1.5, "label must be in [0, 1] for binary:logitraw"),
    ("reg:squaredlogerror", -1.0, "label must be greater than -1 for reg:squaredlogerror"),
    ("reg:quantileerror", np.inf, "label must be finite for reg:quantileerror"),
    ("multi:softmax", 3.0, "label must be in [0, num_class) for multi:softmax, num_class = 3"),
    ("rank:map", 2.0, "rank:map: labels must be 0 or 1 (binary relevance); use rank:ndcg for graded relevance"),
    ("rank:ndcg", -1.0, "rank:ndcg: labels must be finite and >= 0"),
    ("rank:pairwise", 32.0,
     "rank:pairwise: with ndcg_exp_gain the labels must be <= 31 (the gain is 2^label - 1); set ndcg_exp_gain=false for "
     "larger relevance degrees"),
]


@pytest.mark.parametrize("objective,bad,msg", LABEL_REFUSED, ids=[c[0] for c in LABEL_REFUSED])
def test_label_refusal(eng, objective, bad, msg):
    y = binary()
    y[17] = bad
    params = {"objective": objective, "num_class": 3} if objective == "multi:softmax" else {"objective": objective}
    dm = eng.DMatrix(features(), label=y, qid=qid()) if objective.startswith("rank:") else eng.DMatrix(features(), label=y)
    with pytest.raises(eng.XGBoostError) as e:
        eng.train(params, dm, 1, verbose_eval=False)
    assert str(e.value) == msg


def test_aft_nan_bound_refused(eng):
    lo, hi = bounds()
    lo[5] = np.nan
    dm = eng.DMatrix(features(), label_lower_bound=lo, label_upper_bound=hi)
    with pytest.raises(eng.XGBoostError) as e:
        eng.train({"objective": "survival:aft"}, dm, 1, verbose_eval=False)
    assert str(e.value) == "survival:aft: label bounds must not be NaN"


def test_rank_needs_groups_on_every_check(eng):
    """The query groups are checked whenever the train margin is rebuilt, also after the labels passed their check."""
    dm = matrix(eng, "groups")
    bst = eng.train({"objective": "rank:pairwise", "max_depth": 2}, dm, 1, verbose_eval=False)
    eng._check(eng.lib().B2_MatrixSetGroups(dm.handle, None, 0))
    with pytest.raises(eng.XGBoostError) as e:
        eng._check(eng.lib().B2_BoosterResetTrainMargin(bst.handle))
    assert str(e.value) == ("rank:pairwise needs query groups on the train matrix: pass qid (or group) to the "
                            "DMatrix")
