"""Every evaluation metric read through B2_BoosterEvalSet (not the six printed decimals) against its float64 reference,
within |got - want| <= 2^-40 sum w S / sum w (tests/metric_bound.py), at the row counts where the metric kernels' grid
stride wraps, with planted rows at the seams, across weights and at each metric's domain edges; the sums are the same
bits on every call; and the cached evaluation margins follow every edit of the model.

The inputs carry fixed margins: a one-round model with eta = 0 adds +-0 to the evaluation matrix's base_margin, and
every reference reads the engine's own float32 margins from predict(output_margin=True)."""
import ctypes as C

import numpy as np
import pytest

from tests import metric_bound as B
from tests import multi_target_reference as MT
from tests import objective_reference as O
from tests import quantile_reference as Q
from tests import survival_reference as SR
from tests.test_metric_reference import oracle_metric

pytestmark = pytest.mark.gpu
F32 = np.float32


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


@pytest.fixture(scope="module")
def C_rows():
    """Rows at which the metric kernels' grid (at most 16 CTAs of 256 threads per SM) starts a second grid stride."""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256


def evaluate(eng, bst, d, name):
    d._ensure_raw()
    out = C.c_double(0)
    eng._check(eng.lib().B2_BoosterEvalSet(bst.handle, d.handle, name.encode(), C.byref(out)))
    return out.value


# ---- models whose tree adds nothing: the margin is the evaluation matrix's base_margin
SOFTPROB = {"objective": "multi:softprob"}
_models = {}


def null_model(eng, params, outputs=1, family="scalar"):
    key = (repr(sorted(params.items())), outputs, family)
    if key in _models:
        return _models[key]
    X = np.arange(8, dtype=F32).reshape(-1, 1)
    y = np.array([0.25, 0.75] * 4, F32)
    p = dict(params, eta=0.0, max_depth=1)
    if family == "softprob":
        d = eng.DMatrix(X, label=np.arange(8, dtype=F32) % outputs)
        p.update(num_class=outputs)
    elif family == "aft":
        d = eng.DMatrix(X, label_lower_bound=np.ones(8, F32), label_upper_bound=np.full(8, 2, F32))
    elif family == "multi_target":
        d = eng.DMatrix(X, label=np.tile(y[:, None], (1, outputs)), multi_target=True)
    else:
        d = eng.DMatrix(X, label=y)
    bst = eng.train(p, d, 1, verbose_eval=False)
    _models[key] = bst
    return bst


def matrix(eng, bst, margin, label=None, weight=None, lower=None, upper=None, multi_target=False):
    n = len(margin)
    d = eng.DMatrix(np.zeros((n, 1), F32), label=label, weight=weight, base_margin=np.asarray(margin, F32).reshape(-1),
                    label_lower_bound=lower, label_upper_bound=upper, multi_target=multi_target)
    got = bst.predict(d, output_margin=True)
    assert np.array_equal(got.reshape(-1), np.asarray(margin, F32).reshape(-1)), "the model added to the margin"
    return d, got


def check(eng, bst, d, name, want, S, weight=None, exact=False):
    got = evaluate(eng, bst, d, name)
    if exact:
        assert got == want, (name, got, want)
    else:
        B.assert_within(got, want, S, weight, name)
    return got


# ---- references per family on the engine's margins
def scalar_reference(oracle, name, obj, params, m, y, w):
    if obj in oracle.OBJECTIVES and name in oracle.METRICS:
        want = oracle_metric(oracle, obj, name, 1, m, y, w)
    elif name == "error":
        want = MT.metric(name, obj, m.reshape(-1, 1), y.reshape(-1, 1), w)
    else:
        want = O.metric(name, obj, m, y, w, params)
    return want, B.elementwise_terms(name, obj, m, y, params)


def run_scalar(eng, oracle, obj, name, m, y, w=None, params=None, exact=False, big=False):
    params = params or {}
    bst = null_model(eng, dict(params, objective=obj))
    d, got_m = matrix(eng, bst, m, label=y, weight=w)
    if big:   # the oracle adds 10^7 doubles one after the other; the NumPy reference sums pairwise
        want, S = O.metric(name, obj, got_m, y, w, params), B.elementwise_terms(name, obj, got_m, y, params)
    else:
        want, S = scalar_reference(oracle, name, obj, params, got_m, y, w)
    return check(eng, bst, d, name, want, S, w, exact)


def run_softprob(eng, oracle, name, m, y, w=None, exact=False):
    K = m.shape[1]
    bst = null_model(eng, SOFTPROB, K, "softprob")
    d, got_m = matrix(eng, bst, m, label=y, weight=w)
    want = oracle_metric(oracle, "multi:softprob", name, K, got_m, y, w)
    # mlogloss adds one term per row, -log p_y; merror one 0/1
    r = got_m.astype(np.float64)
    p = np.exp(r - r.max(axis=1, keepdims=True))
    p = p[np.arange(len(y)), y.astype(int)] / p.sum(axis=1)
    S = -np.log(np.maximum(p, 1e-16)) if name == "mlogloss" else np.ones(len(y))
    return check(eng, bst, d, name, want, S, w, exact)


def run_aft(eng, name, dist, m, lo, up, w=None, exact=False):
    params = {"objective": "survival:aft", "aft_loss_distribution": dist}
    bst = null_model(eng, params, 1, "aft")
    d, got_m = matrix(eng, bst, m, weight=w, lower=lo, upper=up)
    want = SR.metric(name, params, got_m, lo, up, w)
    S = B.aft_terms(params, got_m, lo, up) if name == "aft-nloglik" else np.ones(len(m))
    return check(eng, bst, d, name, want, S, w, exact)


def run_quantile(eng, alphas, m, y, w=None):
    bst = null_model(eng, {"objective": "reg:quantileerror", "quantile_alpha": [float(a) for a in alphas]}, len(alphas),
                     "quantile")
    d, got_m = matrix(eng, bst, m, label=y, weight=w)
    got_m = got_m.reshape(len(y), -1)
    a = np.asarray(alphas, F32).astype(np.float64)
    u = y.astype(np.float64)[:, None] - got_m
    S = np.abs(np.where(u >= 0, a * u, (a - 1.0) * u)).reshape(-1)
    want = Q.pinball(got_m, y, w, alphas)
    return check(eng, bst, d, "quantile", want, S, None if w is None else np.repeat(w, len(alphas)))


def run_multi_target(eng, obj, name, m, y, w=None, exact=False):
    T = y.shape[1]
    bst = null_model(eng, {"objective": obj}, T, "multi_target")
    d, got_m = matrix(eng, bst, m, label=y, weight=w, multi_target=True)
    got_m = got_m.reshape(y.shape)
    want = MT.metric(name, obj, got_m, y, w)
    S = B.elementwise_terms(name, obj, got_m.reshape(-1), y.reshape(-1))
    return check(eng, bst, d, name, want, S, None if w is None else np.repeat(w, T), exact)


def benign(kind, n, seed):
    """(margin, label or bounds) of n rows for one kernel family."""
    rng = np.random.default_rng(seed)
    if kind == "softprob":
        return rng.normal(size=(n, 3)).astype(F32), rng.integers(0, 3, n).astype(F32)
    if kind == "aft":
        lo = rng.uniform(0.5, 2, n).astype(F32)
        up = np.where(rng.uniform(size=n) < 0.5, lo, lo * F32(3)).astype(F32)
        return rng.normal(0, 0.5, n).astype(F32), (lo, up)
    if kind == "quantile":
        return rng.normal(size=(n, 3)).astype(F32), rng.normal(size=n).astype(F32)
    if kind == "multi_target":
        return rng.normal(size=(n, 2)).astype(F32), rng.uniform(0, 1, (n, 2)).astype(F32)
    return rng.normal(size=n).astype(F32), rng.normal(size=n).astype(F32)


ALPHAS3 = [0.1, 0.5, 0.9]


def run_family(eng, oracle, kind, m, y, w=None, big=False):
    if kind == "rmse":
        return run_scalar(eng, oracle, "reg:squarederror", "rmse", m, y, w, big=big)
    if kind == "mae":
        return run_scalar(eng, oracle, "reg:squarederror", "mae", m, y, w, big=big)
    if kind == "softprob":
        return run_softprob(eng, oracle, "mlogloss", m, y, w)
    if kind == "aft":
        return run_aft(eng, "aft-nloglik", "normal", m, y[0], y[1], w)
    if kind == "quantile":
        return run_quantile(eng, ALPHAS3[:m.shape[1]], m, y, w)
    return run_multi_target(eng, "reg:squarederror", "mae", m, y, w)


def data_kind(kind):
    return kind if kind in ("softprob", "aft", "quantile", "multi_target") else "scalar"


KINDS = ["rmse", "softprob", "aft", "quantile", "multi_target"]
COUNTS = ["1", "31", "32", "33", "255", "256", "257", "C-1", "C", "C+1", "2C+17"]


def rows(spec, C_rows):
    return {"C-1": C_rows - 1, "C": C_rows, "C+1": C_rows + 1, "2C+17": 2 * C_rows + 17}.get(spec) or int(spec)


@pytest.mark.parametrize("count", COUNTS)
@pytest.mark.parametrize("kind", KINDS)
def test_row_counts(eng, oracle, C_rows, kind, count):
    n = rows(count, C_rows)
    m, y = benign(data_kind(kind), n, seed=n)
    run_family(eng, oracle, kind, m, y)


@pytest.mark.parametrize("kind", ["mae", "aft", "quantile1", "multi_target"])
def test_ten_million_rows(eng, oracle, kind):
    n = 10_000_000
    if kind == "quantile1":
        rng = np.random.default_rng(1)
        run_quantile(eng, [0.3], rng.normal(size=(n, 1)).astype(F32), rng.normal(size=n).astype(F32))
    elif kind == "multi_target":   # n * T = 10^7 elements
        m, y = benign("multi_target", n // 2, seed=2)
        run_family(eng, oracle, kind, m, y)
    else:
        m, y = benign(data_kind(kind), n, seed=3)
        run_family(eng, oracle, kind, m, y, big=True)


def test_empty_matrix_is_zero(eng):
    bst = null_model(eng, {"objective": "reg:squarederror"})
    d = eng.DMatrix(np.zeros((0, 1), F32), label=np.zeros(0, F32))
    assert evaluate(eng, bst, d, "rmse") == 0.0


@pytest.mark.parametrize("where", ["0", "n-1", "C-1", "C"])
@pytest.mark.parametrize("kind", ["mae", "softprob", "aft", "quantile", "multi_target"])
def test_planted_row(eng, oracle, C_rows, kind, where):
    """One row whose loss stands far above the others (10^6 times for the absolute losses; mlogloss and aft-nloglik
    clamp it at about 30 times), at the first and last row and at the grid-stride seams: a kernel that dropped or
    double-counted it would miss the bound by far."""
    n = 1_000_000
    j = {"0": 0, "n-1": n - 1, "C-1": C_rows - 1, "C": C_rows}[where]
    m, y = benign(data_kind(kind), n, seed=j)
    if kind == "softprob":
        m[j] = 0
        m[j, int(y[j])] = -1e6                  # p_y underflows: -log(1e-16)
    elif kind == "aft":
        lo, up = y
        lo[j] = up[j] = 1
        m[j] = 2000                             # the density underflows: -log(1e-12)
    else:
        m[j] = y[j] + F32(1e6)
    run_family(eng, oracle, kind, m, y)


WEIGHTS = ["uniform", "wide", "some_zero"]


def make_weight(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return rng.uniform(0.5, 2.0, n).astype(F32)
    if kind == "wide":
        return (10.0 ** rng.uniform(-30, 30, n)).astype(F32)
    w = rng.uniform(0.5, 2.0, n).astype(F32)
    w[rng.uniform(size=n) < 0.3] = 0
    return w


@pytest.mark.parametrize("wkind", WEIGHTS)
@pytest.mark.parametrize("kind", ["rmse", "mae", "softprob", "aft", "quantile", "multi_target"])
def test_weights(eng, oracle, C_rows, kind, wkind):
    n = C_rows + 1001
    m, y = benign(data_kind(kind), n, seed=5)
    run_family(eng, oracle, kind, m, y, make_weight(wkind, n, 6))


def test_all_zero_weights_give_zero(eng):
    n = 1000
    m, y = benign("scalar", n, 7)
    bst = null_model(eng, {"objective": "reg:squarederror"})
    d, _ = matrix(eng, bst, m, label=y, weight=np.zeros(n, F32))
    for name in ("rmse", "mae", "mape", "mphe"):
        assert evaluate(eng, bst, d, name) == 0.0


def test_zero_weight_on_an_infinite_loss_is_nan(eng, oracle):
    """mape of a row with y = 0 is infinite; its weight 0 gives inf * 0 = NaN, in the engine as in the reference."""
    m, y = benign("scalar", 300, 8)
    y[17] = 0
    w = np.ones(300, F32)
    w[17] = 0
    got = run_scalar(eng, oracle, "reg:squarederror", "mape", m, y, w)
    assert np.isnan(got)


@pytest.mark.parametrize("case", B.domain_cases(), ids=lambda c: c[0])
def test_domain_edges(eng, oracle, case):
    _, obj, params, name, m, y = case
    w = np.random.default_rng(len(y)).uniform(0.5, 2.0, len(y)).astype(F32)
    run_scalar(eng, oracle, obj, name, m, y, None, params, exact=name == "error")
    run_scalar(eng, oracle, obj, name, m, y, w, params)


@pytest.mark.parametrize("case", B.class_cases(), ids=lambda c: c[0])
def test_class_edges(eng, oracle, case):
    _, K, m, y = case
    run_softprob(eng, oracle, "mlogloss", m, y)
    run_softprob(eng, oracle, "merror", m, y, exact=True)
    w = np.random.default_rng(K).uniform(0.5, 2, len(y)).astype(F32)
    run_softprob(eng, oracle, "merror", m, y, w)


@pytest.mark.parametrize("dist", ["normal", "logistic", "extreme"])
def test_survival_edges(eng, dist):
    from tests.test_metric_reference import survival_cases
    m, lo, up = survival_cases()
    run_aft(eng, "aft-nloglik", dist, m, lo, up)
    run_aft(eng, "interval-regression-accuracy", dist, m, lo, up, exact=True)
    # exp(0) = 1 on a bound: counted as inside
    z = np.zeros(3, F32)
    assert run_aft(eng, "interval-regression-accuracy", dist, z, lo[:3], up[:3], exact=True) == 1.0


@pytest.mark.parametrize("K", [1, 3, 9])
def test_quantile_alphas(eng, K):
    rng = np.random.default_rng(K)
    n = 5000
    alphas = np.sort(rng.uniform(0.01, 0.99, K)).astype(F32)
    y = rng.normal(size=n).astype(F32)
    m = rng.normal(size=(n, K)).astype(F32)
    m[:100] = y[:100, None]                     # u = 0 exactly
    run_quantile(eng, [float(a) for a in alphas], m, y)
    run_quantile(eng, [float(a) for a in alphas], m, y, rng.uniform(0.5, 2, n).astype(F32))


@pytest.mark.parametrize("T", [2, 17, 64])
@pytest.mark.parametrize("obj,name", [("reg:squarederror", "rmse"), ("reg:squarederror", "mae"),
                                      ("reg:logistic", "logloss"), ("reg:logistic", "error")])
def test_multi_target(eng, C_rows, T, obj, name):
    n = C_rows // T + 37                        # n * T crosses the grid-stride seam
    rng = np.random.default_rng(T)
    m = rng.normal(size=(n, T)).astype(F32)
    y = rng.uniform(0, 1, (n, T)).astype(F32)
    run_multi_target(eng, obj, name, m, y, exact=name == "error")
    run_multi_target(eng, obj, name, m, y, rng.uniform(0.5, 2, n).astype(F32))


# ---- the same bits on every call
REPRO = ["rmse", "mae", "logloss", "mphe", "mlogloss", "aft-nloglik", "quantile", "multi_target_rmse", "auc", "aucpr",
         "ndcg", "map"]


@pytest.mark.parametrize("name", REPRO)
def test_same_bits_on_every_call(eng, C_rows, name):
    n = 2 * C_rows + 17
    rng = np.random.default_rng(9)
    m = rng.normal(size=n).astype(F32)
    y = rng.uniform(0, 1, n).astype(F32)
    if name in ("rmse", "mae", "mphe"):
        bst = null_model(eng, {"objective": "reg:pseudohubererror" if name == "mphe" else "reg:squarederror"})
        d, _ = matrix(eng, bst, m, label=y)
    elif name in ("logloss", "auc", "aucpr"):
        bst = null_model(eng, {"objective": "binary:logistic"})
        d, _ = matrix(eng, bst, m, label=(y > 0.5).astype(F32))
    elif name == "mlogloss":
        mm, yy = benign("softprob", n, 10)
        bst = null_model(eng, SOFTPROB, 3, "softprob")
        d, _ = matrix(eng, bst, mm, label=yy)
    elif name == "aft-nloglik":
        mm, (lo, up) = benign("aft", n, 11)
        bst = null_model(eng, {"objective": "survival:aft"}, 1, "aft")
        d, _ = matrix(eng, bst, mm, lower=lo, upper=up)
    elif name == "quantile":
        mm, yy = benign("quantile", n, 12)
        bst = null_model(eng, {"objective": "reg:quantileerror", "quantile_alpha": ALPHAS3}, 3, "quantile")
        d, _ = matrix(eng, bst, mm, label=yy)
    elif name == "multi_target_rmse":
        mm, yy = benign("multi_target", n, 13)
        bst = null_model(eng, {"objective": "reg:squarederror"}, 2, "multi_target")
        d, _ = matrix(eng, bst, mm, label=yy, multi_target=True)
        name = "rmse"
    else:
        X = rng.uniform(size=(20000, 4)).astype(F32)
        qid = np.repeat(np.arange(2000), 10)
        yr = rng.integers(0, 4, 20000).astype(F32)
        bst = eng.train({"objective": "rank:ndcg", "max_depth": 4}, eng.DMatrix(X, label=yr, qid=qid), 4,
                        verbose_eval=False)
        d = eng.DMatrix(X, label=yr, qid=qid)
    vals = [evaluate(eng, bst, d, name) for _ in range(5)]
    assert len({v.hex() for v in vals}) == 1, vals


def test_csr_matrix_gives_the_bits_of_its_dense_twin(eng):
    import scipy.sparse as sp
    rng = np.random.default_rng(14)
    n, f = 200_000, 6
    X = rng.uniform(1, 2, (n, f)).astype(F32)
    X[rng.uniform(size=X.shape) < 0.3] = np.nan
    y = (np.nan_to_num(X[:, 0]) + np.nan_to_num(X[:, 1]) + rng.normal(0, 0.1, n) > 1.5).astype(F32)
    bst = eng.train({"objective": "binary:logistic", "max_depth": 5}, eng.DMatrix(X, label=y), 5, verbose_eval=False)
    dense = eng.DMatrix(X, label=y)
    csr = eng.DMatrix(sp.csr_matrix(np.nan_to_num(X, nan=0.0)), label=y)
    for name in ("logloss", "rmse", "error", "auc"):
        assert evaluate(eng, bst, dense, name).hex() == evaluate(eng, bst, csr, name).hex(), name


@pytest.mark.timeout(600)
def test_two_gpus_evaluate_like_one():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    rng = np.random.default_rng(15)
    n = 300_001
    X = rng.uniform(size=(n, 4)).astype(F32)
    y = (X[:, 0] + rng.normal(0, 0.3, n)).astype(F32)
    params = {"objective": "reg:squarederror", "max_depth": 4, "eval_metric": ["rmse", "mae", "mphe"]}
    res = []
    for actors in (1, 2):
        r = {}
        dv = RayDMatrix(X, y)
        train(params, RayDMatrix(X, y), num_boost_round=3, evals=[(dv, "v")], evals_result=r,
              ray_params=RayParams(num_actors=actors))
        res.append(r)
    for name in params["eval_metric"]:
        # the public evals_result carries six decimals: the shard order may move the sum's last bits across a
        # rounding boundary of the printed value, no further
        assert np.allclose(res[0]["v"][name], res[1]["v"][name], rtol=0, atol=1.01e-6), name


# ---- the cached evaluation margins follow every edit of the model
def data(n=20000, seed=16, f=5):
    rng = np.random.default_rng(seed)
    X = rng.uniform(size=(n, f)).astype(F32)
    y = (X[:, 0] * 2 + X[:, 1] + rng.normal(0, 0.2, n)).astype(F32)
    return X, y


def assert_metric_fresh(eng, bst, d, y, names=("rmse", "mae")):
    m = bst.predict(d, output_margin=True)
    for name in names:
        want = O.metric(name, "reg:squarederror", m, y)
        B.assert_within(evaluate(eng, bst, d, name), want, B.elementwise_terms(name, "reg:squarederror", m, y), None,
                        name)


def test_cache_follows_base_margin(eng):
    X, y = data()
    bst = eng.train({"max_depth": 4}, eng.DMatrix(X, label=y), 4, verbose_eval=False)
    dv = eng.DMatrix(X[:5000], label=y[:5000])
    assert_metric_fresh(eng, bst, dv, y[:5000])
    dv.set_info(base_margin=np.full(5000, 3.0, F32))
    assert_metric_fresh(eng, bst, dv, y[:5000])
    dv.set_info(base_margin=np.full(5000, -1.0, F32))
    assert_metric_fresh(eng, bst, dv, y[:5000])


def test_cache_follows_dart_weights(eng):
    X, y = data()
    dv = eng.DMatrix(X[:5000], label=y[:5000])
    bst = eng.train({"booster": "dart", "rate_drop": 0.5, "max_depth": 4, "seed": 3}, eng.DMatrix(X, label=y), 6,
                    evals=[(dv, "v")], verbose_eval=False)
    assert_metric_fresh(eng, bst, dv, y[:5000])
    w = np.linspace(0.2, 1.5, bst.num_trees()).astype(F32)
    eng._check(eng.lib().B2_BoosterSetTreeWeights(bst.handle, eng._fp(w), w.size))
    assert_metric_fresh(eng, bst, dv, y[:5000])


def test_cache_follows_set_param_eta(eng):
    X, y = data()
    dv = eng.DMatrix(X[:5000], label=y[:5000])
    sched = eng.LearningRateScheduler([0.3, 0.05, 0.9, 0.5])
    bst = eng.train({"max_depth": 4}, eng.DMatrix(X, label=y), 4, evals=[(dv, "v")], callbacks=[sched],
                    verbose_eval=False)
    assert_metric_fresh(eng, bst, dv, y[:5000])


def test_cache_follows_refresh_and_continuation(eng):
    X, y = data()
    dv = eng.DMatrix(X[:5000], label=y[:5000])
    base = eng.train({"max_depth": 4, "base_score": 0.5}, eng.DMatrix(X, label=y), 4, verbose_eval=False)
    y2 = (y * 0.5 + 1).astype(F32)
    upd = eng.train({"max_depth": 4, "base_score": 0.5, "process_type": "update", "updater": "refresh"},
                    eng.DMatrix(X, label=y2), 4, evals=[(dv, "v")], xgb_model=base, verbose_eval=False)
    assert_metric_fresh(eng, upd, dv, y[:5000])
    cont = eng.train({"max_depth": 4, "base_score": 0.5}, eng.DMatrix(X, label=y2), 3, evals=[(dv, "v")],
                     xgb_model=base, verbose_eval=False)
    assert_metric_fresh(eng, cont, dv, y[:5000])


def test_cache_follows_twenty_more_rounds(eng):
    X, y = data()
    dtrain = eng.DMatrix(X, label=y)
    dv = eng.DMatrix(X[:5000], label=y[:5000])
    bst = eng.train({"max_depth": 4}, dtrain, 3, verbose_eval=False)
    assert_metric_fresh(eng, bst, dv, y[:5000])
    for i in range(20):
        bst.update(dtrain, 3 + i)
    assert_metric_fresh(eng, bst, dv, y[:5000])
