"""The float64 metric references the GPU metric tests compare against, checked at the domain edges of every metric
against an independent scalar restatement (Python's math module, math.fsum for the sums), and the tolerance those tests
use (tests/metric_bound.py), checked to reject what it exists to catch: a binary32 restatement of each metric and a
reference that drops one planted row."""
import math

import numpy as np
import pytest
from scipy import special, stats

from tests import metric_bound as B
from tests import multi_target_reference as MT
from tests import objective_reference as O
from tests import quantile_reference as Q
from tests import survival_reference as SR

F32 = np.float32


def elementwise_fsum(name, obj, params, margin, label, weight=None):
    """The elementwise metrics row by row with math, summed with math.fsum (the binary32 transform is the engine's)."""
    q = [float(v) for v in B.transform(obj, margin)]
    qf = B.transform(obj, margin)
    y = [float(v) for v in np.asarray(label, F32)]
    w = [1.0] * len(y) if weight is None else [float(v) for v in np.asarray(weight, F32)]
    a = float(F32(params.get("huber_slope", 1.0)))
    rho = float(F32(name.split("@")[1])) if "@" in name else 1.5
    vals = []
    for i, (qi, yi) in enumerate(zip(q, y)):
        if name == "rmse":
            v = (qi - yi) ** 2
        elif name == "mae":
            v = abs(qi - yi)
        elif name == "logloss":
            pa = float(max(qf[i], F32(1e-16)))
            pb = float(max(F32(1.0) - qf[i], F32(1e-16)))
            v = -(yi * math.log(pa) + (1.0 - yi) * math.log(pb))
        elif name == "error":
            v = 1.0 if (qf[i] > F32(0.5)) != (F32(yi) > F32(0.5)) else 0.0
        elif name == "rmsle":
            v = (math.log1p(yi) - math.log1p(max(qi, -1.0 + 1e-6))) ** 2
        elif name == "mape":
            v = abs((yi - qi) / yi)
        elif name == "mphe":
            z = (yi - qi) / a
            v = a * a * (math.sqrt(1.0 + z * z) - 1.0)
        elif name == "poisson-nloglik":
            qq = max(qi, 1e-16)
            v = math.lgamma(yi + 1.0) + qq - yi * math.log(qq)
        elif name == "gamma-nloglik":
            v = yi / qi + math.log(qi)
        elif name == "gamma-deviance":
            qq, yy = qi + 1e-6, yi + 1e-6
            v = 2.0 * (math.log(qq / yy) + yy / qq - 1.0)
        elif name.startswith("tweedie-nloglik"):
            v = -yi * qi ** (1.0 - rho) / (1.0 - rho) + qi ** (2.0 - rho) / (2.0 - rho)
        else:
            raise KeyError(name)
        vals.append(v * w[i])
    m = math.fsum(vals) / math.fsum(w)
    return math.sqrt(m) if name in B.SQRT_METRICS else m


def elementwise_reference(oracle, name, obj, params, margin, label, weight=None):
    """The reference the GPU tests use: the oracle for the first metrics of binary:logistic / reg:squarederror, else
    tests/objective_reference.py."""
    if obj in oracle.OBJECTIVES and name in oracle.METRICS:
        return oracle_metric(oracle, obj, name, 1, margin, label, weight)
    if name == "error":   # reg:logistic, binary:logitraw: the multi-target reference's error with one column
        return MT.metric(name, obj, np.reshape(margin, (-1, 1)), np.reshape(label, (-1, 1)), weight)
    return O.metric(name, obj, margin, label, weight, params)


def oracle_metric(oracle, obj, name, K, margin, label, weight=None):
    import ctypes as C
    m, y = np.ascontiguousarray(margin, F32), np.ascontiguousarray(label, F32)
    w = None if weight is None else np.ascontiguousarray(weight, F32)
    s, ws = C.c_double(), C.c_double()
    oracle.lib().or_metric_sums_obj(oracle.OBJECTIVES[obj], oracle.METRICS[name], K, oracle._fp(m), oracle._fp(y),
                                    oracle._fp(w), y.size, C.byref(s), C.byref(ws))
    v = s.value / ws.value if ws.value > 0 else 0.0
    return math.sqrt(v) if name == "rmse" else v


@pytest.mark.parametrize("case", B.domain_cases(), ids=lambda c: c[0])
def test_elementwise_reference_at_domain_edges(oracle, case):
    _, obj, params, name, m, y = case
    w = np.random.default_rng(len(y)).uniform(0.5, 2.0, len(y)).astype(F32)
    for weight in (None, w):
        want = elementwise_reference(oracle, name, obj, params, m, y, weight)
        assert np.isfinite(want), name
        S = B.elementwise_terms(name, obj, m, y, params)
        B.assert_within(elementwise_fsum(name, obj, params, m, y, weight), want, S, weight, name)


def test_planted_edges_are_reached():
    """The cases reach the clamps they are there for: the sigmoid saturates to both logloss clamps, rmsle's prediction
    clamp, exp(margin) under- and overflow of the log link's binary32 exp, a margin of exactly 0."""
    cases = {c[0]: c for c in B.domain_cases()}
    p = B.transform("binary:logistic", cases["binary_logloss"][4])
    assert p.min() < F32(1e-16) and (F32(1.0) - p).min() < F32(1e-16) and np.any(p == F32(0.5))
    assert np.any(cases["rmsle"][4] < F32(-1.0 + 1e-6))
    q = B.transform("count:poisson", cases["poisson"][4])
    assert np.any(q == 0) and q.max() > F32(1e38)


@pytest.mark.parametrize("case", B.class_cases(), ids=lambda c: c[0])
def test_class_reference_at_edges(oracle, case):
    _, K, m, y = case
    p = special.softmax(m.astype(np.float64), axis=1)
    for name in ("mlogloss", "merror"):
        want = oracle_metric(oracle, "multi:softprob", name, K, m, y)
        if name == "merror":
            v = [float(np.argmax(r) != int(c)) for r, c in zip(m, y)]      # argmax takes the first maximum
            assert want == math.fsum(v) / len(v)
        else:
            v = [-math.log(max(p[i, int(c)], 1e-16)) for i, c in enumerate(y)]
            # the oracle's softmax is binary32: compare against float64 at binary32 accuracy here, not the GPU bound
            assert abs(want - math.fsum(v) / len(v)) <= 1e-6 * max(1.0, abs(want))


def test_multi_target_reference_counts_every_element_with_its_row_weight():
    rng = np.random.default_rng(3)
    n, T = 50, 4
    m = rng.normal(size=(n, T)).astype(F32)
    y = rng.uniform(0, 1, (n, T)).astype(F32)
    w = rng.uniform(0.5, 2, n).astype(F32)
    for name in ("rmse", "mae", "logloss", "error", "rmsle", "mape", "mphe"):
        want = MT.metric(name, "reg:logistic", m, y, w)
        got = elementwise_fsum(name, "reg:logistic", {}, m.reshape(-1), y.reshape(-1), np.repeat(w, T))
        S = B.elementwise_terms(name, "reg:logistic", m.reshape(-1), y.reshape(-1))
        B.assert_within(got, want, S, np.repeat(w, T), name)


def aft_scipy(dist, sigma, margin, lower, upper):
    """aft-nloglik per row from scipy's distributions."""
    pdf, cdf = {"normal": (stats.norm.pdf, stats.norm.cdf), "logistic": (stats.logistic.pdf, stats.logistic.cdf),
                "extreme": (lambda z: np.exp(z - np.exp(z)), lambda z: -np.expm1(-np.exp(z)))}[dist]
    m = np.asarray(margin, F32).astype(np.float64)
    lo, up = np.asarray(lower, F32).astype(np.float64), np.asarray(upper, F32).astype(np.float64)
    out = []
    for mi, l, u in zip(m, lo, up):
        if l == u:
            z = (math.log(l) - mi) / sigma
            out.append(-math.log(max(pdf(z) / (sigma * l), SR.K_EPS)))
        else:
            fu = 1.0 if math.isinf(u) else cdf((math.log(u) - mi) / sigma)
            fl = 0.0 if l <= 0 else cdf((math.log(l) - mi) / sigma)
            out.append(-math.log(max(fu - fl, SR.K_EPS)))
    return np.array(out)


def survival_cases():
    lower = np.array([1, 1, 0.5, 1, 0, 0, 2, 1e-3, 1e3], F32)
    upper = np.array([1, 2, 1, np.inf, 1, np.inf, 8, 1e-3, 1e4], F32)
    margins = np.array([0, -1, 0.5, 3, -3], F32)
    m = np.repeat(margins, lower.size)
    return m, np.tile(lower, margins.size), np.tile(upper, margins.size)


@pytest.mark.parametrize("dist", ["normal", "logistic", "extreme"])
def test_survival_reference_at_edges(dist):
    m, lo, up = survival_cases()
    params = {"aft_loss_distribution": dist, "aft_loss_distribution_scale": 1.3}
    v = aft_scipy(dist, SR.sigma_of(params), m, lo, up)
    want = SR.metric("aft-nloglik", params, m, lo, up)
    B.assert_within(math.fsum(v) / len(v), want, B.aft_terms(params, m, lo, up), None, "aft-nloglik")
    # exp(0) = 1 sits on a bound of the rows [1, 1], [1, 2], [0.5, 1]: bounds are included
    acc = SR.metric("interval-regression-accuracy", params, m, lo, up)
    p = np.exp(m.astype(np.float64))
    assert acc == math.fsum(((lo <= p) & (p <= up)).astype(float)) / len(m)
    assert SR.metric("interval-regression-accuracy", params, np.zeros(3, F32), lo[:3], up[:3]) == 1.0


@pytest.mark.parametrize("K", [1, 3, 9])
def test_pinball_reference(K):
    from fractions import Fraction
    rng = np.random.default_rng(K)
    n = 40
    alphas = np.sort(rng.uniform(0.01, 0.99, K)).astype(F32)
    y = rng.normal(size=n).astype(F32)
    m = rng.normal(size=(n, K)).astype(F32)
    m[:5] = y[:5, None]                                           # u = 0 exactly
    w = rng.uniform(0.5, 2, n).astype(F32)
    want = Q.pinball(m, y, w, alphas)
    num = sum(Fraction(float(w[i])) * sum((Fraction(float(a)) - (1 if u < 0 else 0)) * u
                                          for a, u in zip(alphas, (Fraction(float(y[i])) - Fraction(float(v))
                                                                   for v in m[i])))
              for i in range(n))
    exact = num / (sum(Fraction(float(x)) for x in w) * K)
    assert abs(want - float(exact)) <= 2.0 ** -50 * abs(float(exact))


# ---- the bound rejects what it is there to catch
def _benign(name, obj, n, rng):
    if obj in ("reg:logistic", "binary:logistic"):
        return rng.normal(size=n).astype(F32), rng.uniform(0, 1, n).astype(F32).round(2)
    if obj in ("count:poisson", "reg:gamma", "reg:tweedie"):
        return rng.normal(0, 1, n).astype(F32), rng.uniform(0.1, 5, n).astype(F32)
    return rng.normal(size=n).astype(F32), rng.normal(size=n).astype(F32)


def elementwise_binary32(name, obj, params, margin, label):
    """Every operation of an element's loss in binary32 (the sum stays float64)."""
    q, y = B.transform(obj, margin), np.asarray(label, F32)
    one = F32(1.0)
    with np.errstate(all="ignore"):
        if name == "rmse":
            v = (q - y) * (q - y)
        elif name == "mae":
            v = np.abs(q - y)
        elif name == "logloss":
            a, b = np.maximum(q, F32(1e-16)), np.maximum(one - q, F32(1e-16))
            v = -(y * np.log(a) + (one - y) * np.log(b))
        elif name == "rmsle":
            v = (np.log1p(y) - np.log1p(np.maximum(q, F32(-1 + 1e-6)))) ** 2
        elif name == "mape":
            v = np.abs((y - q) / y)
        elif name == "mphe":
            a = F32(params.get("huber_slope", 1.0))
            z = (y - q) / a
            v = a * a * (np.sqrt(one + z * z) - one)
        elif name == "poisson-nloglik":
            v = special.gammaln(y + one).astype(F32) + q - y * np.log(np.maximum(q, F32(1e-16)))
        elif name == "gamma-nloglik":
            v = y / q + np.log(q)
        elif name == "gamma-deviance":
            qq, yy = q + F32(1e-6), y + F32(1e-6)
            v = F32(2) * (np.log(qq / yy) + yy / qq - one)
        else:
            r = F32(name.split("@")[1]) if "@" in name else F32(1.5)
            v = -y * q ** (one - r) / (one - r) + q ** (F32(2) - r) / (F32(2) - r)
    return float(np.mean(v.astype(F32).astype(np.float64)))


ROUNDED = [("rmse", "reg:squarederror", {}), ("mae", "reg:logistic", {}), ("logloss", "reg:logistic", {}),
           ("rmsle", "reg:squaredlogerror", {}), ("mape", "reg:squarederror", {}),
           ("mphe", "reg:pseudohubererror", {"huber_slope": 1.0}), ("poisson-nloglik", "count:poisson", {}),
           ("gamma-nloglik", "reg:gamma", {}), ("gamma-deviance", "reg:gamma", {}),
           ("tweedie-nloglik@1.5", "reg:tweedie", {})]


@pytest.mark.parametrize("name,obj,params", ROUNDED, ids=[r[0] for r in ROUNDED])
def test_bound_rejects_binary32_losses_and_a_dropped_row(name, obj, params):
    rng = np.random.default_rng(7)
    n = 100_000
    m, y = _benign(name, obj, n, rng)
    if name == "rmsle":
        y = np.abs(y)
    want = O.metric(name, obj, m, y, None, params)
    S = B.elementwise_terms(name, obj, m, y, params)
    B.assert_within(want, want, S, None, name)
    got32 = elementwise_binary32(name, obj, params, m, y)
    if name in B.SQRT_METRICS:
        got32 = math.sqrt(got32)
    ok, err, bound = B.within(got32, want, S, None, name)
    assert not ok, (name, err, bound)
    # a planted row whose loss is far above the others, dropped from the sum
    v = S / np.maximum(np.mean(S), 1e-300)
    j = int(np.argmax(v))
    keep = np.ones(n, bool)
    keep[j] = False
    dropped = O.metric(name, obj, m[keep], y[keep], None, params)
    ok, err, bound = B.within(dropped, want, S, None, name)
    assert not ok, (name, err, bound)


def test_bound_rejects_binary32_class_survival_and_pinball():
    rng = np.random.default_rng(11)
    n, K = 50_000, 5
    m = rng.normal(size=(n, K)).astype(F32)
    y = rng.integers(0, K, n).astype(F32)
    p = special.softmax(m.astype(np.float64), axis=1)[np.arange(n), y.astype(int)]
    v = -np.log(p)
    v32 = -np.log(p.astype(F32))
    assert not B.within(float(np.mean(v32, dtype=np.float64)), float(np.mean(v)), v)[0]
    lo = rng.uniform(1, 2, n).astype(F32)
    up = np.where(rng.uniform(size=n) < 0.5, lo, lo * 2).astype(F32)
    mm = rng.normal(size=n).astype(F32)
    params = {"aft_loss_distribution": "normal"}
    va = SR.loss("normal", mm, lo, up, 1.0)
    want = SR.metric("aft-nloglik", params, mm, lo, up)
    assert not B.within(float(np.mean(va.astype(F32), dtype=np.float64)), want, np.abs(va))[0]
    alphas = np.array([0.1, 0.5, 0.9], F32)
    mq = rng.normal(size=(n, 3)).astype(F32)
    yq = rng.normal(size=n).astype(F32)
    u = yq[:, None].astype(np.float64) - mq
    terms = np.where(u >= 0, alphas * u, (alphas - 1.0) * u)
    u32 = (yq[:, None] - mq).astype(F32)
    t32 = np.where(u32 >= 0, alphas * u32, (alphas - F32(1)) * u32).astype(F32)
    want = Q.pinball(mq, yq, None, alphas)
    assert B.within(want, want, terms)[0]
    assert not B.within(float(np.mean(t32, dtype=np.float64)), want, terms)[0]
