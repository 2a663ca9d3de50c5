"""CPU checks of tests/objective_reference.py, the reference for the Poisson, Tweedie, gamma, pseudo-Huber, squared-log
and logistic-variant objectives (DESIGN.md 4.4): the binary32 exp / log1p sequences, gradients against a float64
restatement, intercepts, metrics, label domains, depth-1 known answers, and the golden fixtures of these objectives."""
import json
import os

import numpy as np
import pytest
from scipy.special import gammaln

from tests import objective_reference as R
from tests.golden.make_golden_objectives import CASES, run_case

GOLD = os.path.join(os.path.dirname(__file__), "golden")
F = np.float32


def labels_for(obj, n, rng):
    if obj in ("reg:logistic", "binary:logitraw"):
        y = rng.uniform(0, 1, n)
        y[::3] = 1.0
        y[1::5] = 0.0
    elif obj == "reg:squaredlogerror":
        y = rng.uniform(-0.5, 5, n)
        y[::4] = 1.0
    elif obj == "reg:pseudohubererror":
        y = rng.normal(0, 3, n)
    elif obj == "reg:gamma":
        y = rng.gamma(2.0, 1.0, n) + 1e-3
    else:
        y = rng.poisson(2.0, n).astype(np.float64)
    return y.astype(F)


def float64_gradients(obj, p, y, w, params):
    """The objective table in float64: (g, h, scale of g, scale of h) times the weight; the scales are the magnitudes
    of the added terms, so a tolerance relative to them allows for cancellation and for the rounding of exp's argument."""
    p, y = p.astype(np.float64), y.astype(np.float64)
    if obj in R.REG_LOSS:
        w = np.where(y == 1.0, w * float(params.get("scale_pos_weight", 1.0)), w)
    if obj in ("reg:logistic", "binary:logitraw"):
        s = 1.0 / (1.0 + np.exp(-p))
        g, h, gs, hs = s - y, np.maximum(s * (1 - s), 1e-16), s + np.abs(y), s
    elif obj == "reg:squaredlogerror":
        q = np.maximum(p, float(F(-1.0) + F(1e-6)))
        lq, ly = np.log1p(q), np.log1p(y)
        g, gs = (lq - ly) / (q + 1), (np.abs(lq) + np.abs(ly)) / (q + 1)
        h = np.maximum((-lq + ly + 1) / (q + 1) ** 2, 1e-6)
        hs = (np.abs(lq) + np.abs(ly) + 1) / (q + 1) ** 2
    elif obj == "reg:pseudohubererror":
        d = float(F(params.get("huber_slope", 1.0)))
        s = 1 + ((p - y) / d) ** 2
        g, h = (p - y) / np.sqrt(s), 1 / (s * np.sqrt(s))
        gs, hs = np.abs(g), h
    elif obj == "count:poisson":
        mds = float(F(R.max_delta_step(params)))
        g, h = np.exp(p) - y, np.exp(p + mds)
        gs, hs = np.exp(p) + y, h * (1 + np.abs(p + mds))
    elif obj == "reg:gamma":
        r = y / np.exp(p)
        g, h, gs, hs = 1 - r, r, 1 + r, r * (1 + np.abs(p))
    else:
        rho = float(F(params.get("tweedie_variance_power", 1.5)))
        e1, e2 = np.exp((1 - rho) * p), np.exp((2 - rho) * p)
        g, h = -y * e1 + e2, -y * (1 - rho) * e1 + (2 - rho) * e2
        gs = (y * e1 + e2) * (1 + np.abs(p))
        hs = (y * abs(1 - rho) * e1 + (2 - rho) * e2) * (1 + np.abs(p))
    return g * w, h * w, gs * w, hs * w


def test_expf_is_the_oracles_sequence(oracle):
    rng = np.random.RandomState(0)
    x = np.concatenate([rng.uniform(-110, 95, 20000), rng.uniform(-3, 3, 20000),
                        [-103.0, -103.0001, 88.7, 88.8, 0.0, -0.0, 1e-30]]).astype(F)
    want = np.array([oracle.lib().or_expf(float(v)) for v in x], F)
    assert np.array_equal(R.expf_(x).view(np.uint32), want.view(np.uint32))


def test_log1pf_within_2ulp():
    rng = np.random.RandomState(0)
    tiny = np.finfo(F).tiny
    xs = np.concatenate([
        F(-1) + F(1e-6) * np.arange(1, 50, dtype=F),
        -np.logspace(-45, np.log10(0.999999), 3000),
        np.logspace(-45, 30, 6000),
        rng.uniform(-0.99999, 3, 3000),
        [tiny, -tiny, tiny / 2, -tiny / 2, 1e-45, -1e-45, 0.0, 1e30, np.sqrt(2) - 1, np.sqrt(0.5) - 1, 1.0, -0.5],
    ]).astype(F)
    xs = xs[xs > -1]
    ref = np.log1p(xs.astype(np.float64))
    ulp = np.maximum(np.spacing(np.abs(ref).astype(F)).astype(np.float64), 2.0 ** -149)
    err = np.abs(R.log1pf_(xs).astype(np.float64) - ref) / ulp
    assert err.max() <= 2.0, (xs[np.argmax(err)], err.max())
    sp = R.log1pf_(np.array([-1.0, -2.0, np.inf], F))
    assert sp[0] == -np.inf and np.isnan(sp[1]) and sp[2] == np.inf


@pytest.mark.parametrize("obj", R.OBJECTIVES)
@pytest.mark.parametrize("weighted", [False, True])
def test_gradients_match_float64_restatement(obj, weighted):
    rng = np.random.RandomState(10 * R.OBJECTIVES.index(obj) + weighted)
    n = 5000
    y = labels_for(obj, n, rng)
    p = rng.uniform(-3, 3, n).astype(F)
    w = rng.uniform(0.2, 3.0, n).astype(F) if weighted else None
    for extra in ({}, {"scale_pos_weight": 2.5}, {"huber_slope": 0.7}, {"tweedie_variance_power": 1.2},
                  {"max_delta_step": 0.3}):
        params = dict(extra, objective=obj)
        g, h, bad = R.gradients(params, p, y, w)
        assert bad == 0
        rg, rh, gs, hs = float64_gradients(obj, p, y, np.ones(n) if w is None else w.astype(np.float64), params)
        assert np.all(np.abs(g - rg) <= 1e-6 * gs), (obj, extra, np.max(np.abs(g - rg) / gs))
        assert np.all(np.abs(h - rh) <= 1e-6 * hs), (obj, extra, np.max(np.abs(h - rh) / hs))


def test_nonfinite_gradient_rows_are_zeroed_and_counted():
    y = np.array([1.0, 2.0, 3.0], F)
    p = np.array([0.0, -200.0, 1.0], F)       # exp(-200) underflows: y / exp(p) is infinite
    g, h, bad = R.gradients({"objective": "reg:gamma"}, p, y)
    assert bad == 1 and g[1] == 0 and h[1] == 0 and np.isfinite(g).all()


@pytest.mark.parametrize("obj", R.OBJECTIVES)
def test_intercept_known_answer(obj):
    rng = np.random.RandomState(3)
    n = 4000
    y = labels_for(obj, n, rng)
    w = rng.uniform(0.5, 2.0, n).astype(F)
    g, h, _ = R.gradients({"objective": obj}, np.zeros(n, F), y, w)
    stump = F(-np.sum(g.astype(np.float64)) / np.sum(h.astype(np.float64)))
    got = R.estimate_base_score({"objective": obj}, y, w)
    assert F(got) == R.transform(obj, np.array([stump], F))[0], obj
    if obj == "count:poisson":
        # closed form: g = w (1 - y), h = w e^0.7 at margin 0, so base_score = exp(-G/H)
        G = float(np.sum(w.astype(np.float64) * (1.0 - y)))
        H = float(np.sum(w.astype(np.float64) * R.expf_(np.array([0.7], F))[0]))
        assert F(got) == R.expf_(np.array([-G / H], F))[0]
        assert abs(R.base_margin(obj, got) - np.log(got)) <= 1e-6 * max(1.0, abs(np.log(got)))


def test_metrics_known_answers():
    rng = np.random.RandomState(11)
    y = rng.poisson(2.0, 3000).astype(F)
    m = rng.uniform(-1.5, 1.5, 3000).astype(F)
    q, yd = R.expf_(m).astype(np.float64), y.astype(np.float64)
    want = np.mean(gammaln(yd + 1.0) + q - yd * np.log(q))
    assert abs(R.metric("poisson-nloglik", "count:poisson", m, y) - want) <= 1e-9 * abs(want)
    from scipy.stats import poisson
    assert abs(want - np.mean(-poisson.logpmf(yd, q))) <= 1e-9 * abs(want)
    yg = rng.gamma(2.0, 1.0, 3000).astype(F) + F(1e-3)
    dev = R.metric("gamma-deviance", "reg:gamma", np.zeros(3000, F), yg)
    yg = yg.astype(np.float64)
    assert abs(dev - np.mean(2 * (np.log(1.000001 / (yg + 1e-6)) + (yg + 1e-6) / 1.000001 - 1))) <= 1e-9


@pytest.mark.parametrize("obj,bad_label", [("reg:logistic", 1.5), ("binary:logitraw", -0.1), ("reg:squaredlogerror", -1.0),
                                           ("count:poisson", -1.0), ("reg:tweedie", -0.5), ("reg:gamma", 0.0),
                                           ("count:poisson", np.nan)])
def test_label_domain_errors(oracle, obj, bad_label):
    rng = np.random.RandomState(1)
    X = rng.uniform(size=(200, 3)).astype(F)
    y = np.full(200, 0.5, F)
    y[17] = bad_label
    with pytest.raises(ValueError, match=obj):
        R.train(oracle, {"objective": obj}, X, y, 1)
    y[17] = 0.5
    R.train(oracle, {"objective": obj}, X, y, 1)


@pytest.mark.parametrize("obj", R.OBJECTIVES)
def test_depth1_leaves_are_newton_steps(oracle, obj):
    """max_depth=1, lambda=0, eta=1: each leaf is -G/H of its rows at the base margin (clipped by max_delta_step)."""
    rng = np.random.RandomState(21)
    n = 3000
    X = rng.uniform(0, 10, size=(n, 3)).astype(F)
    y = labels_for(obj, n, rng)
    w = rng.uniform(0.5, 2.0, n).astype(F)
    base = {"reg:logistic": 0.5, "binary:logitraw": 0.0}.get(obj, 1.0)
    params = {"objective": obj, "max_depth": 1, "lambda": 0.0, "eta": 1.0, "min_child_weight": 0.0, "base_score": base}
    model = R.train(oracle, params, X, y, 1, weight=w)
    t = model.tree(0)
    assert t.n_nodes == 3
    g, h, _ = R.gradients(params, np.full(n, R.base_margin(obj, base), F), y, w)
    go_left = X[:, t.split_feature[0]] < t.split_cond[0]
    mds = R.max_delta_step(params)
    for nid, rows in ((t.left[0], go_left), (t.right[0], ~go_left)):
        want = -np.sum(g[rows].astype(np.float64)) / np.sum(h[rows].astype(np.float64))
        if mds:
            want = float(np.clip(want, -mds, mds))
        assert abs(t.value[nid] - want) <= 1e-5 * max(1.0, abs(want)), (obj, nid, t.value[nid], want)


def test_poisson_recovers_rates(oracle):
    """count:poisson on Poisson-sampled counts: mean |log predicted rate - log true rate| below 0.1."""
    rng = np.random.RandomState(8)
    n = 20000
    X = rng.uniform(0, 2, size=(n, 3)).astype(F)
    log_rate = 0.8 * X[:, 0] - 0.5 * X[:, 1] + 0.3
    y = rng.poisson(np.exp(log_rate)).astype(F)
    model = R.train(oracle, {"objective": "count:poisson", "max_depth": 3, "eta": 0.2}, X, y, 60)
    err = np.mean(np.abs(np.log(model.predict(X)) - log_rate))
    assert err < 0.1, err


@pytest.mark.parametrize("name", CASES)
def test_reference_reproduces_objective_golden(oracle, name):
    want = json.load(open(os.path.join(GOLD, name + ".json")))
    assert run_case(name) == want
