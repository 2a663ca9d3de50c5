"""CPU checks of the survival:aft reference (tests/survival_reference.py): the fdlibm exp / log / erf replays, the
gradients against finite differences of the loss, the limits, a known answer and the golden fixtures."""
import json
import os

import numpy as np
import pytest
from scipy.special import erf as sp_erf

from tests import survival_reference as S
from tests.golden.make_golden_survival import CASES, run_case

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def ulps(a, b):
    """Distance in units in the last place (values of equal sign; NaN == NaN and inf == inf count as 0)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    same = (a == b) | (np.isnan(a) & np.isnan(b))
    ia = a.view(np.int64)
    ib = b.view(np.int64)
    ia = np.where(ia < 0, np.int64(-2 ** 63) - ia, ia)
    ib = np.where(ib < 0, np.int64(-2 ** 63) - ib, ib)
    return np.where(same, 0, np.abs(ia - ib))


def test_exp_within_one_ulp():
    rng = np.random.RandomState(0)
    x = np.concatenate([rng.uniform(-746, 710, 300000), rng.uniform(-1.1, 1.1, 100000), rng.uniform(-1e-8, 1e-8, 10000),
                        np.array([0.0, -0.0, 5e-324, -5e-324, 1e-300, 709.78, 709.782712893384, 709.79, -708.39, -708.4,
                                  -720.0, -745.13, -745.1332191019411, -745.14, np.inf, -np.inf])])
    with np.errstate(over="ignore"):
        want = np.exp(x)
    assert ulps(S.exp_(x), want).max() <= 1
    assert np.isnan(S.exp_(np.array([np.nan])))[0]


def test_log_within_one_ulp():
    rng = np.random.RandomState(1)
    y = np.concatenate([np.exp(rng.uniform(-744, 709, 300000)), rng.uniform(0.5, 2.0, 100000),
                        1.0 + rng.uniform(-1e-6, 1e-6, 10000), np.array([5e-324, 1e-310, 2.2250738585072014e-308,
                                                                        1.0, 2.0, np.finfo(np.float64).max, np.inf])])
    assert ulps(S.log_(y), np.log(y)).max() <= 1
    assert np.array_equal(S.log_(np.array([0.0, -0.0])), np.array([-np.inf, -np.inf]))
    assert np.isnan(S.log_(np.array([-1.0, -np.inf, np.nan]))).all()


def test_erf_within_one_ulp():
    """Against mpmath's correctly rounded erf; scipy's (Cephes) erf is itself up to 3 ulp off near |x| = 0.9, so it is
    compared within 4 ulp on the dense sweep."""
    mpmath = pytest.importorskip("mpmath")
    rng = np.random.RandomState(2)
    x = np.concatenate([rng.uniform(-40, 40, 300000), rng.uniform(-1.5, 1.5, 100000), rng.uniform(-7, 7, 100000),
                        np.array([0.0, -0.0, 5e-324, -5e-324, 1e-310, 1e-300, 1e-9, -1e-9, 0.84375, 1.25, 2.857142857142857,
                                  6.0, -6.0, np.inf, -np.inf])])
    got = S.erf_(x)
    assert ulps(got, sp_erf(x)).max() <= 4
    sub = np.concatenate([x[-15:], x[:4000], x[300000:304000], x[400000:402000]])
    mpmath.mp.prec = 120
    exact = np.array([float(mpmath.erf(mpmath.mpf(float(v)))) for v in sub])
    assert ulps(S.erf_(sub), exact).max() <= 1
    assert np.isnan(S.erf_(np.array([np.nan])))[0]


def rows(kind, n, rng):
    """Bounds of one censoring kind around y in [0.2, 5]."""
    y = rng.uniform(0.2, 5.0, n).astype(np.float32)
    if kind == "uncensored":
        return y, y.copy()
    if kind == "right":
        return y, np.full(n, np.inf, np.float32)
    if kind == "left":
        return np.zeros(n, np.float32), y
    return y, (y * np.float32(1.7)).astype(np.float32)


KINDS = ("uncensored", "right", "left", "interval")


def log_cdf_sf(dist, z):
    """(log F, log (1 - F), log f) of the standardised distribution, in numerically stable forms (scipy / log1p),
    independent of the reference's own sequence."""
    from scipy.special import log_ndtr
    if dist == "normal":
        return log_ndtr(z), log_ndtr(-z), -0.5 * z * z - 0.5 * np.log(2 * np.pi)
    if dist == "logistic":
        return -np.logaddexp(0.0, -z), -np.logaddexp(0.0, z), z - 2 * np.logaddexp(0.0, z)
    w = np.exp(z)
    return np.log(-np.expm1(-w)), -w, z - w


def stable_loss(dist, m, lo, up, sigma):
    lo, up = lo.astype(np.float64), up.astype(np.float64)
    with np.errstate(all="ignore"):
        z_u = (np.log(np.where(np.isinf(up), 1.0, up)) - m) / sigma
        z_l = (np.log(np.where(lo > 0, lo, 1.0)) - m) / sigma
        cu, su, _ = log_cdf_sf(dist, z_u)
        cl, sl, pl = log_cdf_sf(dist, z_l)
        unc = -(pl - np.log(sigma) - np.log(np.where(lo > 0, lo, 1.0)))
        right = -sl
        left = -cu
        # F_u - F_l from whichever tail keeps the difference exact
        inter = np.where(z_l > 0, -(sl + np.log1p(-np.exp(su - sl))), -(cu + np.log1p(-np.exp(cl - cu))))
    return np.where(lo == up, unc, np.where(np.isinf(up), right, np.where(lo == 0, left, inter)))


@pytest.mark.parametrize("dist", S.DISTRIBUTIONS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("sigma", [0.6, 1.0, 2.0])
def test_gradients_match_finite_differences(dist, kind, sigma):
    """g = dL/dm and h = d2L/dm2 against Richardson-extrapolated central differences of the loss (in a numerically
    stable form), where the gradient is unclipped and finite (|z| <= 3)."""
    rng = np.random.RandomState(3)
    lo, up = rows(kind, 400, rng)
    y = np.where(up > 0, np.where(np.isinf(up), lo, up), lo).astype(np.float64)
    m = (np.log(y) + sigma * rng.uniform(-3, 3, len(y))).astype(np.float32).astype(np.float64)
    # the reference's own loss agrees with the stable form
    ref = S.loss(dist, m, lo, up, sigma)
    stab = stable_loss(dist, m, lo, up, sigma)
    assert np.max(np.abs(ref - stab) / np.maximum(1.0, np.abs(stab))) <= 1e-9

    def d1(d):
        return (stable_loss(dist, m + d, lo, up, sigma) - stable_loss(dist, m - d, lo, up, sigma)) / (2 * d)

    def d2(d):
        return (stable_loss(dist, m + d, lo, up, sigma) - 2 * stable_loss(dist, m, lo, up, sigma)
                + stable_loss(dist, m - d, lo, up, sigma)) / (d * d)

    g, h = S.grad_hess64(dist, m.astype(np.float32), lo, up, sigma)
    fd_g = (4 * d1(5e-3) - d1(1e-2)) / 3
    fd_h = (4 * d2(5e-3) - d2(1e-2)) / 3
    keep = (np.abs(g) < 14.9) & (h > 1e-6) & (h < 14.9)
    assert keep.sum() > 100
    assert np.max(np.abs(g - fd_g)[keep] / np.maximum(np.abs(fd_g[keep]), 1e-3)) <= 1e-6
    assert np.max(np.abs(h - fd_h)[keep] / np.maximum(np.abs(fd_h[keep]), 1e-3)) <= 1e-6


def exact_grad_hess(dist, kind, y, m, sigma):
    """Clipped g, h of the exact functions at margin m (mpmath; F_u - F_l is taken from the tail it is small in, so
    it does not cancel)."""
    mp = pytest.importorskip("mpmath")
    mp.mp.prec = 200

    def dens(z):   # pdf, cdf, survival function, pdf'
        if dist == "normal":
            f = mp.npdf(z)
            return f, mp.ncdf(z), mp.ncdf(-z), -z * f
        if dist == "logistic":
            w = mp.exp(z)
            f = w / (1 + w) ** 2
            return f, w / (1 + w), 1 / (1 + w), f * (1 - w) / (1 + w)
        w = mp.exp(z)
        f = w * mp.exp(-w)
        return f, -mp.expm1(-w), mp.exp(-w), (1 - w) * f

    s = mp.mpf(sigma)
    m = mp.mpf(float(m))
    zu = (mp.log(mp.mpf(float(y)) * (mp.mpf(1.7) if kind == "interval" else 1)) - m) / s
    zl = (mp.log(mp.mpf(float(y))) - m) / s
    fu, Fu, Su, gu = dens(zu) if kind != "right" else (0, 1, 0, 0)
    fl, Fl, Sl, gl = dens(zl) if kind != "left" else (0, 0, 1, 0)
    dF = (Sl - Su) if (kind != "left" and zl > 0) else (Fu - Fl)
    df, dg = fu - fl, gu - gl
    g = df / (s * dF)
    h = (df * df - dg * dF) / (s * s * dF * dF)
    return float(min(max(g, -15), 15)), float(min(max(h, 1e-16), 15))


@pytest.mark.parametrize("dist", S.DISTRIBUTIONS)
@pytest.mark.parametrize("kind", KINDS)
def test_limits(dist, kind):
    """Where the quotient stops being finite (its denominator below kEps), g and h take their limits.
    Uncensored rows: each limit equals the clipped value at the largest |z| where the quotient is still finite.
    Censored rows: F_u - F_l cancels to 0 in binary64 before the exact quotient reaches its limit (as in xgboost's
    AFT), so there the limits are checked against the exact clipped g and h far out, where they have converged."""
    sigma = 1.0
    lo, up = rows(kind, 1, np.random.RandomState(4))
    y = float(lo[0] if lo[0] > 0 else up[0])
    seen = 0
    for direction in (+1, -1):          # +1: margin -> -inf (z > 0); -1: margin -> +inf
        zs = np.linspace(0.0, 800.0, 160001)
        m = (np.log(y) - direction * sigma * zs).astype(np.float32)
        n = len(m)
        s = S._sides(dist, m, np.repeat(lo, n), np.repeat(up, n), sigma)
        with np.errstate(all="ignore"):
            gq = np.where(s["unc"], s["fp"] / (sigma * s["f"]), s["df"] / (sigma * s["dF"]))
        gden = np.where(s["unc"], sigma * s["f"], sigma * s["dF"])
        lim = (gden < S.K_EPS) & ~np.isfinite(gq)
        if not lim.any():
            continue
        seen += 1
        g, h = S.grad_hess64(dist, m, np.repeat(lo, n), np.repeat(up, n), sigma)
        first = int(np.argmax(lim))
        assert first > 0
        if kind == "uncensored":
            want_g, want_h = g[first - 1], h[first - 1]
        else:
            far = 40.0 if dist == "extreme" else 1e4
            want_g, want_h = exact_grad_hess(dist, kind, y, np.log(y) - direction * sigma * far, sigma)
        assert abs(g[first] - want_g) <= 1e-6 * max(1.0, abs(want_g)), (direction, g[first], want_g)
        assert abs(h[first] - want_h) <= 1e-6 * max(1.0, abs(want_h)), (direction, h[first], want_h)
    assert seen >= 1


@pytest.mark.parametrize("s", [0.3, 1.0, 2.5])
def test_normal_uncensored_known_answer(s):
    """Normal, uncensored: g = (margin - log y) / s^2 and h = 1 / s^2, in binary64 before the rounding to binary32."""
    s = float(np.float32(s))
    rng = np.random.RandomState(5)
    y = rng.uniform(0.1, 10.0, 20000).astype(np.float32)
    z = np.concatenate([rng.uniform(-1, 1, 10000), rng.uniform(-5, 5, 10000)])
    m = (np.log(y.astype(np.float64)) - s * z).astype(np.float32)
    g, h = S.grad_hess64("normal", m, y, y, s)
    ly = S.log_(y.astype(np.float64))
    zz = (ly - m.astype(np.float64)) / s
    want_g = np.clip((m.astype(np.float64) - ly) / (s * s), -15, 15)
    want_h = np.full_like(want_g, 1.0 / (s * s))
    small = np.abs(zz) <= 1
    assert ulps(g[small], want_g[small]).max() <= 4
    tol = 1e-12 * (1 + zz * zz)
    assert np.all(np.abs(g - want_g)[~small] <= tol[~small] * np.abs(want_g[~small]) + 1e-300)
    assert np.all(np.abs(h - want_h) <= tol * want_h)


def test_label_checks():
    n = 4
    ok_lo = np.array([1, 1, 0, 1], np.float32)
    ok_up = np.array([1, np.inf, 2, 3], np.float32)
    S.check_bounds(ok_lo, ok_up, n)
    with pytest.raises(ValueError, match="needs label_lower_bound"):
        S.check_bounds(ok_lo, None, n)
    with pytest.raises(ValueError, match="NaN"):
        S.check_bounds(np.array([1, np.nan, 0, 1], np.float32), ok_up, n)
    with pytest.raises(ValueError, match=">= 0"):
        S.check_bounds(np.array([1, -1, 0, 1], np.float32), ok_up, n)
    with pytest.raises(ValueError, match="upper_bound must be >="):
        S.check_bounds(np.array([1, 1, 3, 1], np.float32), ok_up, n)
    with pytest.raises(ValueError, match="uncensored"):
        S.check_bounds(np.array([0, 1, 0, 1], np.float32), np.array([0, 2, 2, 3], np.float32), n)


def test_metrics_known_values():
    lo = np.array([1.0, 2.0, 0.0, 1.0], np.float32)
    up = np.array([1.0, np.inf, 3.0, 4.0], np.float32)
    m = np.zeros(4, np.float32)                  # prediction exp(0) = 1
    acc = S.metric("interval-regression-accuracy", {}, m, lo, up)
    assert acc == 0.75                           # inclusive bounds: [1, 1] and [0, 3] and [1, 4] hold 1; [2, inf) does not
    v = S.metric("aft-nloglik", {}, m, lo, up, weight=np.array([1, 0, 0, 0], np.float32))
    assert abs(v - (0.5 * np.log(2 * np.pi))) <= 1e-15    # uncensored at z = 0, y = 1, sigma = 1


@pytest.mark.parametrize("name", CASES)
def test_reference_reproduces_survival_golden(oracle, name):
    want = json.load(open(os.path.join(GOLD, name + ".json")))
    assert run_case(name) == want
