"""The tolerance of the evaluation-metric tests (tests/test_gpu_metric_boundaries.py), checked on its own by
tests/test_metric_reference.py.

A metric is a weighted mean sum_j w_j v_j / sum_j w_j over elements j (rows; (row, output) pairs for multi-class,
multi-target and quantile models, each with its row's weight).  The engine must meet

    |got - want| <= 2^-40 * sum_j w_j S_j / sum_j w_j

where want is the float64 reference and S_j is the sum of the absolute values of the terms the reference adds for
element j (for gamma-deviance S = 2 (|log(q'/y')| + y'/q' + 1)).  Double arithmetic per element and double sums of up
to 10^7 elements in any fixed order stay far inside it; one binary32 operation in an element's loss (about 2^-24
relative) breaks it by a factor of about 2^16, and so does a dropped or double-counted row whose loss stands out.
rmse and rmsle are compared before the square root."""
import numpy as np

from tests import objective_reference as O

F32 = np.float32
REL = 2.0 ** -40
SQRT_METRICS = ("rmse", "rmsle")
ZERO_ONE = ("error", "merror", "interval-regression-accuracy")


def transform(obj, margin):
    """The binary32 prediction the metrics read (binary:logistic has reg:logistic's sigmoid)."""
    return O.transform("reg:logistic" if obj == "binary:logistic" else obj, np.asarray(margin, F32).reshape(-1))


def _q(obj, margin):
    return transform(obj, margin).astype(np.float64)


def elementwise_terms(name, obj, margin, label, params=None):
    """S_j of the elementwise metrics (rmse .. tweedie-nloglik@rho) on the transformed prediction q."""
    params = params or {}
    q, y = _q(obj, margin), np.asarray(label, F32).reshape(-1).astype(np.float64)
    with np.errstate(all="ignore"):
        if name == "rmse":
            return (q - y) ** 2
        if name == "mae":
            return np.abs(q - y)
        if name == "logloss":
            qf = transform(obj, margin)
            a = np.maximum(qf, F32(1e-16)).astype(np.float64)
            b = np.maximum(F32(1.0) - qf, F32(1e-16)).astype(np.float64)
            return np.abs(y * np.log(a)) + np.abs((1 - y) * np.log(b))
        if name == "error":
            return np.ones_like(y)
        if name == "rmsle":
            ly, lq = np.log1p(y), np.log1p(np.maximum(q, -1 + 1e-6))
            d = ly - lq
            return d * d + 2 * np.abs(d) * (np.abs(ly) + np.abs(lq))
        if name == "mape":
            return (np.abs(y) + np.abs(q)) / np.abs(y)
        if name == "mphe":
            a = float(F32(params.get("huber_slope", 1.0)))
            z = (y - q) / a
            return a * a * (np.sqrt(1 + z * z) + 1)
        if name == "poisson-nloglik":
            from scipy.special import gammaln
            qq = np.maximum(q, 1e-16)
            return np.abs(gammaln(y + 1)) + qq + np.abs(y * np.log(qq))
        if name == "gamma-nloglik":
            return np.abs(y / q) + np.abs(np.log(q))
        if name == "gamma-deviance":
            qq, yy = q + 1e-6, y + 1e-6
            return 2 * (np.abs(np.log(qq / yy)) + yy / qq + 1)
        if name.startswith("tweedie-nloglik"):
            r = float(F32(name.split("@", 1)[1])) if "@" in name else 1.5
            return np.abs(y * q ** (1 - r) / (1 - r)) + np.abs(q ** (2 - r) / (2 - r))
    raise KeyError(name)


def aft_terms(params, margin, lower, upper):
    """S_j of aft-nloglik: |v|, plus for a censored row the condition of -log(F(u) - F(l)), (F(u) + F(l)) / (F(u) - F(l)):
    the two cdf values carry a rounding of their own size, which the difference keeps."""
    from tests import survival_reference as SR
    dist, sigma = SR.dist_of(params), SR.sigma_of(params)
    m = np.asarray(margin, F32).astype(np.float64)
    lo, up = np.asarray(lower, F32).astype(np.float64), np.asarray(upper, F32).astype(np.float64)
    v = SR.loss(dist, margin, lower, upper, sigma)
    with np.errstate(all="ignore"):
        fu = np.where(np.isinf(up), 1.0, SR.density(dist, (np.log(np.where(np.isinf(up), 1.0, up)) - m) / sigma)[1])
        fl = np.where(lo > 0, SR.density(dist, (np.log(np.where(lo > 0, lo, 1.0)) - m) / sigma)[1], 0.0)
        cond = np.where(lo == up, 0.0, (fu + fl) / np.maximum(fu - fl, SR.K_EPS))
    return np.abs(v) + cond


def within(got, want, S, weight=None, name=""):
    """(ok, error, bound): got within the bound of want, NaN only where want is NaN.  S and weight are per element
    (weight None = 1); rmse / rmsle are compared squared."""
    if np.isnan(want) or np.isnan(got):
        return bool(np.isnan(want) and np.isnan(got)), float("nan"), float("nan")
    S = np.asarray(S, np.float64).reshape(-1)
    w = np.ones_like(S) if weight is None else np.asarray(weight, np.float64).reshape(-1)
    ws = float(np.sum(w))
    bound = REL * float(np.sum(w * S)) / ws if ws > 0 else 0.0
    if name in SQRT_METRICS:
        got, want = got * got, want * want
    err = abs(got - want)
    return bool(err <= bound), err, bound


def assert_within(got, want, S, weight=None, name=""):
    ok, err, bound = within(got, want, S, weight, name)
    assert ok, "%s: got %r, want %r, |error| %.3g > bound %.3g" % (name, got, want, err, bound)


# ---- domain edges shared by the CPU check of the references and the GPU tests: (id, objective, params, metric,
# margin, label).  Every margin is float32 and reaches the metric unchanged (a model whose trees add nothing).
def _grid(margins, labels):
    m, y = np.meshgrid(np.asarray(margins, F32), np.asarray(labels, F32))
    return m.reshape(-1), y.reshape(-1)


def domain_cases():
    below = float(np.nextafter(F32(-1.0), F32(0.0)))          # the float32 just above -1
    cases = []
    m, y = _grid([-100, -20, -1, 0, 1, 20, 100], [0, 1])
    for name in ("logloss", "error", "rmse", "mae"):
        cases.append(("binary_%s" % name, "binary:logistic", {}, name, m, y))
    m, y = _grid([-100, -20, -0.3, 0, 0.3, 20, 100], [0, 0.25, 0.5, 0.75, 1])
    for name in ("logloss", "error", "rmse"):
        cases.append(("reg_logistic_%s" % name, "reg:logistic", {}, name, m, y))
    m, y = _grid([-0.5, 0, 1e-8, 0.3, 1, 1.5], [0, 0.5, 1])
    cases.append(("logitraw_logloss", "binary:logitraw", {}, "logloss", m, y))
    m, y = _grid([-5, -1, below, -0.5, 0, 3, 1e6], [below, -0.5, 0, 1, 1e6])
    cases.append(("rmsle", "reg:squaredlogerror", {}, "rmsle", m, y))
    m, y = _grid([0, 1, -1e30, 1e30, 3e-30], [-1e30, -1, -1e-30, 1e-30, 1e-10, 1, 1e10, 1e30])
    cases.append(("mape", "reg:squarederror", {}, "mape", m, y))
    m, y = _grid([-1e6, -1, -1e-6, 0, 1e-6, 1, 1e6], [-1e3, 0, 1e-3, 1e3])
    for slope in (1e-3, 1.0, 1e3):
        cases.append(("mphe_%g" % slope, "reg:pseudohubererror", {"huber_slope": slope}, "mphe", m, y))
    m, y = _grid([-200, -103.5, -50, 0, 13.8155, 88, 100], [0, 1, 3, 1e6, 1e6 + 1])
    cases.append(("poisson", "count:poisson", {}, "poisson-nloglik", m, y))
    yg = np.asarray([1e-3, 1, 1e6], F32)
    lg = np.log(yg.astype(np.float64))
    m = np.concatenate([lg, lg + 1e-7, lg - 1e-7, lg - 30, lg + 3]).astype(F32)
    y = np.tile(yg, 5)
    for name in ("gamma-nloglik", "gamma-deviance"):
        cases.append((name, "reg:gamma", {}, name, m, y))
    m, y = _grid([-10, -1, 0, 2, 10], [0, 0.5, 3, 1e3])
    for rho in ("1.01", "1.5", "1.99"):
        cases.append(("tweedie_%s" % rho, "reg:tweedie", {}, "tweedie-nloglik@" + rho, m, y))
    return cases


def class_cases():
    """(id, K, margin [n, K], label) for mlogloss / merror: random rows, rows with tied maxima (argmax takes the first),
    rows whose other classes underflow (exp of -200), and rows whose label class underflows (p clamps at 1e-16)."""
    out = []
    for K in (2, 3, 17):
        rng = np.random.default_rng(K)
        n = 64
        m = rng.normal(size=(n, K)).astype(F32)
        y = rng.integers(0, K, n).astype(F32)
        m[:8] = 1.5                                   # every class tied
        m[8:16, :] = -200
        m[8:16, 0] = 0                                # classes 1.. underflow
        m[16:24, :] = 0
        m[16:24, K - 1] = 200                         # the label class 0 underflows
        y[16:24] = 0
        m[24:32, 0] = m[24:32, K - 1] = 7             # a tie of two maxima
        out.append(("K%d" % K, K, m, y))
    return out
