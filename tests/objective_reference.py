"""Reference for the objectives beyond squared error / logistic / softmax (reg:logistic, binary:logitraw,
reg:squaredlogerror, reg:pseudohubererror, count:poisson, reg:gamma, reg:tweedie): a NumPy restatement of their
gradients, intercept, transform, metrics and label domains (DESIGN.md 4.4), and a trainer that grows trees with the
CPU oracle (oracle/hist_oracle.c) from those gradients through its custom-gradient path.

TEST INFRASTRUCTURE ONLY, like the oracle.  The gradients replay the binary32 sequences of objective_kernel.cu
operation for operation: NumPy's float32 +, -, *, / and sqrt round correctly, b2_expf and b2_log1pf are restated on
float32 arrays (expf_ is checked bit for bit against the oracle's or_expf), and the host-side logf of the base margin
is libm's, the function the engine calls.  So gradients, and with them the trees, are bit-equal to the engine's.
"""
import ctypes
import ctypes.util

import numpy as np

F = np.float32
OBJECTIVES = ("reg:logistic", "binary:logitraw", "reg:squaredlogerror", "reg:pseudohubererror", "count:poisson",
              "reg:gamma", "reg:tweedie")
LOG_LINK = ("count:poisson", "reg:gamma", "reg:tweedie")
REG_LOSS = ("reg:logistic", "binary:logitraw", "reg:squaredlogerror")   # scale_pos_weight applies to these
DEFAULT_METRIC = {"reg:logistic": "rmse", "binary:logitraw": "logloss", "reg:squaredlogerror": "rmsle",
                  "reg:pseudohubererror": "mphe", "count:poisson": "poisson-nloglik", "reg:gamma": "gamma-nloglik",
                  "reg:tweedie": "tweedie-nloglik"}
LABEL_DOMAIN = {"reg:logistic": ("label must be in [0, 1]", lambda y: (y >= 0) & (y <= 1)),
                "binary:logitraw": ("label must be in [0, 1]", lambda y: (y >= 0) & (y <= 1)),
                "reg:squaredlogerror": ("label must be greater than -1", lambda y: y > -1),
                "count:poisson": ("label must be nonnegative", lambda y: y >= 0),
                "reg:tweedie": ("label must be nonnegative", lambda y: y >= 0),
                "reg:gamma": ("label must be positive", lambda y: y > 0)}

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.logf.restype = ctypes.c_float
_libm.logf.argtypes = [ctypes.c_float]


def _u32(x):
    return np.ascontiguousarray(x, F).view(np.uint32)


def _f32(u):
    return np.ascontiguousarray(u, np.uint32).view(F)


def expf_(x):
    """b2_expf / or_expf on a float32 array."""
    x = np.minimum(np.asarray(x, F), F(88.7))
    t = x * F(1.44269504088896341)
    n = np.rint(t)
    r = x - n * F(0.693359375)
    r = r - n * F(-2.12194440e-4)
    p = F(1.9875691500e-4)
    for c in (1.3981999507e-3, 8.3334519073e-3, 4.1665795894e-2, 1.6666665459e-1, 5.0000001201e-1):
        p = p * r + F(c)
    e = (p * (r * r) + r) + F(1.0)
    ni = np.where(np.isfinite(n), n, 0).astype(np.int64)
    n1 = np.sign(ni) * (np.abs(ni) // 2)        # C division truncates toward zero
    n2 = ni - n1
    e = e * _f32(((n1 + 127) << 23).astype(np.uint32))
    e = e * _f32(((n2 + 127) << 23).astype(np.uint32))
    return np.where(x < F(-103.0), F(0.0), e).astype(F)


def sigmoid_(x):
    nx = np.minimum(-np.asarray(x, F), F(88.7))
    return (F(1.0) / ((expf_(nx) + F(1.0)) + F(1e-16))).astype(F)


def log1pf_(x):
    """b2_log1pf on a float32 array (the fdlibm reduction with a correction term for the rounding of 1+x)."""
    x = np.asarray(x, F)
    ix = _u32(x)
    with np.errstate(all="ignore"):
        no_red = ((ix < 0x3ed413d0) | ((ix >> 31) == 1)) & (ix <= 0xbe95f619)
        u = F(1.0) + x
        iu = (_u32(u).astype(np.int64) + (0x3f800000 - 0x3f3504f3)) & 0xffffffff
        k = (iu >> 23).astype(np.int64) - 0x7f
        c = np.where(k >= 2, F(1.0) - (u - x), x - (u - F(1.0))).astype(F)
        c = np.where(k < 25, c / u, F(0.0)).astype(F)
        f = _f32(((iu & 0x007fffff) + 0x3f3504f3).astype(np.uint32)) - F(1.0)
        k = np.where(no_red, 0, k)
        c = np.where(no_red, F(0.0), c).astype(F)
        f = np.where(no_red, x, f).astype(F)
        s = f / (F(2.0) + f)
        z = s * s
        w = z * z
        t1 = w * (_f32(np.uint32(0x3ecccce1)) + w * _f32(np.uint32(0x3e789e26)))
        t2 = z * (_f32(np.uint32(0x3f2aaaaa)) + w * _f32(np.uint32(0x3e91e9ee)))
        R = t2 + t1
        hfsq = (F(0.5) * f) * f
        dk = k.astype(F)
        r = (dk * _f32(np.uint32(0x3717f7d1)) - hfsq) + f
        r = r + c
        r = s * (hfsq + R) + r
        r = r + dk * _f32(np.uint32(0x3f317180))
    r = np.where((ix & 0x7fffffff) < 0x33800000, x, r)
    r = np.where(x == np.inf, x, r)
    r = np.where(x > F(-1.0), r, np.where(x == F(-1.0), F(-np.inf), F(np.nan)))
    return r.astype(F)


def objective_param(params):
    """The parameter the gradient kernel of an objective takes."""
    obj = params["objective"]
    if obj == "reg:pseudohubererror":
        return F(params.get("huber_slope", 1.0))
    if obj == "count:poisson":
        return F(max_delta_step(params))
    if obj == "reg:tweedie":
        return F(params.get("tweedie_variance_power", 1.5))
    return F(0.0)


def max_delta_step(params):
    """count:poisson without a max_delta_step uses 0.7, in the hessian and as the leaf-step clamp."""
    d = params.get("max_delta_step")
    return float(d) if d is not None else (0.7 if params["objective"] == "count:poisson" else 0.0)


def gradients(params, margin, label, weight=None):
    """(g, h, number of non-finite rows) in binary32 for one scalar objective; non-finite pairs are (0, 0)."""
    obj = params["objective"]
    p, y = np.asarray(margin, F).reshape(-1), np.asarray(label, F)
    w = np.ones_like(y) if weight is None else np.asarray(weight, F)
    a = objective_param(params)
    with np.errstate(all="ignore"):
        if obj in REG_LOSS:
            w = np.where(y == F(1.0), w * F(params.get("scale_pos_weight", 1.0)), w).astype(F)
        if obj in ("reg:logistic", "binary:logitraw"):
            s = sigmoid_(p)
            g, h = s - y, np.maximum(s * (F(1.0) - s), F(1e-16))
        elif obj == "reg:squaredlogerror":
            kmin = F(-1.0) + F(1e-6)
            q = np.where(p < kmin, kmin, p).astype(F)
            lq, ly, q1 = log1pf_(q), log1pf_(y), q + F(1.0)
            g = (lq - ly) / q1
            h = ((-lq + ly) + F(1.0)) / (q1 * q1)
            h = np.where(h < F(1e-6), F(1e-6), h)
        elif obj == "reg:pseudohubererror":
            z = p - y
            zd = z / a
            s = F(1.0) + zd * zd
            sq = np.sqrt(s)
            g, h = z / sq, F(1.0) / (s * sq)
        elif obj == "count:poisson":
            g, h = expf_(p) - y, expf_(p + a)
        elif obj == "reg:gamma":
            r = y / expf_(p)
            g, h = F(1.0) - r, r
        elif obj == "reg:tweedie":
            e1, e2 = expf_((F(1.0) - a) * p), expf_((F(2.0) - a) * p)
            g = -(y * e1) + e2
            h = ((-y) * (F(1.0) - a)) * e1 + (F(2.0) - a) * e2
        else:
            raise KeyError(obj)
        g, h = (g * w).astype(F), (h * w).astype(F)
        bad = ~((np.abs(g) <= np.finfo(F).max) & (np.abs(h) <= np.finfo(F).max))
    g[bad] = 0.0
    h[bad] = 0.0
    return g, h, int(bad.sum())


def transform(obj, m):
    m = np.asarray(m, F)
    if obj == "reg:logistic":
        return sigmoid_(m)
    if obj in LOG_LINK:
        return expf_(m)
    return m


def check_labels(obj, y):
    msg, ok = LABEL_DOMAIN.get(obj, (None, None))
    if ok is not None and not np.all(ok(np.asarray(y, F))):
        raise ValueError("%s for %s" % (msg, obj))


def _quant_exponent(vmax):
    bits = int(np.float32(vmax).view(np.uint32))
    return 0 if bits == 0 else ((bits >> 23) & 0xff) - 126


def estimate_base_score(params, label, weight=None):
    """One Newton step of a stump from margin 0 with 40-bit fixed-point sums, then the prediction transform."""
    n = len(label)
    g, h, _ = gradients(params, np.zeros(n, F), label, weight)
    kg = np.ldexp(1.0, 40 - _quant_exponent(np.max(np.abs(g)) if n else 0.0))
    kh = np.ldexp(1.0, 40 - _quant_exponent(np.max(np.abs(h)) if n else 0.0))
    G = float(np.sum(np.rint(g.astype(np.float64) * kg).astype(np.int64))) / kg
    H = float(np.sum(np.rint(h.astype(np.float64) * kh).astype(np.int64))) / kh
    stump = F(0.0) if H <= 1e-6 else F(-G / H)
    return float(transform(params["objective"], np.array([stump], F))[0])


def base_margin(obj, b):
    """Margin of base_score b: the inverse transform, evaluated with libm's logf like the engine's host code."""
    b = F(b)
    if obj == "reg:logistic":
        return float(F(-_libm.logf(float(F(1.0) / b - F(1.0)))))
    if obj in LOG_LINK:
        return float(F(_libm.logf(float(b))))
    return float(b)


def metric(name, obj, margin, label, weight=None, params=None):
    """Metric on the transformed prediction, float64 sums (the engine allreduces (sum w*loss, sum w))."""
    from scipy.special import gammaln
    params = params or {}
    q = transform(obj, np.asarray(margin, F).reshape(-1)).astype(np.float64)
    y = np.asarray(label, F).astype(np.float64)
    w = np.ones_like(y) if weight is None else np.asarray(weight, F).astype(np.float64)
    with np.errstate(all="ignore"):
        if name in ("rmse", "mae"):
            v = (q - y) ** 2 if name == "rmse" else np.abs(q - y)
        elif name == "logloss":
            qf = transform(obj, np.asarray(margin, F).reshape(-1))
            a = np.maximum(qf, F(1e-16)).astype(np.float64)
            b = np.maximum(F(1.0) - qf, F(1e-16)).astype(np.float64)
            v = -(y * np.log(a) + (1 - y) * np.log(b))
        elif name == "rmsle":
            v = (np.log1p(y) - np.log1p(np.maximum(q, -1 + 1e-6))) ** 2
        elif name == "mape":
            v = np.abs((y - q) / y)
        elif name == "mphe":
            d = float(F(params.get("huber_slope", 1.0)))
            v = d * d * (np.sqrt(1 + ((y - q) / d) ** 2) - 1)
        elif name == "poisson-nloglik":
            qq = np.maximum(q, 1e-16)
            v = gammaln(y + 1) + qq - y * np.log(qq)
        elif name == "gamma-nloglik":
            v = y / q + np.log(q)
        elif name == "gamma-deviance":
            v = 2 * (np.log((q + 1e-6) / (y + 1e-6)) + (y + 1e-6) / (q + 1e-6) - 1)
        elif name.startswith("tweedie-nloglik"):
            r = float(F(name.split("@", 1)[1])) if "@" in name else 1.5
            v = -y * q ** (1 - r) / (1 - r) + q ** (2 - r) / (2 - r)
        else:
            raise KeyError(name)
    m = float(np.sum(v * w) / np.sum(w))
    return float(np.sqrt(m)) if name in ("rmse", "rmsle") else m


class Model:
    """Oracle booster grown from the reference gradients; `margin` is its prediction cache of the train rows."""

    def __init__(self, params, bst, base_score):
        self.params, self.bst, self.base_score = params, bst, base_score

    @property
    def margin(self):
        return self.bst.margin[:, 0]

    def tree(self, i):
        return self.bst.tree(i)

    @property
    def num_trees(self):
        return self.bst.num_trees

    def predict_margin(self, X):
        return self.bst.predict_margin(X)[:, 0]

    def predict(self, X):
        return transform(self.params["objective"], self.predict_margin(X))

    def metric(self, name, margin, label, weight=None):
        return metric(name, self.params["objective"], margin, label, weight, self.params)


def train(oracle, params, X, y, rounds, weight=None, is_cat=None, base_margin_rows=None):
    """Trees of `rounds` rounds: the oracle's tree growth (cuts, histograms, splits, sampling, max_delta_step clamp)
    fed with this module's gradients through its custom-gradient path."""
    obj = params["objective"]
    X = np.ascontiguousarray(X, F)
    y = np.ascontiguousarray(y, F)
    check_labels(obj, y)
    b = params.get("base_score")
    b = estimate_base_score(params, y, weight) if b is None else float(F(b))
    oparams = {k: v for k, v in params.items() if k not in ("objective", "base_score", "max_delta_step",
                                                             "eval_metric", "scale_pos_weight")}
    oparams.update(objective="reg:squarederror", base_score=base_margin(obj, b), max_delta_step=max_delta_step(params))
    cuts = oracle.Cuts.from_data(X, int(params.get("max_bin", 256)), np.nan, is_cat=is_cat, weight=weight)
    bins = cuts.bin(X)
    bst = oracle.Booster(oparams, cuts)
    bst.init_margin(X.shape[0], base_margin_rows)
    for _ in range(rounds):
        g, h, bad = gradients(params, bst.margin[:, 0], y, weight)
        if bad:
            raise FloatingPointError("%s: a gradient or hessian is not finite" % obj)
        bst.boost(bins, y, weight, custom_g=g, custom_h=h)
    return Model(params, bst, b)
