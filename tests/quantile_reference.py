"""reg:quantileerror on top of the oracle: pinball gradients and the leaf refresh in NumPy, the trees grown by the oracle
from those gradients as custom gradients.

What the engine implements (csrc/quantile_kernel.cu, csrc/tree.cu quantile_select, csrc/round.cu estimate_base_score;
DESIGN.md 2), written out literally with np.sort so that the GPU tests can replay a trained model round by round:
  * gradients of output k at margin m: d = fp32(m_k - y), g = fp32((d >= 0 ? fp32(1 - alpha_k) : -alpha_k) * w), h = w;
  * after tree k of a round is grown, every leaf value becomes fp32(q * eta), q the alpha_k-quantile of the residuals
    r = fp32(y - m_k) of the leaf's rows with a nonzero hessian (`leaf_quantile`); a leaf without such rows keeps the
    oracle's Newton value;
  * the intercept (base_score=None) is the fp32 mean over k of the alpha_k-quantile of the labels (`intercept`).
Weights enter the weighted rule as fixed-point integers rint(h * 2^(32 - e)), e the frexp exponent of the tree's largest
hessian, so their sums are exact."""
import numpy as np

from tests.dart_reference import hash4, leaves_on_bins

F32 = np.float32


def alphas_of(params):
    from xgboost_ray_b200.engine import quantile_alphas
    return quantile_alphas(params.get("quantile_alpha"))


def frexp_exponent(vmax):
    """e with 2^(e-1) <= vmax < 2^e (0 for 0), the engine's fixed-point exponent."""
    vmax = F32(vmax)
    return 0 if vmax == 0 else int(np.frexp(vmax)[1])


def fixed_mass(h, e):
    """Fixed-point weights rint(h * 2^(32 - e)) as int64 (exact: a float32 times a power of two, rounded once)."""
    return np.rint(np.asarray(h, np.float64) * 2.0 ** (32 - e)).astype(np.int64)


def leaf_quantile(r, alpha, mass=None):
    """alpha-quantile of the float32 residuals r.  mass None: the unweighted interpolating rule (numpy's "weibull");
    else int64 fixed-point weights and the weighted rule (the first value in ascending order whose cumulative weight
    reaches ceil(alpha W); the minimum when that is 0).  None for no rows."""
    r = np.array(r, F32).reshape(-1)
    r[r == 0] = F32(0.0)                       # -0 and +0 are one value
    n = r.size
    if n == 0:
        return None
    a = float(F32(alpha))
    if mass is None:
        v = np.sort(r)
        n1 = float(n + 1)
        if a <= 1.0 / n1:
            return v[0]
        if a >= n / n1:
            return v[-1]
        x = a * n1
        j = int(np.floor(x)) - 1
        d = (x - 1.0) - j
        return F32(float(v[j]) + d * float(F32(v[j + 1] - v[j])))
    mass = np.asarray(mass, np.int64).reshape(-1)
    order = np.argsort(r, kind="stable")
    v, cm = r[order], np.cumsum(mass[order])
    # the engine's sums are exact integers: check that float64 holds them exactly here
    assert int(cm[-1]) < 2 ** 63 and all(int(c) == c for c in cm.tolist())
    target = int(np.ceil(a * float(int(cm[-1]))))
    if target < 1:
        return v[0]
    return v[min(int(np.argmax(cm >= target)), n - 1)]


def weighted_quantile_fp32(r, alpha, w):
    """The weighted rule with running float32 weight sums (the alternative the engine's exact sums replace)."""
    r = np.asarray(r, F32)
    order = np.argsort(r, kind="stable")
    v, ws = r[order], np.asarray(w, F32)[order]
    cum = np.zeros(len(ws), F32)
    s = F32(0)
    for i, x in enumerate(ws):
        s = F32(s + x)
        cum[i] = s
    thr = F32(F32(alpha) * s)
    return v[min(int(np.argmax(cum >= thr)), len(v) - 1)]


def segment_quantile(r, h, alpha, weighted, e):
    keep = h != 0
    return leaf_quantile(r[keep], alpha, fixed_mass(h[keep], e) if weighted else None)


def intercept(y, weight, alphas):
    """base_score when none is given: the fp32 mean over the alphas of the quantile of the labels."""
    y = np.asarray(y, F32)
    h = np.ones(y.size, F32) if weight is None else np.asarray(weight, F32)
    e = frexp_exponent(np.max(np.abs(h))) if h.size else 0
    s = F32(0.0)
    for a in alphas:
        q = segment_quantile(y, h, a, weight is not None, e)
        s = F32(s + (F32(0.0) if q is None else q))
    return F32(s / F32(len(alphas)))


def gradients(margin, y, weight, alphas):
    """[n][T] float32 pinball gradients and hessians at margin [n][T]."""
    m = np.asarray(margin, F32)
    y = np.asarray(y, F32)[:, None]
    w = (np.ones(m.shape[0], F32) if weight is None else np.asarray(weight, F32))[:, None]
    a = np.asarray(alphas, F32)[None, :]
    d = (m - y).astype(F32)
    coef = np.where(d >= 0, (F32(1.0) - a).astype(F32), -a).astype(F32)
    return (coef * w).astype(F32), np.broadcast_to(w, m.shape).astype(F32).copy()


def pinball(margin, y, weight, alphas):
    """The quantile metric: weighted mean over rows and alphas of rho_alpha(y - p)."""
    m = np.asarray(margin, np.float64).reshape(len(y), -1)
    u = np.asarray(y, np.float64)[:, None] - m
    a = np.asarray(alphas, F32).astype(np.float64)[None, :]
    loss = np.where(u >= 0, a * u, (a - 1.0) * u).sum(axis=1)
    w = np.ones(len(y)) if weight is None else np.asarray(weight, np.float64)
    return float((loss * w).sum() / (w.sum() * m.shape[1]))


class Model:
    """Trees in the engine's order with refreshed leaf values, the margins they give, and the intercept."""

    def __init__(self, trees, margin, base_score):
        self.trees, self.margin, self.base_score = trees, margin, base_score

    @property
    def num_trees(self):
        return len(self.trees)

    def tree(self, i):
        return self.trees[i]


def train(oracle, params, X, y, rounds, weight=None, is_cat=None, base_margin=None):
    """`rounds` rounds of reg:quantileerror grown by the oracle from the pinball gradients, leaves refreshed here."""
    alphas = alphas_of(params)
    T = alphas.size
    eta = F32(params.get("eta", params.get("learning_rate", 0.3)))
    X = np.ascontiguousarray(X, F32)
    y = np.ascontiguousarray(y, F32)
    base = params.get("base_score")
    base = intercept(y, weight, alphas) if base is None else F32(base)
    op = {k: v for k, v in params.items() if k not in ("quantile_alpha", "eval_metric")}
    op.update(objective="multi:softprob" if T > 1 else "reg:squarederror", num_class=T, base_score=float(base))
    cuts = oracle.Cuts.from_data(X, int(params.get("max_bin", 256)), np.nan, is_cat=is_cat, weight=weight)
    bins = cuts.bin(X)
    bst = oracle.Booster(op, cuts)
    n = X.shape[0]
    if base_margin is not None:
        margin = np.array(np.asarray(base_margin, F32).reshape(n, -1), F32)
        if margin.shape[1] != T:
            margin = np.repeat(margin, T, axis=1)
    else:
        margin = np.full((n, T), base, F32)
    sub = float(params.get("subsample", 1.0))
    seed = int(params.get("seed", params.get("random_state", 0)) or 0)
    thr = min(int(sub * 4294967296.0), 0xFFFFFFFF)
    trees = []
    for r in range(rounds):
        g, h = gradients(margin, y, weight, alphas)
        bst.boost(bins, y, weight, custom_g=g.reshape(-1), custom_h=h.reshape(-1))
        for k in range(T):
            ti = r * T + k
            t = bst.tree(ti)
            hk = h[:, k].copy()
            if sub < 1.0:
                keep = np.array([hash4(seed, ti, 0, i) < thr for i in range(n)])
                hk[~keep] = 0
            e = frexp_exponent(np.max(np.abs(hk))) if n else 0
            nid = leaves_on_bins(t, bins, cuts.has_missing)
            res = (y - margin[:, k]).astype(F32)
            value = t.value.copy()
            for leaf in np.nonzero(t.split_feature < 0)[0]:
                rows = nid == leaf
                q = segment_quantile(res[rows], hk[rows], alphas[k], weight is not None, e)
                if q is not None:
                    value[leaf] = F32(q * eta)
            t.value = value
            margin[:, k] = (margin[:, k] + value[nid]).astype(F32)
            trees.append(t)
    return Model(trees, margin, base)
