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


def q_key(r):
    """The kernel's order-preserving uint32 key of float32 values (negative: all bits flipped; else the sign set)."""
    u = np.asarray(r, F32).reshape(-1).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def q_unkey(k):
    k = np.uint32(k)
    return np.array([k & np.uint32(0x7FFFFFFF) if k & np.uint32(0x80000000) else ~k], np.uint32).view(F32)[0]


def radix_select(r, alpha, mass=None):
    """The selection as the kernel runs it (quantile_kernel.cu): four 8-bit passes over the keys, high byte first.  Each
    pass counts (or sums the masses of) the rows whose key matches a target's prefix so far, per digit, and picks the
    digit where the exclusive running sum is below the target and the inclusive one reaches it.  The two targets of the
    unweighted rule (order statistics j and j+1, 1-based ranks) share the histogram of slot 0 until their prefixes
    differ; after that the second target counts its own rows.  Returns (value, split), split the pass at which the two
    prefixes first differ (None: never).  (None, None) for no rows.  A second statement of `leaf_quantile`, to say in
    which pass a disagreement starts; `leaf_quantile` stays the reference."""
    r = np.array(r, F32).reshape(-1)
    r[r == 0] = F32(0.0)
    n = r.size
    if n == 0:
        return None, None
    keys = q_key(r)
    a = float(F32(alpha))
    rank, frac, by_mass = [1, 1], 0.0, False
    if mass is not None:
        mass = np.asarray(mass, np.int64).reshape(-1)
        target = int(np.ceil(a * float(int(mass.sum()))))
        if target >= 1:
            rank, by_mass = [target, target], True
    else:
        n1 = float(n + 1)
        if a <= 1.0 / n1:
            rank = [1, 1]
        elif a >= n / n1:
            rank = [n, n]
        else:
            x = a * n1
            j = int(np.floor(x)) - 1
            frac = (x - 1.0) - j
            rank = [j + 1, j + 2]
    prefix, split = [0, 0], None
    for p in range(4):
        shift = 24 - 8 * p
        digit = ((keys >> np.uint32(shift)) & np.uint32(0xFF)).astype(np.int64)
        apart = prefix[0] != prefix[1]
        picks = []
        for s in range(2):
            want = prefix[1 if (s == 1 and apart) else 0]
            rows = np.ones(n, bool) if p == 0 else (keys >> np.uint32(shift + 8)) == np.uint32(want >> (shift + 8))
            hist = np.zeros(256, np.int64)
            np.add.at(hist, digit[rows], mass[rows] if by_mass else 1)
            incl = np.cumsum(hist)
            ex = incl - hist
            hit = np.nonzero((ex < rank[s]) & (incl >= rank[s]))[0]
            assert hit.size == 1, "pass %d target %d: %d digits reach rank %d" % (p, s, hit.size, rank[s])
            picks.append((int(hit[0]), int(ex[hit[0]])))
        for s, (d, before) in enumerate(picks):
            prefix[s] |= d << shift
            rank[s] -= before
        if split is None and prefix[0] != prefix[1]:
            split = p
    v0, v1 = q_unkey(prefix[0]), q_unkey(prefix[1])
    return F32(float(v0) + frac * float(F32(v1 - v0))), split


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
    """Trees in the engine's order with refreshed leaf values, the margins they give, and the intercept.  `segments`
    (set by train) holds, per tree, its alpha and the (residuals, fixed-point masses or None) of every refreshed leaf."""

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
    trees, segments = [], []
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
            segs = []
            # the rows of every leaf in row order, from one stable sort (a depth-16 tree has up to 65,536 leaves)
            order = np.argsort(nid, kind="stable")
            leaves = np.nonzero(t.split_feature < 0)[0]
            starts = np.searchsorted(nid[order], leaves, side="left")
            ends = np.searchsorted(nid[order], leaves, side="right")
            for leaf, lo, hi in zip(leaves, starts, ends):
                rows = order[lo:hi]
                rows = rows[hk[rows] != 0]
                if rows.size == 0:
                    continue
                mass = fixed_mass(hk[rows], e) if weight is not None else None
                value[leaf] = F32(leaf_quantile(res[rows], alphas[k], mass) * eta)
                segs.append((res[rows], mass))
            t.value = value
            margin[:, k] = (margin[:, k] + value[nid]).astype(F32)
            trees.append(t)
            segments.append((alphas[k], segs))
    model = Model(trees, margin, base)
    model.segments = segments
    return model


# ---- label sets at the boundaries of the radix select
def f32_bits(u):
    return np.array([u], np.uint32).view(F32)[0]


TINY = f32_bits(0x00000001)                     # 2^-149, the smallest subnormal
HALF_MAX = f32_bits(0x7EFFFFFF)                 # FLT_MAX / 2, exactly
# (v_j, v_{j+1}, pass): adjacent order statistics whose keys share `pass` leading bytes, so the two targets of the
# interpolating rule take different digits first in that pass
SPLIT_PAIRS = [
    (F32(1.0), F32(2.0), 0),
    (F32(1.0), F32(1.0078125), 1),
    (F32(1.0), f32_bits(0x3F800100), 2),                # 1 + 256 ulp
    (F32(1.0), f32_bits(0x3F800001), 3),                # 1 + 1 ulp
    (-TINY, F32(0.0), 0),                               # the sign boundary: keys 0x7ffffffe and 0x80000000
    (F32(-2.0), F32(-1.0), 0),
    (f32_bits(0xBF800100), F32(-1.0), 2),
    (f32_bits(0xBF800001), F32(-1.0), 3),
    (-HALF_MAX, HALF_MAX, 0),
    (f32_bits(0x007FFFFF), f32_bits(0x00800000), 1),    # the largest subnormal and FLT_MIN
    (TINY, F32(2 * TINY), 3),
    (-HALF_MAX, f32_bits(0xFEFFFFFE), 3),
]
# every value of the pairs, both zeros and a few neighbours: the labels of the random boundary sets
POOL = np.unique(np.array(
    [v for a, b, _ in SPLIT_PAIRS for v in (a, b)] + [-0.0, 0.0, 0.5, -0.5, 3.0, -TINY * 3, f32_bits(0x3F810001),
                                                      f32_bits(0x3F7FFFFF), f32_bits(0x7EFFFFFE)], F32).view(np.uint32)).view(F32)


def pair_set(n, lo, hi, rng, ties=False):
    """n labels whose order statistics k - 1 and k (0-based, k = n // 2) are lo and hi, and the alpha that makes them
    the interpolating rule's j and j + 1.  The other labels come from POOL below lo and above hi, or (ties) are all lo
    below and all hi above, so that a tie straddles the target."""
    k = max(n // 2, 1)
    lower, upper = POOL[POOL < lo], POOL[POOL > hi]
    below = np.full(k - 1, lo, F32) if ties or lower.size == 0 else rng.choice(np.append(lower, lo), k - 1)
    above = np.full(n - k - 1, hi, F32) if ties or upper.size == 0 else rng.choice(np.append(upper, hi), n - k - 1)
    y = np.concatenate([below, [lo, hi], above]).astype(F32)
    return y[rng.permutation(n)], F32((k + 0.5) / (n + 1))


def edge_alphas(n):
    """alphas at the edges of the unweighted rule for n rows: the smallest, 1/(n+1) and n/(n+1) rounded to float32
    (exact when n + 1 is a power of two), the largest below 1, and one with alpha (n + 1) an integer (frac = 0) when
    n + 1 is even"""
    a = [F32(1e-7), F32(1.0 / (n + 1)), F32(n / (n + 1)), F32(0.99999994)]
    if (n + 1) % 2 == 0 and n > 1:
        a.append(F32(0.5))
    return a


def boundary_sets(n, seed=0):
    """(name, labels, alphas) at n rows: every split pair placed at the target, the tied variants, random POOL labels at
    the edge alphas, and n = 1 sets of one POOL value each"""
    rng = np.random.RandomState(seed + n)
    if n == 1:
        return [("single %r" % float(v), np.array([v], F32), [F32(0.3)]) for v in POOL]
    out = []
    for lo, hi, p in SPLIT_PAIRS:
        y, a = pair_set(n, lo, hi, rng)
        out.append(("pair %r %r (pass %d)" % (float(lo), float(hi), p), y, [a]))
        if n > 4:
            y, a = pair_set(n, lo, hi, rng, ties=True)
            out.append(("tied pair %r %r (pass %d)" % (float(lo), float(hi), p), y, [a]))
    y = rng.choice(POOL, n)
    out.append(("pool", y, edge_alphas(n)))
    if n > 2:
        signed = np.where(np.arange(n) % 2 == 0, F32(-0.0), F32(0.0)).astype(F32)
        signed[: n // 4] = rng.choice(POOL, n // 4)
        out.append(("signed zeros", signed[rng.permutation(n)], [F32(0.5), F32(0.25), F32(0.9)]))
    return out


def boundary_weights(kind, n, rng):
    """float32 weights: 'int' integers 0-4 (max a power of two, so the masses are exact multiples of 2^29), 'half'
    masses on half-way points (with max weight 1: 2^-32 -> mass 0.5 -> 0, 3 * 2^-32 -> 1.5 -> 2) and masses that round
    to 0, mixed with unit weights and zeros"""
    if kind == "int":
        w = rng.randint(0, 5, n).astype(F32)
        w[0] = 4.0
        return w
    if kind == "pow2":            # ones and twos summing to a power of two (see boundary_alpha)
        total = 1 << int(np.ceil(np.log2(n)))
        w = np.ones(n, F32)
        w[rng.choice(n, total - n, replace=False)] = 2.0
        return w
    w = rng.choice(np.array([2.0 ** -32, 3 * 2.0 ** -32, 5 * 2.0 ** -32, 2.0 ** -34, 0.0, 1.0, 0.5], F32), n)
    w[0] = 1.0
    return w


def boundary_alpha(y, w, rng):
    """For 'pow2' weights (total W a power of two): an alpha with alpha W exactly the cumulative weight up to some value
    v of y that has a larger value after it, so the weighted rule must pick v and not the next; None if y has one
    value"""
    y = np.array(y, F32)
    y[y == 0] = F32(0.0)
    order = np.argsort(y, kind="stable")
    v, cum = y[order], np.cumsum(np.asarray(w, np.float64)[order])
    ends = np.nonzero(v[:-1] < v[1:])[0]
    if ends.size == 0:
        return None
    a = cum[rng.choice(ends)] / cum[-1]
    assert F32(a) == a
    return F32(a)
