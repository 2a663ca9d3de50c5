"""Reference for learning to rank: a NumPy restatement of the query groups, the group-aligned sharding rule, the
LambdaMART gradients of rank:pairwise / rank:ndcg (xgboost 2.x, lambdarank_pair_method=topk; DESIGN.md 2, item 13),
1/IDCG and the ndcg / map / pre metrics, and a trainer that grows trees with the CPU oracle (oracle/hist_oracle.c) from
those gradients through its custom-gradient path.

TEST INFRASTRUCTURE ONLY, like the oracle.  The gradients replay rank_kernel.cu operation for operation: binary32 where
the kernel rounds to binary32 (the margin difference, the sigmoid, the per-row accumulation), binary64 otherwise, and
the sums in the kernel's fixed order with np.add.accumulate (sequential, unlike np.sum).  log and exp are the fdlibm
replays of tests/survival_reference.py, the sigmoid is objective_reference.sigmoid_.  So the gradient pairs are
bit-equal to the engine's.
"""
import numpy as np

from tests import objective_reference as OR
from tests import survival_reference as SR

D = np.float64
F = np.float32
LN2 = float(np.log(2.0))
OBJECTIVES = ("rank:pairwise", "rank:ndcg")


# ------------------------------------------------------------------------------------------------ groups and shards
def group_ptr(qid):
    """Row offsets of the groups of a non-decreasing qid: a group is a maximal run of equal ids."""
    q = np.asarray(qid).reshape(-1)
    if q.size and np.any(q[1:] < q[:-1]):
        raise ValueError("qid must be non-decreasing")
    starts = [i for i in range(q.size) if i == 0 or q[i] != q[i - 1]]
    return np.array(starts + [q.size], np.int64)


def sort_by_qid(qid):
    """Stable (merge sort) row order that makes qid non-decreasing; the identity when it already is."""
    q = np.asarray(qid).reshape(-1)
    return np.argsort(q, kind="mergesort")


def shard_rows(ptr, sharding, rank, world):
    """Rows of `rank` when every group goes whole to one rank: group g to rank g mod W (interleaved) or the group list
    split like numpy.array_split (batch)."""
    ng = len(ptr) - 1
    if ng < world:
        raise ValueError("%d query groups cannot be spread over %d actors" % (ng, world))
    if sharding == "interleaved":
        groups = range(rank, ng, world)
    else:
        groups = np.array_split(np.arange(ng), world)[rank]
    rows = [np.arange(ptr[g], ptr[g + 1]) for g in groups]
    return np.concatenate(rows).astype(np.int64) if rows else np.zeros(0, np.int64)


# ------------------------------------------------------------------------------------------------ building blocks
def disc(n):
    """ln2 / log(r + 2) for r < n (fdlibm log)."""
    return LN2 / SR.log_(np.arange(n, dtype=D) + 2.0)


def gain(y, exp_gain):
    """2^y - 1 (exact for an integer y, exp(y ln2) - 1 otherwise) or y."""
    y = np.asarray(y, F).astype(D)
    if not exp_gain:
        return y
    whole = y == np.floor(y)
    yi = np.where(whole, y, 0.0).astype(np.int64)
    return np.where(whole, np.ldexp(1.0, yi) - 1.0, SR.exp_(y * LN2) - 1.0)


def model_order(v):
    """Positions of a group sorted by v descending, ties by position (a stable sort); -0.0 counts as +0.0."""
    v = np.asarray(v, F) + F(0.0)
    return np.argsort(-v, kind="stable")


def inv_idcg(y, k, exp_gain):
    """1 / sum_{t < min(k, n)} G(y_t) D_t with y sorted descending; 0 when the sum is 0."""
    ys = np.asarray(y, F)[model_order(y)]
    t = min(k, len(ys))
    terms = gain(ys[:t], exp_gain) * disc(len(ys))[:t]
    s = np.add.accumulate(np.r_[0.0, terms])[-1]
    return 0.0 if s == 0.0 else 1.0 / s


def pair_values(objective, sa, ya, ra, sb, yb, rb, exp_gain, dsc, inv, scale):
    """(float lambda, float H, a_high) of pairs (a, b) with different labels (arrays)."""
    ah = ya > yb
    d = np.where(ah, sa - sb, sb - sa).astype(F)
    sig = OR.sigmoid_(d).astype(D)
    if objective == "rank:ndcg":
        gh, gl = gain(np.where(ah, ya, yb), exp_gain), gain(np.where(ah, yb, ya), exp_gain)
        dh, dl = dsc[np.where(ah, ra, rb)], dsc[np.where(ah, rb, ra)]
        delta = np.abs(((gh * dh + gl * dl) - (gl * dh + gh * dl)) * inv)
    else:
        delta = np.ones(d.shape, D)
    if scale:
        delta = delta / (np.abs(d).astype(D) + 0.01)
    lam = (sig - 1.0) * delta
    hh = np.maximum(sig * (1.0 - sig), 1e-16)
    H = (hh * delta) * 2.0
    return lam.astype(F), H.astype(F), ah


def group_gradients(objective, m, y, k, exp_gain, normalise=True):
    """Gradient pairs of one group (rows in group order) -> (g, h) float32 in group order."""
    m = np.asarray(m, F) + F(0.0)
    y = np.asarray(y, F)
    n = len(m)
    if n < 2:
        return np.zeros(n, F), np.zeros(n, F)
    order = model_order(m)
    M, Y = m[order], y[order]
    kk = min(k, n)
    dsc = disc(n)
    inv = inv_idcg(y, k, exp_gain) if objective == "rank:ndcg" else 0.0
    scale = bool(M[0] != M[n - 1])
    # pair table: rows i < kk, columns j; valid where j > i and the labels differ
    I = np.arange(kk)[:, None]
    J = np.arange(n)[None, :]
    valid = (J > I) & (Y[:kk, None] != Y[None, :])
    lam, H, ah = pair_values(objective, np.broadcast_to(M[:kk, None], (kk, n)), np.broadcast_to(Y[:kk, None], (kk, n)),
                             np.broadcast_to(I, (kk, n)), np.broadcast_to(M[None, :], (kk, n)),
                             np.broadcast_to(Y[None, :], (kk, n)), np.broadcast_to(J, (kk, n)), exp_gain, dsc, inv, scale)
    lam = np.where(valid, lam, F(0.0)).astype(F)
    H = np.where(valid, H, F(0.0)).astype(F)
    # row r as the second member of (i, r): + lambda when r is high (i low), - lambda when r is low
    as_second_g = np.where(ah, -lam, lam).astype(F)          # [i, r]
    as_first_g = np.where(ah, lam, -lam).astype(F)           # [r, j]
    z = np.zeros((n, 1), F)
    g1 = np.add.accumulate(np.concatenate([z, as_second_g.T], axis=1), axis=1)[:, -1]   # (i, r), i ascending
    h1 = np.add.accumulate(np.concatenate([z, H.T], axis=1), axis=1)[:, -1]
    g = g1.astype(F).copy()
    h = h1.astype(F).copy()
    g[:kk] = np.add.accumulate(np.concatenate([g1[:kk, None], as_first_g], axis=1), axis=1)[:, -1]   # then (r, j)
    h[:kk] = np.add.accumulate(np.concatenate([h1[:kk, None], H], axis=1), axis=1)[:, -1]
    if normalise:
        P = np.add.accumulate(np.concatenate([np.zeros((kk, 1)), -2.0 * lam.astype(D)], axis=1), axis=1)[:, -1]
        S = np.add.accumulate(np.r_[0.0, P])[-1]
        norm = (SR.log_(1.0 + S) / LN2) / S if S > 0.0 else 1.0
        g = (g.astype(D) * norm).astype(F)
        h = (h.astype(D) * norm).astype(F)
    go, ho = np.zeros(n, F), np.zeros(n, F)
    go[order], ho[order] = g, h
    return go, ho


def num_pair(params):
    k = int(params.get("lambdarank_num_pair_per_sample", 32))
    if k < 1:
        raise ValueError("lambdarank_num_pair_per_sample must be >= 1")
    return k


def exp_gain_of(params):
    v = params.get("ndcg_exp_gain", True)
    return v not in (False, 0, "0", "false", "False")


def gradients(params, margin, label, ptr):
    """(g, h, bad) of every row; `ptr` are the group offsets of the rows."""
    obj, k, eg = params["objective"], num_pair(params), exp_gain_of(params)
    margin = np.asarray(margin, F)
    label = np.asarray(label, F)
    g, h = np.zeros(len(margin), F), np.zeros(len(margin), F)
    for b, e in zip(ptr[:-1], ptr[1:]):
        g[b:e], h[b:e] = group_gradients(obj, margin[b:e], label[b:e], k, eg)
    bad = not (np.all(np.isfinite(g)) and np.all(np.isfinite(h)))
    return g, h, bad


def check_labels(params, y):
    y = np.asarray(y, F)
    if not np.all(np.isfinite(y) & (y >= 0)):
        raise ValueError("labels must be finite and >= 0")
    if exp_gain_of(params) and np.any(y > 31):
        raise ValueError("with ndcg_exp_gain the labels must be <= 31")


# ------------------------------------------------------------------------------------------------ metrics
def parse_metric(name):
    """('ndcg' | 'map' | 'pre', k or 0 for the whole group, minus)."""
    minus = name.endswith("-")
    s = name[:-1] if minus else name
    base, _, k = s.partition("@")
    return base, int(k) if k else 0, minus


def group_metric(name, pred, y, exp_gain=True):
    base, k, minus = parse_metric(name)
    pred, y = np.asarray(pred, F), np.asarray(y, F)
    n = len(y)
    kk = k if k > 0 else n
    t = min(n, kk)
    ys = y[model_order(pred)]
    if base == "ndcg":
        dsc = disc(n)
        dcg = np.add.accumulate(np.r_[0.0, gain(ys[:t], exp_gain) * dsc[:t]])[-1]
        idcg = np.add.accumulate(np.r_[0.0, gain(y[model_order(y)][:t], exp_gain) * dsc[:t]])[-1]
        return (0.0 if minus else 1.0) if idcg == 0.0 else dcg / idcg
    if base == "map":
        rel = int(np.count_nonzero(y != 0))
        if rel == 0:
            return 0.0 if minus else 1.0
        ap, hits = 0.0, 0
        for i in range(t):
            if ys[i] != 0:
                hits += 1
                ap += hits / (i + 1)
        return ap / rel
    if base == "pre":
        return int(np.count_nonzero(ys[:t] != 0)) / kk
    raise ValueError("unknown ranking metric %s" % name)


def metric(name, pred, y, ptr, exp_gain=True):
    """Mean over the groups of the per-group value."""
    vals = [group_metric(name, pred[b:e], y[b:e], exp_gain) for b, e in zip(ptr[:-1], ptr[1:])]
    return float(np.sum(vals) / len(vals)) if vals else 0.0


# ------------------------------------------------------------------------------------------------ training
class Model(OR.Model):
    def predict(self, X):
        return self.predict_margin(X)

    def metric(self, name, margin, label, ptr):
        return metric(name, margin, label, ptr, exp_gain_of(self.params))


def train(oracle, params, X, y, qid, rounds, is_cat=None, base_margin_rows=None):
    """Trees of `rounds` rounds: the oracle's tree growth fed with this module's gradients through its custom-gradient
    path, like objective_reference.train.  The rows must already be sorted by qid."""
    X = np.ascontiguousarray(X, F)
    y = np.ascontiguousarray(y, F)
    ptr = group_ptr(qid)
    check_labels(params, y)
    b = float(F(params.get("base_score", 0.5)))
    oparams = {k: v for k, v in params.items() if k not in ("objective", "base_score", "eval_metric",
                                                             "lambdarank_pair_method", "lambdarank_num_pair_per_sample",
                                                             "lambdarank_unbiased", "ndcg_exp_gain")}
    oparams.update(objective="reg:squarederror", base_score=b)
    cuts = oracle.Cuts.from_data(X, int(params.get("max_bin", 256)), np.nan, is_cat=is_cat)
    bins = cuts.bin(X)
    bst = oracle.Booster(oparams, cuts)
    bst.init_margin(X.shape[0], base_margin_rows)
    for _ in range(rounds):
        g, h, bad = gradients(params, bst.margin[:, 0], y, ptr)
        if bad:
            raise FloatingPointError("%s: a gradient or hessian is not finite" % params["objective"])
        bst.boost(bins, y, None, custom_g=g, custom_h=h)
    return Model(dict(params), bst, b)
