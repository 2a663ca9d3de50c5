"""Reference for rank:map (LambdaMART with the Delta-AP pair weight; DESIGN.md 2, item 13): a NumPy restatement of
the hit prefixes, the pair weight and the gradients, and a trainer that grows trees with the CPU oracle from them.

TEST INFRASTRUCTURE ONLY, like the oracle.  Everything except the pair weight is rank:ndcg's rule and is taken from
tests/ranking_reference.py (model order, sigmoid, the |d| + 0.01 scaling, lambda / H, the per-row accumulation order
and the log2(1 + S) / S normalisation), replayed operation for operation as in rank_kernel.cu, so the gradient pairs
are bit-equal to the engine's.
"""
import numpy as np

from tests import objective_reference as OR
from tests import ranking_reference as RR
from tests import survival_reference as SR

D = np.float64
F = np.float32
MAP_OBJECTIVE = "rank:map"
PREFIX_THREADS = 128                # rank_kernel.cu's CTA size: the chunk count of the hit prefixes


def hit_prefixes(hits):
    """(R, A) of a group in model order: R_p = hits at positions <= p (exact integers) and A_p = the sum of 1/(q + 1)
    over the hits q <= p, in rank_kernel.cu's order: PREFIX_THREADS chunks of ceil(n / PREFIX_THREADS) positions, each
    summed ascending from 0.0; the chunk totals turned into exclusive carries ascending from 0.0; A_p = carry + local
    prefix.  Adding 0.0 for a miss leaves a sum unchanged, so the kernel, which adds hits only, gets the same bits."""
    r = np.asarray(hits, bool).reshape(-1)
    n = len(r)
    R = np.cumsum(r, dtype=np.int64)
    terms = np.where(r, 1.0 / (np.arange(n, dtype=D) + 1.0), 0.0)
    c = max(1, -(-n // PREFIX_THREADS))
    starts = range(0, n, c)
    local = [np.add.accumulate(np.r_[0.0, terms[b:b + c]])[1:] for b in starts]
    carry = np.add.accumulate(np.r_[0.0, [v[-1] for v in local]])[:-1]
    A = np.concatenate([carry[t] + v for t, v in enumerate(local)]) if n else np.zeros(0, D)
    return R, A


def map_delta(R, A, n_hits, ra, rb, ah):
    """|Delta AP| of swapping model positions ra < rb with different labels; ah: the hit is at ra.  The binary64
    operation sequence of rank_kernel.cu (DESIGN.md 2, item 13):
      ah:     N dAP = (R_b/(b+1) - R_a/(a+1)) - (A_{b-1} - A_a)
      not ah: N dAP = ((R_a+1)/(a+1) - R_b/(b+1)) + (A_{b-1} - A_a)."""
    ra, rb, ah = np.asarray(ra), np.asarray(rb), np.asarray(ah)
    ta = np.where(ah, R[ra], R[ra] + 1).astype(D) / (ra + 1).astype(D)
    tb = R[rb].astype(D) / (rb + 1).astype(D)
    between = A[np.maximum(rb - 1, 0)] - A[ra]
    num = np.where(ah, (tb - ta) - between, (ta - tb) + between)
    return np.abs(num / D(n_hits if n_hits > 0 else 1))


def group_gradients(m, y, k, normalise=True):
    """Gradient pairs of one group (rows in group order) -> (g, h) float32 in group order: ranking_reference's
    group_gradients with Delta = |Delta AP|."""
    m = np.asarray(m, F) + F(0.0)
    y = np.asarray(y, F)
    n = len(m)
    if n < 2:
        return np.zeros(n, F), np.zeros(n, F)
    order = RR.model_order(m)
    M, Y = m[order], y[order]
    kk = min(k, n)
    R, A = hit_prefixes(Y != 0)
    scale = bool(M[0] != M[n - 1])
    # pair table: rows i < kk, columns j; valid where j > i and the labels differ
    I = np.broadcast_to(np.arange(kk)[:, None], (kk, n))
    J = np.broadcast_to(np.arange(n)[None, :], (kk, n))
    valid = (J > I) & (Y[:kk, None] != Y[None, :])
    ah = Y[:kk, None] > Y[None, :]
    d = np.where(ah, M[:kk, None] - M[None, :], M[None, :] - M[:kk, None]).astype(F)
    sig = OR.sigmoid_(d).astype(D)
    delta = map_delta(R, A, int(R[-1]), I, J, ah)
    if scale:
        delta = delta / (np.abs(d).astype(D) + 0.01)
    lam = ((sig - 1.0) * delta).astype(F)
    H = ((np.maximum(sig * (1.0 - sig), 1e-16) * delta) * 2.0).astype(F)
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
        norm = (SR.log_(1.0 + S) / RR.LN2) / S if S > 0.0 else 1.0
        g = (g.astype(D) * norm).astype(F)
        h = (h.astype(D) * norm).astype(F)
    go, ho = np.zeros(n, F), np.zeros(n, F)
    go[order], ho[order] = g, h
    return go, ho


def gradients(params, margin, label, ptr):
    """(g, h, bad) of every row; `ptr` are the group offsets of the rows."""
    k = RR.num_pair(params)
    margin = np.asarray(margin, F)
    label = np.asarray(label, F)
    g, h = np.zeros(len(margin), F), np.zeros(len(margin), F)
    for b, e in zip(ptr[:-1], ptr[1:]):
        g[b:e], h[b:e] = group_gradients(margin[b:e], label[b:e], k)
    bad = not (np.all(np.isfinite(g)) and np.all(np.isfinite(h)))
    return g, h, bad


def check_labels(y):
    """rank:map takes binary relevance only."""
    y = np.asarray(y, F)
    if not np.all((y == 0) | (y == 1)):
        raise ValueError("rank:map: labels must be 0 or 1")


def train(oracle, params, X, y, qid, rounds):
    """Trees of `rounds` rounds: the oracle's tree growth fed with this module's gradients through its custom-gradient
    path, like ranking_reference.train.  The rows must already be sorted by qid."""
    X = np.ascontiguousarray(X, F)
    y = np.ascontiguousarray(y, F)
    ptr = RR.group_ptr(qid)
    check_labels(y)
    b = float(F(params.get("base_score", 0.5)))
    oparams = {k: v for k, v in params.items() if k not in ("objective", "base_score", "eval_metric",
                                                             "lambdarank_pair_method", "lambdarank_num_pair_per_sample",
                                                             "lambdarank_unbiased", "ndcg_exp_gain")}
    oparams.update(objective="reg:squarederror", base_score=b)
    cuts = oracle.Cuts.from_data(X, int(params.get("max_bin", 256)), np.nan)
    bins = cuts.bin(X)
    bst = oracle.Booster(oparams, cuts)
    bst.init_margin(X.shape[0], None)
    for _ in range(rounds):
        g, h, bad = gradients(params, bst.margin[:, 0], y, ptr)
        if bad:
            raise FloatingPointError("rank:map: a gradient or hessian is not finite")
        bst.boost(bins, y, None, custom_g=g, custom_h=h)
    return RR.Model(dict(params), bst, b)
