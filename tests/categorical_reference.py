"""NumPy restatement of the categorical split scan at one node (DESIGN.md §2 items 5 and 6; xgboost's EnumerateOneHot /
EnumeratePart, src/tree/hist/evaluate_splits.h), written from the rules and not from either implementation.

Input: the node's quantised per-category integer sums (g, h) of every categorical feature, the node's totals (the rows a
feature does not see are its missing rows), the quantisation scales 2^(e - qbits) and the training parameters.  Every
sum is an exact integer; it becomes a float64 only by one multiply with the power-of-two scale, and the other side of a
split is the node total minus that double, as in the oracle and the kernel.  Rules restated:

* a feature of nf categories (the cuts are the codes 0..max, so nf = largest code + 1 and codes without rows are present
  with (0, 0)) is scanned one-hot when nf < max_cat_to_onehot, otherwise by sorted partition;
* one-hot: for each category in code order, the category goes right with the missing rows left (default_left = 1),
  then with them right (default_left = 0);
* partition: the categories are stable-sorted ascending by the binary32 CalcWeight of their (G, H); forward, the k + 1
  lightest go right and the missing rows left, k = 0 .. n_iter - 1; then backward, the t + 1 heaviest go left and the
  missing rows right; n_iter = min(max_cat_threshold, nf) - 1;
* a candidate needs both children's hessian >= min_child_weight; its loss_chg is binary32(gain(L) + gain(R) - root_gain)
  with root_gain = binary32(gain(node)); it is taken only if finite and > 0, and it replaces the best only with a
  strictly larger loss_chg, so ties keep the earlier candidate in enumeration order (features ascending).
"""
import numpy as np

from tests.fixed_sums_reference import calc_weight, quant_exponent

F = np.float32


def quantize(v, qbits):
    """(q int64, e): q = rint(v * 2^(qbits - e)), e the frexp exponent of max |v| (DESIGN.md §2 item 5)."""
    e = quant_exponent(v)
    return np.rint(np.asarray(v, F).astype(np.float64) * np.ldexp(1.0, qbits - e)).astype(np.int64), e


def train_params(params):
    """The scan's parameters as the engine holds them: binary32 values widened to float64."""
    d = lambda k, alt, v: float(F(params.get(k, params.get(alt, v))))   # noqa: E731
    return {"min_child_weight": d("min_child_weight", "min_child_weight", 1.0), "reg_lambda": d("lambda", "reg_lambda", 1.0),
            "alpha": d("alpha", "reg_alpha", 0.0), "max_delta_step": d("max_delta_step", "max_delta_step", 0.0),
            "max_cat_to_onehot": int(params.get("max_cat_to_onehot", 4)),
            "max_cat_threshold": int(params.get("max_cat_threshold", 64))}


def calc_gain(G, H, min_child_weight=1.0, reg_lambda=1.0, alpha=0.0, max_delta_step=0.0):
    """xgboost's CalcGain in float64 (b2_calc_gain, common.cuh)."""
    if H < min_child_weight or H <= 0.0:
        return 0.0
    t = G
    if alpha != 0.0:
        t = G - alpha if G > alpha else (G + alpha if G < -alpha else 0.0)
    if max_delta_step == 0.0:
        return (t * t) / (H + reg_lambda)
    w = calc_weight(G, H, min_child_weight, reg_lambda, alpha, max_delta_step)
    ret = -((2.0 * G) * w + (H + reg_lambda) * (w * w))
    return ret if alpha == 0.0 else ret + alpha * abs(w)


def node_histogram(codes, qg, qh):
    """Per-feature category sums of one node from its rows.  codes [n, Fc] float (NaN = missing, else an integer code
    in [0, 255]); qg, qh [n] quantised gradient pairs.  Returns (cat_g [Fc, 256], cat_h [Fc, 256], nf [Fc], tot_g, tot_h)
    with nf the cuts' category count (largest code + 1, 1 when the feature has no value)."""
    codes = np.asarray(codes, np.float64)
    qg, qh = np.asarray(qg, np.int64), np.asarray(qh, np.int64)
    Fc = codes.shape[1]
    cat_g, cat_h = np.zeros((Fc, 256), np.int64), np.zeros((Fc, 256), np.int64)
    nf = np.ones(Fc, np.int64)
    for f in range(Fc):
        ok = ~np.isnan(codes[:, f])
        c = codes[ok, f].astype(np.int64)
        np.add.at(cat_g[f], c, qg[ok])
        np.add.at(cat_h[f], c, qh[ok])
        if c.size:
            nf[f] = int(c.max()) + 1
    return cat_g, cat_h, nf, int(qg.sum()), int(qh.sum())


def sorted_categories(g, h, sg, sh, p):
    """Category codes 0..nf-1 stable-sorted ascending by binary32 CalcWeight, and those weights."""
    kw = {k: p[k] for k in ("min_child_weight", "reg_lambda", "alpha", "max_delta_step")}
    w = np.array([F(calc_weight(float(gi) * sg, float(hi) * sh, **kw)) for gi, hi in zip(g, h)], F)
    return np.argsort(w, kind="stable"), w


def feature_candidates(g, h, tot_g, tot_h, sg, sh, p):
    """Every candidate of one feature in enumeration order: dicts with loss_chg (binary32, None when a child is below
    min_child_weight), kind ('onehot' | 'forward' | 'backward'), default_left, right (set of codes that go right),
    bin (the category of a one-hot split, -1 for a partition) and the left child's integer sums."""
    nf = len(g)
    kw = {k: p[k] for k in ("min_child_weight", "reg_lambda", "alpha", "max_delta_step")}
    mcw = kw["min_child_weight"]
    G, H = float(tot_g) * sg, float(tot_h) * sh
    root_gain = float(F(calc_gain(G, H, **kw)))

    def cand(kind, dl, right, bin_, right_is_int, ig, ih):
        # right_is_int: the integer sums are the right child's, else the left child's
        a_h = float(ih) * sh
        b_h = H - a_h
        rh, lh = (a_h, b_h) if right_is_int else (b_h, a_h)
        c = {"kind": kind, "default_left": dl, "right": right, "bin": bin_,
             "left_g": tot_g - ig if right_is_int else ig, "left_h": tot_h - ih if right_is_int else ih, "loss_chg": None}
        if lh >= mcw and rh >= mcw:
            a_g = float(ig) * sg
            b_g = G - a_g
            rg, lg = (a_g, b_g) if right_is_int else (b_g, a_g)
            c["loss_chg"] = F((calc_gain(lg, lh, **kw) + calc_gain(rg, rh, **kw)) - root_gain)
        return c

    out = []
    real_g, real_h = int(np.sum(g)), int(np.sum(h))
    if nf < p["max_cat_to_onehot"]:
        mg, mh = tot_g - real_g, tot_h - real_h
        for b in range(nf):
            out.append(cand("onehot", 1, {b}, b, True, int(g[b]), int(h[b])))
            out.append(cand("onehot", 0, {b}, b, True, int(g[b]) + mg, int(h[b]) + mh))
        return out
    idx, _ = sorted_categories(g, h, sg, sh, p)
    pg, ph = np.cumsum(g[idx]), np.cumsum(h[idx])
    n_iter = min(p["max_cat_threshold"], nf) - 1
    for k in range(n_iter):
        out.append(cand("forward", 1, set(idx[:k + 1].tolist()), -1, True, int(pg[k]), int(ph[k])))
    for t in range(n_iter):
        i = nf - 1 - t
        out.append(cand("backward", 0, set(idx[:i].tolist()), -1, False, real_g - int(pg[i - 1]), real_h - int(ph[i - 1])))
    return out


def best_split(cat_g, cat_h, nf, tot_g, tot_h, sg, sh, params, features=None):
    """The node's best categorical candidate over `features` (default: all, ascending), or None.  Adds 'feature'."""
    p = train_params(params)
    best = None
    for f in (range(len(nf)) if features is None else features):
        for c in feature_candidates(cat_g[f][:nf[f]], cat_h[f][:nf[f]], tot_g, tot_h, sg, sh, p):
            chg = c["loss_chg"]
            if chg is None or not (chg > 0) or np.isinf(chg):
                continue
            if best is None or chg > best["loss_chg"]:
                best = dict(c, feature=f)
    return best


def tied_across(split, cat_g, cat_h, nf, sg, sh, params):
    """True when a partition split's set is cut through a group of equal binary32 weights: some code in the set and
    some code outside it weigh the same, so only the tie rule decides which of them goes right."""
    f = split["feature"]
    _, w = sorted_categories(cat_g[f][:nf[f]], cat_h[f][:nf[f]], sg, sh, train_params(params))
    inside = {float(w[c]) for c in split["right"]}
    return any(float(w[c]) in inside for c in range(nf[f]) if c not in split["right"])


def root_histogram(codes, g, h, qbits):
    """(cat_g, cat_h, nf, tot_g, tot_h, sg, sh) of a tree's root from the rows' codes and binary32 gradient pairs."""
    qg, eg = quantize(g, qbits)
    qh, eh = quantize(h, qbits)
    return node_histogram(codes, qg, qh) + (np.ldexp(1.0, eg - qbits), np.ldexp(1.0, eh - qbits))


def root_split(codes, g, h, qbits, params):
    """best_split at the root of one tree: returns (split or None, root_histogram(...))."""
    hist = root_histogram(codes, g, h, qbits)
    return best_split(*hist, params), hist


# ---- inputs
def tied_column(rng, nf, m, empty=(), few=(), few_m=2):
    """A shuffled column in which every code below nf has exactly m rows, codes in `few` few_m rows and codes in `empty`
    none (they stay in the cuts while a larger code has rows)."""
    counts = np.full(nf, m)
    counts[list(few)] = few_m
    counts[list(empty)] = 0
    col = np.repeat(np.arange(nf), counts).astype(F)
    rng.shuffle(col)
    return col


def tie_case(seed, nf=48, m=40, n_missing=300, n_other=3, values=(0.5, 1.0, 2.0, 4.0)):
    """Codes [n, 1 + n_other] and labels: feature 0 is tie-heavy -- its labels come from a table of repeated `values`, so
    categories of one value have identical (G, H); codes 5, 17 and 30 have no rows (weight +0.0), codes 3, 11, 12, 20,
    21, 33 and 40 have label 0 (G = 0, weight -0.0), codes 8 and 25 have two rows (below min_child_weight 3, weight 0),
    and missing rows have label 1.5.  The other features are random codes.  Use base_score 0 (g = -y exactly)."""
    rng = np.random.RandomState(seed)
    table = rng.choice(np.asarray(values, F), size=nf)
    zero = [3, 11, 12, 20, 21, 33, 40]
    table[zero] = 0.0
    c0 = tied_column(rng, nf, m, empty=(5, 17, 30), few=(8, 25))
    c0 = np.concatenate([c0, np.full(n_missing, np.nan, F)])
    rng.shuffle(c0)
    y = np.where(np.isnan(c0), F(1.5), table[np.nan_to_num(c0).astype(int)]).astype(F)
    n = len(c0)
    others = [rng.randint(0, k, size=n).astype(F) for k in (7, 60, 256)[:n_other]]
    return np.column_stack([c0] + others).astype(F), y


def random_case(seed, cards, n, nan_frac=0.0, weighted=False):
    """Codes [n, len(cards)] (feature f uses codes 0..cards[f]-1, each present; NaN at nan_frac, never in a feature of
    256 codes), labels that sum a random effect per (feature, code) and noise, and optional sample weights."""
    rng = np.random.RandomState(seed)
    cols, y = [], rng.normal(scale=0.3, size=n)
    for k in cards:
        c = rng.randint(0, k, size=n).astype(F)
        c[:k] = np.arange(k)
        y += rng.normal(size=k)[c.astype(int)] * rng.uniform(0.2, 2.0)
        if nan_frac > 0 and k < 256:
            miss = rng.uniform(size=n) < nan_frac
            miss[:k] = False
            c[miss] = np.nan
            y[miss] += rng.normal()
        cols.append(c)
    w = rng.uniform(0.25, 2.0, size=n).astype(F) if weighted else None
    return np.column_stack(cols).astype(F), y.astype(F), w


def root_matches(t, split, hist):
    """Assert that tree t (a dict of node arrays) splits its root as `split` does; hist is the root_histogram."""
    _, _, _, tot_g, tot_h, sg, sh = hist
    assert split is not None and split["loss_chg"] > 1e-6, split
    assert t["split_feature"][0] == split["feature"], (t["split_feature"][0], split["feature"])
    assert t["split_type"][0] == 1
    w = t["cat_bits"][0]
    assert [b for b in range(256) if (int(w[b >> 5]) >> (b & 31)) & 1] == sorted(split["right"])
    assert t["default_left"][0] == split["default_left"] and t["split_bin"][0] == split["bin"]
    assert F(t["loss_chg"][0]).view(np.uint32) == F(split["loss_chg"]).view(np.uint32), (t["loss_chg"][0], split["loss_chg"])
    left, right = t["left"][0], t["right"][0]
    assert t["sum_hess"][left] == float(split["left_h"]) * sh
    assert t["sum_hess"][right] == float(tot_h - split["left_h"]) * sh
