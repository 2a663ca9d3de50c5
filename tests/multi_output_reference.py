"""Reference growth of vector-leaf trees (multi_strategy="multi_output_tree", DESIGN.md §2 item 19).  TEST INFRASTRUCTURE.

The level loop of tests/interaction_reference.py (the oracle's own primitives: oracle.Cuts, oracle.quantize per target,
oracle.hist_int per target, or_select_features), restated for T targets with the rules of item 19 written out literally:
  * target k is quantised with its own exponents, so its integer histograms are the single-target ones of column k;
  * gain(node) = sum over k (ascending, from 0.0) of CalcGain(G_k, H_k); parent_gain = fp32(gain(parent));
    loss_chg = fp32((gain(L) + gain(R)) - parent_gain), R_k = G_k - L_k in double;
  * no per-child min_child_weight filter (a target below it adds 0); the scalar enumeration order and tie-break;
    a backward scan on f when f's real-bin sums differ from the node totals for some target;
  * the winner expands when loss_chg > 1e-6, !(loss_chg < gamma) and each child has a nonzero hessian sum in some target;
  * leaf value of target k = fp32(fp32(CalcWeight) * eta) from the 40-bit fixed-point sums of the leaf's rows; an internal
    node's vector holds the same formula on its qbits sums;
  * row subsampling (the oracle's draw, restated in row_keep): a row is kept for tree t iff
    hash4(seed, t, rank, row) < subsample * 2^32; a dropped row keeps its place in the partition and receives the leaf
    vector, but carries (0, 0) in every target, before the quantisation exponents are taken.
predict_margin / pred_leaf walk the trees on raw binary32 values: a missing value (NaN, or equal to a non-NaN `missing`)
follows default_left, any other value goes left when x < split_cond; each tree's leaf vector is added in binary32.
With T = 1 and min_child_weight = 0 this is the oracle's scalar tree and prediction (tests/test_multi_output_reference.py
checks both).  Categorical features are not restated."""
from types import SimpleNamespace

import numpy as np

from oracle import oracle as O
from tests import multi_target_reference as MT
from tests.interaction_reference import (LEAF_BITS, MISSING_BIN, RT_EPS, SCOPE_LEVEL0, SCOPE_NODE0, SCOPE_TREE, _P,
                                         _select, allowed_features)

F32 = np.float32
_M64 = (1 << 64) - 1


def _mix64(x):
    """hist_oracle.c mix64 on a uint64 array (wrapping multiplies)"""
    x = x ^ (x >> np.uint64(30))
    x = x * np.uint64(0xbf58476d1ce4e5b9)
    x = x ^ (x >> np.uint64(27))
    x = x * np.uint64(0x94d049bb133111eb)
    return x ^ (x >> np.uint64(31))


def row_keep(seed, tree, rank, n, subsample):
    """the oracle's row draw for one tree: keep row i iff hash4(seed, tree, rank, i) < subsample * 2^32 (subsample as
    binary32 widened to double; a threshold at or past 2^32 - 1 keeps every row)"""
    thr_d = float(F32(subsample)) * 4294967296.0
    thr = 0xFFFFFFFF if thr_d >= 4294967295.0 else int(thr_d)
    h0 = ((seed & 0xFFFFFFFF) * 0x9e3779b97f4a7c15 + (tree & 0xFFFFFFFF)) & _M64
    h = _mix64(np.full(n, h0, np.uint64))
    h = _mix64(h + np.uint64(rank & 0xFFFFFFFF))
    h = _mix64(h + np.arange(n, dtype=np.uint64))
    return (h >> np.uint64(32)) < np.uint64(thr)


def node_gain(p, G, H):
    """sum_k CalcGain(G_k, H_k) in ascending k from 0.0 (float64 adds, round to nearest)"""
    acc = 0.0
    for k in range(len(G)):
        acc = acc + float(p.gain(G[k], H[k]))
    return acc


def _acc_gain(p, Gs, Hs):
    """per-candidate sums over the targets: Gs, Hs lists of T float64 arrays -> (sum_k gain) in ascending k"""
    acc = np.zeros_like(Gs[0], dtype=np.float64)
    for k in range(len(Gs)):
        acc = acc + p.gain(Gs[k], Hs[k])
    return acc


def best_split(p, cuts, hists, sg, sh, inv_g, inv_h, feats):
    """the first candidate of the largest finite loss_chg > 0 in enumeration order (feature ascending; per feature the
    forward bins ascending, then the backward bins descending); hists[k] = target k's integer histogram [F][256][2].
    Every feature's candidates are formed at once as [features][256] arrays, element by element with the operations of
    the per-feature scan, so each loss_chg is the same binary32 value; the enumeration order is the flattened order of
    [forward bins | backward bins reversed] per feature, and np.argmax keeps the first of equal maxima."""
    T = len(hists)
    G = [sg[k] * inv_g[k] for k in range(T)]
    H = [sh[k] * inv_h[k] for k in range(T)]
    parent_gain = float(F32(node_gain(p, G, H)))
    fa = np.array(sorted(feats), np.int64)
    if fa.size == 0:
        return None
    nf = (cuts.ptrs[fa + 1] - cuts.ptrs[fa]).astype(np.int64)
    fa, nf = fa[nf > 0], nf[nf > 0]
    if fa.size == 0:
        return None
    real = np.arange(256)[None, :] < nf[:, None]               # the feature's real bins
    hg = [np.where(real, hists[k][fa, :, 0], 0) for k in range(T)]
    hh = [np.where(real, hists[k][fa, :, 1], 0) for k in range(T)]
    cg = [np.cumsum(a, axis=1) for a in hg]
    ch = [np.cumsum(a, axis=1) for a in hh]
    tg = [a[:, -1:] for a in cg]                                # sums over the real bins
    th = [a[:, -1:] for a in ch]
    with np.errstate(all="ignore"):
        # forward: left = bins <= i, missing -> right
        lg = [cg[k] * inv_g[k] for k in range(T)]
        lh = [ch[k] * inv_h[k] for k in range(T)]
        chg_f = ((_acc_gain(p, lg, lh) + _acc_gain(p, [G[k] - lg[k] for k in range(T)],
                                                    [H[k] - lh[k] for k in range(T)])) - parent_gain).astype(F32)
        nzl_f = np.any([ch[k] != 0 for k in range(T)], axis=0)
        nzr_f = np.any([(sh[k] - ch[k]) != 0 for k in range(T)], axis=0)
        # backward at bin i: right = real bins >= i, missing -> left; only where some target has missing sums
        bgi = [tg[k] - (cg[k] - hg[k]) for k in range(T)]
        bhi = [th[k] - (ch[k] - hh[k]) for k in range(T)]
        rg = [bgi[k] * inv_g[k] for k in range(T)]
        rh = [bhi[k] * inv_h[k] for k in range(T)]
        chg_b = ((_acc_gain(p, [G[k] - rg[k] for k in range(T)], [H[k] - rh[k] for k in range(T)])
                  + _acc_gain(p, rg, rh)) - parent_gain).astype(F32)
        nzl_b = np.any([(sh[k] - bhi[k]) != 0 for k in range(T)], axis=0)
        nzr_b = np.any([bhi[k] != 0 for k in range(T)], axis=0)
    back = np.any([(tg[k][:, 0] != sg[k]) | (th[k][:, 0] != sh[k]) for k in range(T)], axis=0)

    def usable(chg, ok):
        return np.where(ok & np.isfinite(chg) & (chg > F32(0.0)), chg.astype(np.float64), -np.inf)

    cand = np.concatenate([usable(chg_f, real), usable(chg_b, real & back[:, None])[:, ::-1]], axis=1)
    flat = int(np.argmax(cand))
    j, c = divmod(flat, 512)
    if cand[j, c] == -np.inf:
        return None
    f = int(fa[j])
    if c < 256:
        i = c
        return dict(chg=chg_f[j, i], feature=f, bin=i, cond=float(cuts.vals[cuts.ptrs[f] + i]), default_left=0,
                    nz_l=bool(nzl_f[j, i]), nz_r=bool(nzr_f[j, i]))
    i = 511 - c
    cond = float(cuts.mins[f]) if i == 0 else float(cuts.vals[cuts.ptrs[f] + i - 1])
    return dict(chg=chg_b[j, i], feature=f, bin=i - 1, cond=cond, default_left=1, nz_l=bool(nzl_b[j, i]),
                nz_r=bool(nzr_b[j, i]))


def grow_tree(p, cuts, bins, g, h, sets, tree_index, fwq=None):
    """One vector-leaf tree on (bins, g [n][T], h [n][T]); returns (tree namespace, per-row leaf vectors [n][T])."""
    n, F = bins.shape
    T = g.shape[1]
    g, h = np.ascontiguousarray(g, F32), np.ascontiguousarray(h, F32)
    if p.subsample < 1.0:   # one draw for the tree: the dropped rows carry (0, 0) in every target
        keep = row_keep(p.seed, tree_index, p.rank, n, p.subsample)[:, None]
        g, h = np.where(keep, g, F32(0.0)), np.where(keep, h, F32(0.0))
    q = [(O.quantize(g[:, k], p.qbits), O.quantize(h[:, k], p.qbits)) for k in range(T)]
    qg, qh = [a[0][0] for a in q], [a[1][0] for a in q]
    eg, eh = [a[0][1] for a in q], [a[1][1] for a in q]
    inv_g = [np.ldexp(1.0, e - p.qbits) for e in eg]
    inv_h = [np.ldexp(1.0, e - p.qbits) for e in eh]
    kg = [np.ldexp(1.0, LEAF_BITS - e) for e in eg]
    kh = [np.ldexp(1.0, LEAF_BITS - e) for e in eh]
    use_cols = p.bytree < 1.0 or p.bylevel < 1.0 or p.bynode < 1.0
    mask_tree = _select(p.seed, tree_index, SCOPE_TREE, None, fwq, F, p.bytree) if use_cols else None
    t = dict(left=[], right=[], parent=[], split_feature=[], split_bin=[], split_cond=[], default_left=[], loss_chg=[],
             sum_hess=[], vec=[])

    def add(parent):
        for k, v in (("left", -1), ("right", -1), ("parent", parent), ("split_feature", -1), ("split_bin", -1),
                     ("split_cond", 0.0), ("default_left", 0), ("loss_chg", 0.0), ("sum_hess", 0.0),
                     ("vec", np.zeros(T, F32))):
            t[k].append(v)
        return len(t["left"]) - 1

    def hists(rows):
        return [O.hist_int(bins, qg[k], qh[k], rows) for k in range(T)]

    def set_node(nid, sg, sh):
        H = [sh[k] * inv_h[k] for k in range(T)]
        t["sum_hess"][nid] = sum(H)
        t["vec"][nid] = np.array([F32(F32(p.weight(sg[k] * inv_g[k], H[k])) * p.eta) for k in range(T)], F32)

    out = np.zeros((n, T), F32)
    ih = hists(None)
    sg = [int(ih[k][0, :, 0].sum()) for k in range(T)]
    sh = [int(ih[k][0, :, 1].sum()) for k in range(T)]
    root = add(-1)
    set_node(root, sg, sh)
    level = [dict(nid=root, depth=0, rows=np.arange(n, dtype=np.int32), sg=sg, sh=sh, path=frozenset(), hist=ih)]
    while level:
        mask_level = (_select(p.seed, tree_index, SCOPE_LEVEL0 + level[0]["depth"], mask_tree, fwq, F, p.bylevel)
                      if use_cols else None)
        nxt = []
        for w in level:
            split = None
            if w["depth"] < p.max_depth:
                feats = set(range(F)) if mask_level is None else set(np.nonzero(mask_level)[0].tolist())
                if use_cols and p.bynode < 1.0:
                    node_mask = _select(p.seed, tree_index, SCOPE_NODE0 + w["nid"], mask_level, fwq, F, p.bynode)
                    feats = set(np.nonzero(node_mask)[0].tolist())
                if sets:
                    feats &= allowed_features(w["path"], sets, F)
                split = best_split(p, cuts, w["hist"], w["sg"], w["sh"], inv_g, inv_h, feats)
                if split is not None and not (split["chg"] > RT_EPS and split["nz_l"] and split["nz_r"]
                                              and not (split["chg"] < p.gamma)):
                    split = None
            nid = w["nid"]
            if split is None:   # leaf: per target, the weight from the 40-bit fixed-point sums of its rows
                r = w["rows"]
                v = np.zeros(T, F32)
                for k in range(T):
                    G = float(int(np.rint(g[r, k].astype(np.float64) * kg[k]).astype(np.int64).sum())) / kg[k]
                    H = float(int(np.rint(h[r, k].astype(np.float64) * kh[k]).astype(np.int64).sum())) / kh[k]
                    v[k] = F32(F32(p.weight(G, H)) * p.eta)
                t["vec"][nid] = v
                out[r] = v
                continue
            f = split["feature"]
            l, r_ = add(nid), add(nid)
            t["left"][nid], t["right"][nid], t["split_feature"][nid], t["split_bin"][nid] = l, r_, f, split["bin"]
            t["split_cond"][nid], t["default_left"][nid], t["loss_chg"][nid] = split["cond"], split["default_left"], split["chg"]
            nf = int(cuts.ptrs[f + 1] - cuts.ptrs[f])
            lg, lh = [], []
            for k in range(T):   # the chosen feature's prefix, plus its missing rows when they go left
                hg, hh = w["hist"][k][f, :nf, 0], w["hist"][k][f, :nf, 1]
                pg, ph = int(hg[:split["bin"] + 1].sum()), int(hh[:split["bin"] + 1].sum())
                if split["default_left"]:
                    pg += w["sg"][k] - int(hg.sum())
                    ph += w["sh"][k] - int(hh.sum())
                lg.append(pg)
                lh.append(ph)
            rg = [w["sg"][k] - lg[k] for k in range(T)]
            rh = [w["sh"][k] - lh[k] for k in range(T)]
            set_node(l, lg, lh)
            set_node(r_, rg, rh)
            b = bins[w["rows"], f]
            go_left = np.where((b == MISSING_BIN) & bool(cuts.has_missing[f]), bool(split["default_left"]), b <= split["bin"])
            path = w["path"] | {f}
            for child, rows, cg, ch in ((l, w["rows"][go_left], lg, lh), (r_, w["rows"][~go_left], rg, rh)):
                hist = hists(rows) if w["depth"] + 1 < p.max_depth else None
                nxt.append(dict(nid=child, depth=w["depth"] + 1, rows=rows, sg=cg, sh=ch, path=path, hist=hist))
        level = nxt
    nn = len(t["left"])
    tree = SimpleNamespace(
        left=np.array(t["left"], np.int32), right=np.array(t["right"], np.int32), parent=np.array(t["parent"], np.int32),
        split_feature=np.array(t["split_feature"], np.int32), split_bin=np.array(t["split_bin"], np.int32),
        split_cond=np.array(t["split_cond"], F32), default_left=np.array(t["default_left"], np.uint8),
        loss_chg=np.array(t["loss_chg"], F32), sum_hess=np.array(t["sum_hess"], np.float64),
        leaf_vector=np.stack(t["vec"]).astype(F32), n_nodes=nn)
    return tree, out


class Model:
    """the trees, the train margins [n][T], base_score and the margin every row starts from (base_value)"""

    def __init__(self, trees, margin, base_score, base_value):
        self._trees, self.margin, self.base_score, self.base_value = trees, margin, base_score, base_value

    @property
    def num_trees(self):
        return len(self._trees)

    def tree(self, i):
        return self._trees[i]


def _tree_range(model, iteration_range):
    if iteration_range is None or tuple(iteration_range) == (0, 0):
        return 0, model.num_trees
    return int(iteration_range[0]), int(iteration_range[1])


def pred_leaf(model, X, missing=np.nan, iteration_range=None):
    """[n][trees] leaf node ids of the raw binary32 rows X: a missing value (NaN, or == missing when missing is not NaN;
    -0.0 == 0.0) follows default_left, any other value goes left when x < split_cond"""
    X = np.ascontiguousarray(X, F32)
    n = X.shape[0]
    rows = np.arange(n)
    b, e = _tree_range(model, iteration_range)
    out = np.zeros((n, e - b), np.int32)
    for j, t in enumerate(model._trees[b:e]):
        nid = np.zeros(n, np.int64)
        while True:
            inner = t.split_feature[nid] >= 0
            if not inner.any():
                break
            x = X[rows, np.maximum(t.split_feature[nid], 0)]
            miss = np.isnan(x) if np.isnan(missing) else (np.isnan(x) | (x == F32(missing)))
            left = np.where(miss, t.default_left[nid] != 0, x < t.split_cond[nid])
            nid = np.where(inner, np.where(left, t.left[nid], t.right[nid]), nid)
        out[:, j] = nid
    return out


def predict_margin(model, X, missing=np.nan, iteration_range=None):
    """[n][T] margins: base_value plus each tree's leaf vector, added in binary32 one tree at a time in tree order"""
    leaves = pred_leaf(model, X, missing, iteration_range)
    b, _ = _tree_range(model, iteration_range)
    T = model.tree(0).leaf_vector.shape[1]
    out = np.full((leaves.shape[0], T), F32(model.base_value), F32)
    for j in range(leaves.shape[1]):
        out = (out + model.tree(b + j).leaf_vector[leaves[:, j]]).astype(F32)
    return out


def train(params, X, Y, rounds, weight=None, sets=None, feature_weights=None, gradients=None, base_margin=None):
    """`rounds` vector-leaf trees on numeric X with the label Y [n][T] (one of the multi-target objectives of
    tests/multi_target_reference.py), or with gradients(margin [n][T]) -> (g, h) [n][T] (a custom objective)."""
    p = _P({k: v for k, v in params.items() if k not in ("multi_strategy", "objective", "base_score")}, rows_sampled=True)
    X = np.ascontiguousarray(X, F32)
    Y = np.ascontiguousarray(Y, F32)
    n, T = Y.shape
    obj = params.get("objective", "reg:squarederror")
    b = params.get("base_score")
    b = MT.intercept(params, Y, weight) if b is None else float(F32(b))
    cuts = O.Cuts.from_data(X, int(params.get("max_bin", 256)), weight=weight)
    bins = cuts.bin(X)
    fwq = None
    if feature_weights is not None:
        qf = np.asarray(feature_weights, np.float64) * 65536.0
        fwq = np.where(qf >= 4294967295.0, 0xFFFFFFFF, np.rint(qf)).astype(np.uint32)
    base_value = F32(b) if gradients is not None else F32(MT.base_margin_of(obj, b))
    if base_margin is not None:
        margin = np.array(np.asarray(base_margin, F32).reshape(n, T), F32)
    else:
        margin = np.full((n, T), base_value, F32)
    trees = []
    for r in range(rounds):
        if gradients is None:
            g, h, bad = MT.column_gradients(params, margin, Y, weight)
            assert not bad
        else:
            g, h = gradients(margin.copy())
        tree, leaf = grow_tree(p, cuts, bins, np.asarray(g, F32).reshape(n, T), np.asarray(h, F32).reshape(n, T), sets,
                               r, fwq)
        trees.append(tree)
        margin = (margin + leaf).astype(F32)
    return Model(trees, margin, b, base_value)


def assert_engine_matches(bst, ref, leaf_tol=1e-5):
    """the engine's vector trees against the reference's: topology, splits and loss_chg exactly, leaf vectors within
    leaf_tol"""
    trees = bst.get_trees()
    assert len(trees) == ref.num_trees
    for i, t in enumerate(trees):
        o = ref.tree(i)
        assert len(t["left"]) == o.n_nodes, "tree %d node count" % i
        for k in ("left", "right", "split_feature", "split_bin", "default_left"):
            assert np.array_equal(t[k], getattr(o, k)), "tree %d %s" % (i, k)
        inner = o.split_feature >= 0
        assert np.array_equal(t["split_cond"][inner].view(np.uint32), o.split_cond[inner].view(np.uint32)), "tree %d conds" % i
        assert np.array_equal(t["loss_chg"], o.loss_chg), "tree %d loss_chg" % i
        assert np.max(np.abs(t["leaf_vector"] - o.leaf_vector)) <= leaf_tol, "tree %d leaf vectors" % i
