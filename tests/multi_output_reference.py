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
    node's vector holds the same formula on its qbits sums.
With T = 1 and min_child_weight = 0 this is the oracle's scalar tree (tests/test_multi_output_reference.py checks it).
Row subsampling and categorical features are not restated."""
from types import SimpleNamespace

import numpy as np

from oracle import oracle as O
from tests import multi_target_reference as MT
from tests.interaction_reference import (LEAF_BITS, MISSING_BIN, RT_EPS, SCOPE_LEVEL0, SCOPE_NODE0, SCOPE_TREE, _P,
                                         _first_max, _select, allowed_features)

F32 = np.float32


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
    """the first candidate of the largest finite loss_chg > 0 (feature ascending; forward bins ascending, backward bins
    descending); hists[k] = target k's integer histogram [F][256][2]"""
    T = len(hists)
    G = [sg[k] * inv_g[k] for k in range(T)]
    H = [sh[k] * inv_h[k] for k in range(T)]
    parent_gain = float(F32(node_gain(p, G, H)))
    best = None
    for f in sorted(feats):
        nf = int(cuts.ptrs[f + 1] - cuts.ptrs[f])
        if nf <= 0:
            continue
        cg = [np.cumsum(hists[k][f, :nf, 0]) for k in range(T)]
        ch = [np.cumsum(hists[k][f, :nf, 1]) for k in range(T)]
        # forward: left = bins <= i, missing -> right
        lg = [cg[k] * inv_g[k] for k in range(T)]
        lh = [ch[k] * inv_h[k] for k in range(T)]
        chg = ((_acc_gain(p, lg, lh) + _acc_gain(p, [G[k] - lg[k] for k in range(T)],
                                                  [H[k] - lh[k] for k in range(T)])) - parent_gain).astype(F32)
        nz_l = np.any([ch[k] != 0 for k in range(T)], axis=0)
        nz_r = np.any([(sh[k] - ch[k]) != 0 for k in range(T)], axis=0)
        i = _first_max(chg, np.ones(nf, bool))
        if i is not None and (best is None or chg[i] > best["chg"]):
            best = dict(chg=chg[i], feature=f, bin=i, cond=float(cuts.vals[cuts.ptrs[f] + i]), default_left=0,
                        nz_l=bool(nz_l[i]), nz_r=bool(nz_r[i]))
        if any(cg[k][-1] != sg[k] or ch[k][-1] != sh[k] for k in range(T)):   # backward: missing -> left
            bgi = [cg[k][-1] - np.concatenate([[0], cg[k][:-1]]) for k in range(T)]
            bhi = [ch[k][-1] - np.concatenate([[0], ch[k][:-1]]) for k in range(T)]
            rg = [bgi[k] * inv_g[k] for k in range(T)]
            rh = [bhi[k] * inv_h[k] for k in range(T)]
            chg = ((_acc_gain(p, [G[k] - rg[k] for k in range(T)], [H[k] - rh[k] for k in range(T)])
                    + _acc_gain(p, rg, rh)) - parent_gain).astype(F32)
            nz_l = np.any([(sh[k] - bhi[k]) != 0 for k in range(T)], axis=0)
            nz_r = np.any([bhi[k] != 0 for k in range(T)], axis=0)
            j = _first_max(chg[::-1], np.ones(nf, bool))
            if j is not None:
                i = nf - 1 - j
                if best is None or chg[i] > best["chg"]:
                    cond = float(cuts.mins[f]) if i == 0 else float(cuts.vals[cuts.ptrs[f] + i - 1])
                    best = dict(chg=chg[i], feature=f, bin=i - 1, cond=cond, default_left=1, nz_l=bool(nz_l[i]),
                                nz_r=bool(nz_r[i]))
    return best


def grow_tree(p, cuts, bins, g, h, sets, tree_index, fwq=None):
    """One vector-leaf tree on (bins, g [n][T], h [n][T]); returns (tree namespace, per-row leaf vectors [n][T])."""
    n, F = bins.shape
    T = g.shape[1]
    g, h = np.ascontiguousarray(g, F32), np.ascontiguousarray(h, F32)
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
    def __init__(self, trees, margin, base_score):
        self._trees, self.margin, self.base_score = trees, margin, base_score

    @property
    def num_trees(self):
        return len(self._trees)

    def tree(self, i):
        return self._trees[i]


def train(params, X, Y, rounds, weight=None, sets=None, feature_weights=None, gradients=None, base_margin=None):
    """`rounds` vector-leaf trees on numeric X with the label Y [n][T] (one of the multi-target objectives of
    tests/multi_target_reference.py), or with gradients(margin [n][T]) -> (g, h) [n][T] (a custom objective)."""
    p = _P({k: v for k, v in params.items() if k not in ("multi_strategy", "objective", "base_score")})
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
    if base_margin is not None:
        margin = np.array(np.asarray(base_margin, F32).reshape(n, T), F32)
    else:
        margin = np.full((n, T), F32(b) if gradients is not None else MT.base_margin_of(obj, b), F32)
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
    return Model(trees, margin, b)


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
