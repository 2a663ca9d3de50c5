"""Reference tree growth with interaction_constraints (DESIGN.md §2 item 14).  TEST INFRASTRUCTURE ONLY.

The CPU oracle (oracle/) grows trees without constraints.  This module restates its level loop for numeric features in
NumPy, on the oracle's own primitives: cuts and bins (oracle.Cuts), gradients (oracle.gradients, or a caller's),
fixed-point quantisation (oracle.quantize), exact integer histograms (oracle.hist_int) and nested column sampling
(or_select_features).  The gain, weight, tie-break (NeedReplace), expand test, partition and 40-bit leaf refinement
follow hist_oracle.c operation for operation; with fixed-point histograms every sum is an exact multiple of the scale,
so the order of the additions does not matter.  Each node's features are then filtered by the constraint rule written
out literally: every feature at the root, elsewhere the union of every set that contains the node's whole path.  No
bitmask is involved, so the engine's compat tables are checked against an independent statement.

With no constraints this must grow exactly the oracle's trees; tests/test_interaction_constraints.py checks that
before any constrained tree is trusted.  Categorical features and row subsampling are not restated (they raise).
"""
import ctypes as C
from types import SimpleNamespace

import numpy as np

from oracle import oracle as O

F32 = np.float32
MISSING_BIN = 255
RT_EPS = F32(1e-6)
LEAF_BITS = 40
SCOPE_TREE, SCOPE_LEVEL0, SCOPE_NODE0 = 1, 16, 4096


def allowed_features(path, sets, n_features):
    """The rule as stated: every feature at the root; elsewhere the union of the sets that contain every feature of the
    path from the root (`path`, a set of feature indices)."""
    if not path:
        return set(range(n_features))
    out = set()
    for s in sets:
        if set(path) <= set(s):
            out |= set(s)
    return out


def _select(seed, tree, scope, parent, fwq, n_features, frac):
    L = O.lib()
    L.or_select_features.restype = C.c_int
    L.or_select_features.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint8), C.POINTER(C.c_uint32),
                                     C.c_int32, C.c_double, C.POINTER(C.c_uint8)]
    out = np.zeros(n_features, np.uint8)
    pp = None if parent is None else np.ascontiguousarray(parent, np.uint8).ctypes.data_as(C.POINTER(C.c_uint8))
    fp = None if fwq is None else fwq.ctypes.data_as(C.POINTER(C.c_uint32))
    L.or_select_features(seed, tree, scope, pp, fp, n_features, frac, out.ctypes.data_as(C.POINTER(C.c_uint8)))
    return out


class _P:
    """the OrParams fields the growth reads, as the C code sees them (binary32 values widened to double)"""

    def __init__(self, params, rows_sampled=False):
        """rows_sampled: the caller applies the row draw itself (tests/multi_output_reference.py), so subsample < 1 is
        accepted; here it raises"""
        p = O.make_params(params)
        self.raw = p
        self.max_depth, self.qbits, self.K = p.max_depth, p.qbits, p.num_class
        self.eta, self.gamma = F32(p.eta), F32(p.gamma)
        self.mcw, self.lam, self.alpha, self.mds = (float(F32(v)) for v in (p.min_child_weight, p.lambda_, p.alpha,
                                                                            p.max_delta_step))
        self.bytree, self.bylevel, self.bynode = (float(F32(v)) for v in (p.colsample_bytree, p.colsample_bylevel,
                                                                          p.colsample_bynode))
        self.seed, self.rank, self.subsample = p.seed, p.rank, float(F32(p.subsample))
        if p.subsample < 1.0 and not rows_sampled:
            raise NotImplementedError("row subsampling is not restated here")
        if self.qbits <= 0:
            raise NotImplementedError("only the fixed-point histograms are restated here")

    def weight(self, G, H):
        G, H = np.asarray(G, np.float64), np.asarray(H, np.float64)
        with np.errstate(all="ignore"):
            t = G if self.alpha == 0.0 else np.where(G > self.alpha, G - self.alpha, np.where(G < -self.alpha, G + self.alpha, 0.0))
            dw = -t / (H + self.lam)
            if self.mds != 0.0:
                dw = np.where(np.abs(dw) > self.mds, np.copysign(self.mds, dw), dw)
        return np.where((H < self.mcw) | (H <= 0.0), 0.0, dw)

    def gain(self, G, H):
        G, H = np.asarray(G, np.float64), np.asarray(H, np.float64)
        with np.errstate(all="ignore"):
            if self.mds == 0.0:
                t = G if self.alpha == 0.0 else np.where(G > self.alpha, G - self.alpha, np.where(G < -self.alpha, G + self.alpha, 0.0))
                r = (t * t) / (H + self.lam)
            else:
                w = self.weight(G, H)
                r = -((2.0 * G) * w + (H + self.lam) * (w * w))
                if self.alpha != 0.0:
                    r = r + self.alpha * np.abs(w)
        return np.where((H < self.mcw) | (H <= 0.0), 0.0, r)


def _first_max(chg, ok):
    """index of the first largest finite candidate > 0 among ok (NeedReplace: a later candidate must be strictly
    larger), None when there is none"""
    v = np.where(ok & np.isfinite(chg) & (chg > F32(0.0)), chg, -np.inf).astype(np.float64)
    i = int(np.argmax(v))
    return i if v[i] > -np.inf else None


def _best_split(p, cuts, ihist, sg, sh, inv_g, inv_h, feats):
    """evaluate_node for numeric features: the first candidate of the largest finite loss_chg > 0 in enumeration order
    (feature ascending; forward bins ascending, then backward bins descending)."""
    G, H = sg * inv_g, sh * inv_h
    root_gain = float(F32(p.gain(G, H)))
    best = None
    for f in sorted(feats):
        nf = int(cuts.ptrs[f + 1] - cuts.ptrs[f])
        if nf <= 0:
            continue
        hg, hh = ihist[f, :nf, 0], ihist[f, :nf, 1]
        cg, ch = np.cumsum(hg), np.cumsum(hh)
        # forward: left = bins <= i, missing -> right
        eg, eh = cg * inv_g, ch * inv_h
        rg, rh = G - eg, H - eh
        ok = (eh >= p.mcw) & (rh >= p.mcw)
        chg = ((p.gain(eg, eh) + p.gain(rg, rh)) - root_gain).astype(F32)
        i = _first_max(chg, ok)
        if i is not None and (best is None or chg[i] > best["chg"]):
            best = dict(chg=chg[i], feature=f, bin=i, cond=float(cuts.vals[cuts.ptrs[f] + i]), default_left=0,
                        lg=int(cg[i]), lh=int(ch[i]))
        if cg[-1] != sg or ch[-1] != sh:   # the node has missing values on f: backward, missing -> left
            bgi, bhi = cg[-1] - np.concatenate([[0], cg[:-1]]), ch[-1] - np.concatenate([[0], ch[:-1]])
            bg, bh = bgi * inv_g, bhi * inv_h
            lg, lh = G - bg, H - bh
            ok = (bh >= p.mcw) & (lh >= p.mcw)
            chg = ((p.gain(lg, lh) + p.gain(bg, bh)) - root_gain).astype(F32)
            j = _first_max(chg[::-1], ok[::-1])       # enumeration runs from the last bin down
            if j is not None:
                i = nf - 1 - j
                if best is None or chg[i] > best["chg"]:
                    cond = float(cuts.mins[f]) if i == 0 else float(cuts.vals[cuts.ptrs[f] + i - 1])
                    best = dict(chg=chg[i], feature=f, bin=i - 1, cond=cond, default_left=1, lg=int(sg - bgi[i]),
                                lh=int(sh - bhi[i]))
    return best


def grow_tree(p, cuts, bins, g, h, sets, tree_index, fwq=None):
    """One tree on (bins, g, h); returns (tree namespace, per-row leaf values as binary32)."""
    n, F = bins.shape
    g, h = np.ascontiguousarray(g, F32), np.ascontiguousarray(h, F32)
    qg, eg = O.quantize(g, p.qbits)
    qh, eh = O.quantize(h, p.qbits)
    inv_g, inv_h = np.ldexp(1.0, eg - p.qbits), np.ldexp(1.0, eh - p.qbits)
    kg, kh = np.ldexp(1.0, LEAF_BITS - eg), np.ldexp(1.0, LEAF_BITS - eh)
    use_cols = p.bytree < 1.0 or p.bylevel < 1.0 or p.bynode < 1.0
    mask_tree = _select(p.seed, tree_index, SCOPE_TREE, None, fwq, F, p.bytree) if use_cols else None
    t = dict(left=[], right=[], parent=[], split_feature=[], split_bin=[], split_cond=[], default_left=[], value=[],
             base_weight=[], loss_chg=[])

    def add(parent):
        for k, v in (("left", -1), ("right", -1), ("parent", parent), ("split_feature", -1), ("split_bin", -1),
                     ("split_cond", 0.0), ("default_left", 0), ("value", 0.0), ("base_weight", 0.0), ("loss_chg", 0.0)):
            t[k].append(v)
        return len(t["left"]) - 1

    out = np.zeros(n, F32)
    rows0 = np.arange(n, dtype=np.int32)
    ih = O.hist_int(bins, qg, qh, None)
    sg, sh = int(ih[0, :, 0].sum()), int(ih[0, :, 1].sum())
    root = add(-1)
    t["base_weight"][root] = F32(p.weight(sg * inv_g, sh * inv_h))
    level = [dict(nid=root, depth=0, rows=rows0, sg=sg, sh=sh, path=frozenset(), hist=ih)]
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
                split = _best_split(p, cuts, w["hist"], w["sg"], w["sh"], inv_g, inv_h, feats)
                if split is not None:
                    hl, hr = split["lh"] * inv_h, (w["sh"] - split["lh"]) * inv_h
                    if not (split["chg"] > RT_EPS and hl != 0.0 and hr != 0.0 and not (split["chg"] < p.gamma)):
                        split = None
            nid = w["nid"]
            if split is None:   # leaf: weight from the 40-bit fixed-point sums of the fp32 gradients of its rows
                r = w["rows"]
                G = float(int(np.rint(g[r].astype(np.float64) * kg).astype(np.int64).sum())) / kg
                H = float(int(np.rint(h[r].astype(np.float64) * kh).astype(np.int64).sum())) / kh
                t["base_weight"][nid] = F32(p.weight(G, H))
                lv = F32(F32(t["base_weight"][nid]) * p.eta)
                t["value"][nid] = lv
                out[r] = lv
                continue
            f = split["feature"]
            l, r_ = add(nid), add(nid)
            t["left"][nid], t["right"][nid], t["split_feature"][nid], t["split_bin"][nid] = l, r_, f, split["bin"]
            t["split_cond"][nid], t["default_left"][nid], t["loss_chg"][nid] = split["cond"], split["default_left"], split["chg"]
            t["value"][nid] = t["base_weight"][nid]
            lg, lh = split["lg"], split["lh"]
            rg, rh = w["sg"] - lg, w["sh"] - lh
            t["base_weight"][l] = F32(p.weight(lg * inv_g, lh * inv_h))
            t["base_weight"][r_] = F32(p.weight(rg * inv_g, rh * inv_h))
            b = bins[w["rows"], f]
            go_left = np.where((b == MISSING_BIN) & bool(cuts.has_missing[f]), bool(split["default_left"]), b <= split["bin"])
            path = w["path"] | {f}
            for child, rows, cg, ch in ((l, w["rows"][go_left], lg, lh), (r_, w["rows"][~go_left], rg, rh)):
                hist = O.hist_int(bins, qg, qh, rows) if w["depth"] + 1 < p.max_depth else None
                nxt.append(dict(nid=child, depth=w["depth"] + 1, rows=rows, sg=cg, sh=ch, path=path, hist=hist))
        level = nxt
    nn = len(t["left"])
    tree = SimpleNamespace(
        left=np.array(t["left"], np.int32), right=np.array(t["right"], np.int32), parent=np.array(t["parent"], np.int32),
        split_feature=np.array(t["split_feature"], np.int32), split_bin=np.array(t["split_bin"], np.int32),
        split_cond=np.array(t["split_cond"], F32), default_left=np.array(t["default_left"], np.uint8),
        value=np.array(t["value"], F32), base_weight=np.array(t["base_weight"], F32), loss_chg=np.array(t["loss_chg"], F32),
        split_type=np.zeros(nn, np.uint8), cat_bits=np.zeros((nn, 8), np.uint32), n_nodes=nn)
    return tree, out


class Model:
    """The trees of a reference run, with the oracle Booster's tree(i) / num_trees interface."""

    def __init__(self, trees, margin):
        self._trees, self.margin = trees, margin

    @property
    def num_trees(self):
        return len(self._trees)

    def tree(self, i):
        return self._trees[i]

    def trees(self):
        return list(self._trees)


def train(params, X, y, rounds, sets=None, weight=None, feature_weights=None, gradients=None):
    """`rounds` rounds on numeric X under the constraint `sets` (a list of index lists; None or [] = none).
    params needs base_score.  gradients(margin [n] or [n, K]) -> (g, h) replaces the oracle's objective (a custom
    objective; the margin then starts at params["base_score"] itself, as in the oracle's custom path)."""
    if params.get("base_score") is None:
        raise ValueError("give base_score")
    p = _P(params)
    X = np.ascontiguousarray(X, F32)
    y = np.ascontiguousarray(y, F32)
    cuts = O.Cuts.from_data(X, int(params.get("max_bin", 256)), weight=weight)
    bins = cuts.bin(X)
    n, K = X.shape[0], p.K
    fwq = None
    if feature_weights is not None:
        q = np.asarray(feature_weights, np.float64) * 65536.0
        fwq = np.where(q >= 4294967295.0, 0xFFFFFFFF, np.rint(q)).astype(np.uint32)
    margin = np.full((n, K), float(O.lib().or_base_margin(C.byref(p.raw))), F32)
    w = None if weight is None else np.ascontiguousarray(weight, F32)
    trees = []
    for _ in range(rounds):
        if gradients is None:
            g, h = O.gradients(params.get("objective", "reg:squarederror"), margin, y, w, K)
        else:
            g, h = gradients(margin[:, 0] if K == 1 else margin)
        g, h = np.asarray(g, F32).reshape(n, K), np.asarray(h, F32).reshape(n, K)
        for k in range(K):
            tree, leaf = grow_tree(p, cuts, bins, g[:, k], h[:, k], sets, len(trees), fwq)
            trees.append(tree)
            margin[:, k] = margin[:, k] + leaf
    return Model(trees, margin)
