"""NumPy restatement of the refresh updater (process_type="update", updater="refresh"; DESIGN.md 2 item 20).

Each tree is walked on the raw rows (x < cond -> left, missing -> default direction, a categorical split sends the
categories of its set right), the round's gradient pairs are quantised to 40-bit fixed point with the exponents of the
round's max |g| and |h| (tests/fixed_sums_reference.py), every node's sums are exact Python integers (a split's are its
children's), and CalcWeight / CalcGain are those of tests/interaction_reference.py::_P.  Trees are dicts in the layout of
engine.Booster.get_tree()."""
import numpy as np

from tests.fixed_sums_reference import LEAF_BITS, quant_exponent
from tests.interaction_reference import _P

F32 = np.float32


def leaf_of_rows(tree, X, missing=np.nan):
    """node id of the leaf every row of X reaches (predict's traversal on raw floats)"""
    X = np.asarray(X, F32)
    nid = np.zeros(X.shape[0], np.int64)
    st = tree.get("split_type")
    for _ in range(len(tree["left"])):
        feat = tree["split_feature"][nid]
        active = feat >= 0
        if not active.any():
            break
        rows = np.nonzero(active)[0]
        f = feat[rows]
        v = X[rows, f]
        miss = np.isnan(v) if np.isnan(missing) else (np.isnan(v) | (v == F32(missing)))
        go_left = v < tree["split_cond"][nid[rows]]
        if st is not None:
            cat = st[nid[rows]] != 0
            c = np.where((v >= 0) & (v < 256), np.nan_to_num(v, nan=0.0), 0).astype(np.int64)
            words = tree["cat_bits"][nid[rows], c >> 5]
            in_set = ((words >> (c & 31)) & 1).astype(bool) & (v >= 0) & (v < 256)
            go_left = np.where(cat, ~in_set, go_left)
        go_left = np.where(miss, tree["default_left"][nid[rows]] != 0, go_left)
        nid[rows] = np.where(go_left, tree["left"][nid[rows]], tree["right"][nid[rows]])
    return nid


def fixed(v, e):
    """rint(v * 2^(40 - e)) per row, as int64 (|q| <= 2^40)"""
    return np.rint(np.asarray(v, F32).astype(np.float64) * np.ldexp(1.0, LEAF_BITS - e)).astype(np.int64)


def node_fixed_sums(tree, leaf, qg, qh):
    """exact integer (G, H) sums of every node: a leaf's rows, a split's children added up"""
    n = len(tree["left"])
    sg, sh = [0] * n, [0] * n
    for nid in np.unique(leaf):
        sel = leaf == nid
        sg[nid], sh[nid] = int(qg[sel].sum()), int(qh[sel].sum())
    # children before parents: node ids by decreasing depth
    depth = np.zeros(n, np.int64)
    for nid in range(n):
        for c in (tree["left"][nid], tree["right"][nid]):
            if tree["split_feature"][nid] >= 0:
                depth[c] = depth[nid] + 1
    order = [0]
    for nid in order:
        if tree["split_feature"][nid] >= 0:
            order += [int(tree["left"][nid]), int(tree["right"][nid])]
    for nid in reversed(order):
        if tree["split_feature"][nid] >= 0:
            sg[nid] = sg[tree["left"][nid]] + sg[tree["right"][nid]]
            sh[nid] = sh[tree["left"][nid]] + sh[tree["right"][nid]]
    return sg, sh


def refresh_tree(tree, X, g, h, params, refresh_leaf=True, num_parallel_tree=1, missing=np.nan, eg=None, eh=None):
    """the refreshed copy of `tree` from the gradient pairs (g, h) of its class on the rows of X"""
    p = _P(dict(params, subsample=1.0))
    eg = quant_exponent(g) if eg is None else eg
    eh = quant_exponent(h) if eh is None else eh
    leaf = leaf_of_rows(tree, X, missing)
    sg, sh = node_fixed_sums(tree, leaf, fixed(g, eg), fixed(h, eh))
    kg, kh = np.ldexp(1.0, LEAF_BITS - eg), np.ldexp(1.0, LEAF_BITS - eh)
    G = np.array([float(v) / kg for v in sg])
    H = np.array([float(v) / kh for v in sh])
    w = p.weight(G, H).astype(F32)
    gain = p.gain(G, H)
    out = {k: np.array(v, copy=True) for k, v in tree.items()}
    out["sum_hess"] = H
    out["base_weight"] = w
    internal = tree["split_feature"] >= 0
    li, ri = np.where(internal, tree["left"], 0), np.where(internal, tree["right"], 0)
    out["loss_chg"] = np.where(internal, ((gain[li] + gain[ri]) - gain).astype(F32), tree["loss_chg"]).astype(F32)
    scale = F32(F32(p.eta) / F32(num_parallel_tree))
    leaf_val = (w * scale).astype(F32) if refresh_leaf else np.asarray(tree["value"], F32)
    out["value"] = np.where(internal, w, leaf_val).astype(F32)
    out["_sums"] = (sg, sh)
    return out


def refresh_model(trees, X, params, K, num_parallel_tree, base_margin, grad_fn, refresh_leaf=True, missing=np.nan):
    """Rounds in order: the gradients of round r at base_margin plus the refreshed rounds before it (grad_fn(margin) ->
    (g, h), each [n, K]); returns the refreshed trees and the final margin"""
    X = np.asarray(X, F32)
    n = X.shape[0]
    margin = np.array(base_margin, F32).reshape(n, K)
    per = K * num_parallel_tree
    out = []
    for r in range(len(trees) // per):
        g, h = grad_fn(margin.copy())
        g, h = np.asarray(g, F32).reshape(n, K), np.asarray(h, F32).reshape(n, K)
        new_round = []
        for slot in range(per):
            k = slot // num_parallel_tree
            t = refresh_tree(trees[r * per + slot], X, g[:, k], h[:, k], params, refresh_leaf, num_parallel_tree, missing)
            new_round.append((k, t))
        for k, t in new_round:
            margin[:, k] = (margin[:, k] + t["value"][leaf_of_rows(t, X, missing)]).astype(F32)
            out.append(t)
    return out, margin
