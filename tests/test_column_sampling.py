"""Column-sampling selection (xgboost_ray_b200/csrc/sampling.cuh) on the CPU.

The host draws the tree and level masks with b2_col_select: each feature's key once, one sort by (key, f).  The
split scan asks b2_col_selected per feature (rank among F keys), and the oracle's select_features ranks precomputed
keys.  All three must pick the same set for every seed, tree, scope, fraction, parent mask and weight vector:
identical models depend on it.  The header is compiled here with the host C compiler."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "xgboost_ray_b200", "csrc")

SHIM = r"""
#include <stdlib.h>
#include "sampling.cuh"
static int n_parent(const uint8_t* parent, int F) {
  int n = 0;
  for (int f = 0; f < F; ++f) n += (!parent || parent[f]) ? 1 : 0;
  return n;
}
int sel_sorted(uint32_t seed, uint32_t tree, uint32_t scope, const uint8_t* parent, const uint32_t* wq, int F, double frac,
               uint8_t* out) {
  B2ColRank* scratch = (B2ColRank*)malloc((size_t)(F > 0 ? F : 1) * sizeof(B2ColRank));
  const int n = b2_col_select(seed, tree, scope, parent, wq, F, b2_sample_count(frac, n_parent(parent, F)), scratch, out);
  free(scratch);
  return n;
}
int sel_per_feature(uint32_t seed, uint32_t tree, uint32_t scope, const uint8_t* parent, const uint32_t* wq, int F,
                    double frac, uint8_t* out) {
  const int n_sel = b2_sample_count(frac, n_parent(parent, F));
  int n = 0;
  for (int f = 0; f < F; ++f) { out[f] = b2_col_selected(seed, tree, scope, f, parent, wq, F, n_sel) ? 1 : 0; n += out[f]; }
  return n;
}
"""


@pytest.fixture(scope="module")
def sel(tmp_path_factory, oracle):
    d = tmp_path_factory.mktemp("sampling")
    src, so = str(d / "shim.c"), str(d / "libsel.so")
    with open(src, "w") as fh:
        fh.write(SHIM)
    subprocess.check_call(["/usr/bin/gcc", "-O2", "-fPIC", "-shared", "-std=c11", "-Wall", "-Werror", "-I", CSRC, "-o", so, src])
    L = C.CDLL(so)
    args = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_int32, C.c_double, C.c_void_p]
    O = oracle.lib()
    for fn in (L.sel_sorted, L.sel_per_feature, O.or_select_features):
        fn.argtypes = args
        fn.restype = C.c_int32

    def run(fn, seed, tree, scope, parent, wq, F, frac):
        out = np.full(F, 7, np.uint8)
        p = None if parent is None else np.ascontiguousarray(parent, np.uint8)
        w = None if wq is None else np.ascontiguousarray(wq, np.uint32)
        n = fn(seed, tree, scope, None if p is None else p.ctypes.data, None if w is None else w.ctypes.data, F, frac,
               out.ctypes.data)
        assert int(out.sum()) == n and set(np.unique(out)) <= {0, 1}
        return out
    return {"sorted": lambda *a: run(L.sel_sorted, *a), "per_feature": lambda *a: run(L.sel_per_feature, *a),
            "oracle": lambda *a: run(O.or_select_features, *a)}


SCOPE_TREE, SCOPE_LEVEL0, SCOPE_NODE0 = 1, 16, 4096


def _weights(kind, F, rng):
    if kind == "none":
        return None
    if kind == "equal":                     # every key tie is broken by the feature index alone
        return np.full(F, 3 << 16, np.uint32)
    if kind == "zeros":                     # zero weights sort last, in index order
        w = rng.randint(1, 1 << 20, size=F).astype(np.uint32)
        w[rng.uniform(size=F) < 0.4] = 0
        return w
    if kind == "all_zero":
        return np.zeros(F, np.uint32)
    w = rng.randint(0, 4, size=F).astype(np.uint32) << 16   # few distinct weights, zeros among them
    return w


def _parent(kind, F, rng):
    if kind == "none":
        return None
    if kind == "half":
        return (rng.uniform(size=F) < 0.5).astype(np.uint8)
    if kind == "one":
        p = np.zeros(F, np.uint8); p[rng.randint(F)] = 1
        return p
    return np.zeros(F, np.uint8)            # empty parent set: nothing can be selected


@pytest.mark.parametrize("F", [1, 2, 3, 7, 31, 32, 33, 100, 480, 511, 512, 513, 1000, 2048])
def test_sorted_selection_equals_per_feature_and_oracle(sel, F):
    rng = np.random.RandomState(F)
    for i, (wk, pk) in enumerate([(w, p) for w in ("none", "equal", "zeros", "all_zero", "coarse")
                                  for p in ("none", "half", "one", "empty")]):
        wq, parent = _weights(wk, F, rng), _parent(pk, F, rng)
        for frac in ((0.01, 0.3, 0.5, 0.999, 1.0) if F <= 512 else (0.3, 0.999)):   # F^2 per-feature cost
            seed, tree = int(rng.randint(0, 1 << 31)), int(rng.randint(0, 5000))
            scope = (SCOPE_TREE, SCOPE_LEVEL0 + i % 14, SCOPE_NODE0 + int(rng.randint(0, 1 << 14)))[i % 3]
            a = sel["sorted"](seed, tree, scope, parent, wq, F, frac)
            b = sel["per_feature"](seed, tree, scope, parent, wq, F, frac)
            c = sel["oracle"](seed, tree, scope, parent, wq, F, frac)
            ctx = (F, wk, pk, frac, seed, tree, scope)
            assert np.array_equal(a, b), ctx
            assert np.array_equal(a, c), ctx
            n_par = F if parent is None else int(parent.sum())
            assert a.sum() == min(max(1, int(frac * n_par)), n_par), ctx
            if parent is not None:
                assert not (a & (parent == 0)).any(), ctx
            if wq is not None and a.sum():         # a zero-weight feature only once every weighted one is in
                cand = np.ones(F, bool) if parent is None else parent.astype(bool)
                if (a.astype(bool) & (wq == 0)).any():
                    assert (a.astype(bool) | ~cand | (wq == 0)).all(), ctx
                    zero_sel = np.nonzero(a.astype(bool) & (wq == 0))[0]
                    zero_cand = np.nonzero(cand & (wq == 0))[0]
                    assert np.array_equal(zero_sel, zero_cand[:len(zero_sel)]), ctx   # lowest indices first


@pytest.mark.parametrize("F", [4096, 5000])
def test_sorted_selection_wide(sel, F):
    """The widest masks, nested tree -> level as the engine draws them, against both references."""
    rng = np.random.RandomState(F + 1)
    wq = _weights("zeros", F, rng)
    for wv in (None, wq):
        tree_mask = sel["sorted"](99, 7, SCOPE_TREE, None, wv, F, 0.5)
        assert np.array_equal(tree_mask, sel["oracle"](99, 7, SCOPE_TREE, None, wv, F, 0.5))
        level = sel["sorted"](99, 7, SCOPE_LEVEL0 + 3, tree_mask, wv, F, 0.7)
        assert np.array_equal(level, sel["oracle"](99, 7, SCOPE_LEVEL0 + 3, tree_mask, wv, F, 0.7))
        assert level.sum() == int(0.7 * tree_mask.sum())
    # the per-feature form is F^2 key evaluations: one mask at this width is enough
    assert np.array_equal(sel["sorted"](5, 1, SCOPE_TREE, None, wq, F, 0.25), sel["per_feature"](5, 1, SCOPE_TREE, None, wq, F, 0.25))


def test_equal_keys_break_ties_by_index(sel):
    """All weights zero: every key is the same, so the n lowest feature indices of the parent set are chosen."""
    F = 300
    rng = np.random.RandomState(3)
    parent = (rng.uniform(size=F) < 0.6).astype(np.uint8)
    out = sel["sorted"](1, 2, SCOPE_TREE, parent, np.zeros(F, np.uint32), F, 0.25)
    idx = np.nonzero(parent)[0]
    want = np.zeros(F, np.uint8); want[idx[:int(0.25 * len(idx))]] = 1
    assert np.array_equal(out, want)
