"""Wide matrices (480 to 4,300 features) against the oracle, on both sides of every boundary where a kernel layout
depends on the feature count F:

  F = 480   15 groups of 32 slots (G = ceil(F / 32)): an odd number of groups, the last histogram CTA type holds one
  F = 512   16 groups: exactly 8 group-pair CTA types, the widest tiled binning
  F = 513   17 groups: more pairs than the plan holds -> one group per histogram CTA; untiled binning
  F = 1000  F mod 8 != 0 (key extraction in batches of 8), 32 groups
  F = 2048  64 groups
  F = 4300  135 groups: one histogram stream per group on 132 SMs; split features past 4,096

Device memory: the level histograms take 2 * 2^(D-1) * G * 128 KiB at depth D, so depth 8 is used up to F = 2048
(2 GiB of histograms there) and depth 6 at F = 4300 (1.06 GiB).  With the bin matrix, the raw rows and the CUDA
context the largest case peaked at 2,650 MiB of device memory on an H100 (DESIGN.md §7)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import shap_reference as R
from tests.test_gpu_parity import LEAF_TOL, assert_same_model, run_both

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def wide_X(n, F, seed, nan_frac=0.0):
    """Uniform [0, 10) with low-cardinality columns (every 5th: 5 values) and constant columns (every 97th from 7)."""
    rng = np.random.RandomState(seed)
    X = rng.uniform(0, 10, size=(n, F)).astype(np.float32)
    X[:, 5::5] = np.floor(X[:, 5::5] / 2)
    X[:, 7::97] = 2.5
    if nan_frac > 0:
        X[rng.uniform(size=X.shape).astype(np.float32) < nan_frac] = np.nan
    return X, rng


def node_depths(t):
    sf, left, right = t["split_feature"], t["left"], t["right"]
    d = np.zeros(len(sf), np.int64)
    stack = [0]
    while stack:
        i = stack.pop()
        if sf[i] >= 0:
            d[left[i]] = d[right[i]] = d[i] + 1
            stack += [int(left[i]), int(right[i])]
    return d


def split_features(bst):
    return np.concatenate([t["split_feature"][t["split_feature"] >= 0] for t in bst.get_trees()])


# ------------------------------------------------------------------ cuts and bins (sketch.cu: tiled <= 512 < untiled)
@pytest.mark.parametrize("F,variant", [(511, "plain"), (512, "weights"), (513, "plain"), (1000, "categorical"),
                                       (4300, "plain")])
def test_cuts_and_bins_bit_exact_wide(eng, oracle, F, variant):
    n = 3000
    X, rng = wide_X(n, F, F, nan_frac=0.05)
    X[:, F - 2] = np.nan                                        # all missing
    w = rng.gamma(2.0, 1.0, size=n).astype(np.float32) if variant == "weights" else None
    is_cat, kw = None, {}
    if variant == "categorical":
        # categorical columns inside 8-column extraction batches: 0..7 holds two, 512..519 one, 992..999 the last one
        cat_cols = [2, 5, 515, 999]
        for j in cat_cols:
            X[:, j] = rng.randint(0, 7 + j % 30, size=n)
            X[rng.uniform(size=n) < 0.05, j] = np.nan
        is_cat = np.zeros(F, np.uint8); is_cat[cat_cols] = 1
        kw = {"feature_types": ["c" if c else "q" for c in is_cat], "enable_categorical": True}
    oc = oracle.Cuts.from_data(X, 256, is_cat=is_cat, weight=w)
    dm = eng.DMatrix(X, weight=w, **kw)
    dm._ensure_quantized(256, keep_raw=True)
    ptrs, vals, mins, hm = dm.get_cuts()
    assert np.array_equal(ptrs, oc.ptrs)
    assert np.array_equal(vals.view(np.uint32), oc.vals.view(np.uint32))
    assert np.array_equal(mins.view(np.uint32), oc.mins.view(np.uint32))
    assert np.array_equal(hm, oc.has_missing)
    assert np.array_equal(dm.get_bins(), oc.bin(X))
    assert hm[F - 2]                                                        # the all-missing column


# ------------------------------------------------------------------ whole trees at every boundary
TREE_CASES = [(480, "reg:squarederror", 8, False), (480, "binary:logistic", 8, False),
              (512, "reg:squarederror", 8, False), (512, "binary:logistic", 7, False),
              (513, "reg:squarederror", 8, False), (513, "binary:logistic", 7, False),
              (1000, "reg:squarederror", 7, False), (1000, "binary:logistic", 8, True),
              (2048, "reg:squarederror", 8, False), (2048, "binary:logistic", 6, True),
              (4300, "reg:squarederror", 6, False), (4300, "binary:logistic", 6, True)]


def wide_label(X, objective, rng):
    n, F = X.shape
    info = [3, F // 2 + 1, F - 1] + ([520] if F > 520 else []) + ([4100] if F > 4100 else [])
    Z = np.nan_to_num(X[:, info], nan=5.0)
    s = Z.sum(axis=1) + 2.0 * np.sin(Z[:, 0]) + 1.5 * Z[:, -1] + rng.normal(scale=0.5, size=n)
    return (s.astype(np.float32) if objective == "reg:squarederror" else (s > np.median(s)).astype(np.float32)), info


@pytest.mark.parametrize("F,objective,depth,nan_weights", TREE_CASES)
def test_trees_identical_wide(eng, oracle, F, objective, depth, nan_weights, tmp_path):
    n = 16000 if F <= 1000 else 10000 if F <= 2048 else 8000
    X, rng = wide_X(n, F, 100 + F, nan_frac=0.05 if nan_weights else 0.0)
    y, info = wide_label(X, objective, rng)
    w = rng.uniform(0.5, 2.0, size=n).astype(np.float32) if nan_weights else None
    params = {"objective": objective, "max_depth": depth, "eta": 0.3, "base_score": 0.5, "hist_qbits": 18}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 3, weight=w)
    assert_same_model(ebst, obst)
    m = ebst.predict(dm, output_margin=True, training=True)
    assert np.max(np.abs(m - obst.margin[:, 0])) <= 1e-5
    Xt, _ = wide_X(2000, F, 7 + F, nan_frac=0.05 if nan_weights else 0.0)
    pe = ebst.predict(eng.DMatrix(Xt))
    assert np.max(np.abs(pe - obst.predict(Xt))) <= 1e-5
    sf = split_features(ebst)
    assert set(info) & set(sf.tolist())
    if F > 513:
        assert (sf >= 513).any(), "no split on a feature past the pair plan"
    if F > 4096:
        assert (sf >= 4096).any(), "no split on a feature past 4,096"
        # JSON model I/O at this width: split_indices past 4,096 survive the round trip
        f = str(tmp_path / "wide.json")
        ebst.save_model(f)
        back = eng.Booster(model_file=f)
        assert np.array_equal(back.predict(eng.DMatrix(Xt)), pe)
        keys = ebst.get_fscore()
        assert any(k.startswith("f4") and len(k) == 5 for k in keys), sorted(keys)[-5:]
        assert max(int(k[1:]) for k in keys) == int(sf.max())


# ------------------------------------------------------------------ exact ties across CTAs and kernels
# Copies of one column at several positions have identical cuts, bins and histograms, so every candidate on them has
# bit-identical gain.  The oracle (XGBoost's SplitEntry::NeedReplace) keeps the lowest feature index; the device must too,
# however the copies are spread: same narrow-scan CTA (4 slots), same group, other group of the same histogram CTA type,
# other type, another narrow CTA, past 512 and past 4,096.
TIE_LAYOUTS = {
    480: dict(depth=7, num=[4, 6, 9, 40, 100, 470], nan=[20, 21, 300], cat=[50, 51, 52, 53, 54]),
    4300: dict(depth=6, num=[4, 6, 9, 40, 100, 470, 700, 4100, 4299], nan=[20, 21, 3000, 4200], cat=[50, 51, 52, 53, 4250]),
}


@pytest.mark.parametrize("F", sorted(TIE_LAYOUTS))
def test_exact_ties_pick_lowest_feature(eng, oracle, F):
    lay = TIE_LAYOUTS[F]
    n = 16000 if F < 1000 else 8000
    X, rng = wide_X(n, F, 300 + F)
    c = np.round(rng.uniform(0, 10, size=n), 1).astype(np.float32)
    d = rng.uniform(0, 10, size=n).astype(np.float32)
    d[rng.uniform(size=n) < 0.15] = np.nan                         # missing rows: ties in both default directions
    k = rng.randint(0, 12, size=n).astype(np.float32)              # 12 categories: partition splits
    for j in lay["num"]:
        X[:, j] = c
    for j in lay["nan"]:
        X[:, j] = d
    for j in lay["cat"]:
        X[:, j] = k
    y = (3.0 * (c > 5) + 0.5 * c + np.sin(1.3 * c) * 1.5 + 2.0 * (np.nan_to_num(d, nan=0.0) > 3)
         + 1.5 * (k % 4 == 1) + rng.normal(scale=0.3, size=n)).astype(np.float32)
    is_cat = np.zeros(F, np.uint8); is_cat[lay["cat"]] = 1
    params = {"objective": "reg:squarederror", "max_depth": lay["depth"], "eta": 0.3, "base_score": 0.5}
    obst, _ = oracle.train(params, X, y, 3, is_cat=is_cat)
    dm = eng.DMatrix(X, label=y, feature_types=["c" if v else "q" for v in is_cat], enable_categorical=True)
    ebst = eng.train(params, dm, num_boost_round=3, verbose_eval=False)
    assert_same_model(ebst, obst)
    used = {"num": [], "nan": [], "cat": []}
    for t in ebst.get_trees():
        dep = node_depths(t)
        for nid in np.nonzero(t["split_feature"] >= 0)[0]:
            f = int(t["split_feature"][nid])
            for kind in used:
                if f in lay[kind]:
                    assert f == lay[kind][0], "split %d (depth %d) names copy %d, not the lowest %d" % (nid, dep[nid], f, lay[kind][0])
                    used[kind].append((int(dep[nid]), int(t["default_left"][nid])))
    depths = {dd for dd, _ in used["num"]}
    assert min(depths) <= 2 and max(depths) >= 5, depths          # narrow (<= 16 nodes) and wide levels
    assert used["nan"] and used["cat"]
    assert any(dl for _, dl in used["nan"]), "no default-left split on the copies with missing values"


# ------------------------------------------------------------------ categorical features spread over every group
@pytest.mark.parametrize("extra", [{"max_cat_to_onehot": 64}, {}], ids=["onehot", "partition"])
def test_categorical_wide(eng, oracle, extra):
    F, n = 600, 12000
    X, rng = wide_X(n, F, 77, nan_frac=0.03)
    cat_cols = list(range(3, F, 4))                               # 150 categorical columns, in each of the 19 groups
    for j in cat_cols:
        X[:, j] = rng.randint(0, 3 + j % 37, size=n)
        X[rng.uniform(size=n) < 0.03, j] = np.nan
    Z = np.nan_to_num(X, nan=1.0)
    y = ((Z[:, 0] > 5) * 1.0 + (Z[:, 303] % 3 == 0) * 2.0 + (Z[:, 599] % 5 < 2) * 1.5 + (Z[:, 3] == 1) * 1.0
         + (Z[:, 598] > 4) * 0.7 + rng.normal(scale=0.3, size=n)).astype(np.float32)
    is_cat = np.zeros(F, np.uint8); is_cat[cat_cols] = 1
    params = dict({"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5}, **extra)
    obst, _ = oracle.train(params, X, y, 3, is_cat=is_cat)
    dm = eng.DMatrix(X, label=y, feature_types=["c" if v else "q" for v in is_cat], enable_categorical=True)
    ebst = eng.train(params, dm, num_boost_round=3, verbose_eval=False)
    assert_same_model(ebst, obst)
    cat_split = np.concatenate([t["split_feature"][(t["split_feature"] >= 0) & (t["split_type"] == 1)] for t in ebst.get_trees()])
    assert (cat_split >= 513).any() and (cat_split < 32).any()
    assert np.max(np.abs(ebst.predict(dm, output_margin=True) - obst.predict(X, output_margin=True))) <= LEAF_TOL


# ------------------------------------------------------------------ column sampling at width
def _select(oracle, seed, tree, scope, parent, fwq, F, frac):
    L = oracle.lib()
    L.or_select_features.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_int32, C.c_double,
                                     C.c_void_p]
    out = np.zeros(F, np.uint8)
    L.or_select_features(seed, tree, scope, None if parent is None else parent.ctypes.data, fwq.ctypes.data, F, frac,
                         out.ctypes.data)
    return out


def test_column_sampling_wide(eng, oracle):
    F, n, depth, seed = 2048, 10000, 7, 4242
    X, rng = wide_X(n, F, 55, nan_frac=0.02)
    fw = rng.randint(1, 5, size=F).astype(np.float32)
    fw[rng.uniform(size=F) < 0.2] = 0.0                           # zero weights sort last
    Z = np.nan_to_num(X, nan=5.0)
    y = (Z[:, ::64].sum(axis=1) + Z[:, 2000] * 2 + rng.normal(size=n)).astype(np.float32)
    params = {"objective": "reg:squarederror", "max_depth": depth, "eta": 0.3, "base_score": 0.5, "seed": seed,
              "colsample_bytree": 0.7, "colsample_bylevel": 0.6, "colsample_bynode": 0.5}
    dm = eng.DMatrix(X, label=y)
    dm.set_info(feature_weights=fw)
    ebst = eng.train(params, dm, num_boost_round=3, verbose_eval=False)
    obst, _ = oracle.train(params, X, y, 3, feature_weights=fw)
    assert_same_model(ebst, obst)
    fwq = np.rint(fw.astype(np.float64) * 65536.0).astype(np.uint32)
    for ti, t in enumerate(ebst.get_trees()):
        tree_mask = _select(oracle, seed, ti, 1, None, fwq, F, 0.7)
        assert tree_mask.sum() == int(0.7 * F) and not (tree_mask & (fw == 0)).any()
        dep = node_depths(t)
        for nid in np.nonzero(t["split_feature"] >= 0)[0]:
            level = _select(oracle, seed, ti, 16 + int(dep[nid]), tree_mask, fwq, F, 0.6)
            assert level[t["split_feature"][nid]], "tree %d node %d splits on feature %d outside its level's mask" % (
                ti, nid, t["split_feature"][nid])
    assert (split_features(ebst) >= 1024).any()


# ------------------------------------------------------------------ prediction paths
def _base_value(bst):
    bs = float(bst.params.get("base_score", 0.5))
    return float(-np.log(1.0 / bs - 1.0)) if bst.params.get("objective") == "binary:logistic" else bs


def test_predict_leaf_and_contribs_wide(eng, oracle):
    F, n = 2048, 8000
    X, rng = wide_X(n, F, 91, nan_frac=0.03)
    y, _ = wide_label(X, "binary:logistic", rng)
    params = {"objective": "binary:logistic", "max_depth": 6, "eta": 0.3, "base_score": 0.5}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 3)
    assert_same_model(ebst, obst)
    xs = X[:300]
    d = eng.DMatrix(xs)
    assert np.max(np.abs(ebst.predict(d) - obst.predict(xs))) <= 1e-5
    trees = ebst.get_trees()
    assert np.array_equal(ebst.predict(d, pred_leaf=True), R.leaf_index(trees, xs))
    phi = ebst.predict(d, pred_contribs=True, strict_shape=True)
    ref = R.shap_contribs(trees, xs, base_value=_base_value(ebst))
    margin = ebst.predict(d, output_margin=True).reshape(len(xs), 1)
    tol = 1e-5 * np.maximum(1.0, np.abs(margin))[:, :, None]
    assert phi.shape == (len(xs), 1, F + 1)
    assert np.all(np.abs(phi - ref) <= tol), float(np.max(np.abs(phi - ref)))
    assert (np.abs(phi[:, 0, 513:F]) > 0).any()                  # attributions reach the far columns


def test_interactions_wide(eng):
    F, n = 600, 4000
    X, rng = wide_X(n, F, 92, nan_frac=0.03)
    y, _ = wide_label(X, "reg:squarederror", rng)
    bst = eng.train({"objective": "reg:squarederror", "max_depth": 5, "eta": 0.3, "base_score": 0.5},
                    eng.DMatrix(X, label=y), num_boost_round=2, verbose_eval=False)
    xs = X[:16]
    d = eng.DMatrix(xs)
    inter = bst.predict(d, pred_interactions=True, strict_shape=True)
    ref = R.shap_contribs(bst.get_trees(), xs, interactions=True, base_value=_base_value(bst))
    margin = bst.predict(d, output_margin=True).reshape(len(xs), 1)
    tol = 1e-5 * np.maximum(1.0, np.abs(margin))[:, :, None, None]
    assert inter.shape == (len(xs), 1, F + 1, F + 1)
    assert np.all(np.abs(inter - ref) <= tol), float(np.max(np.abs(inter - ref)))
    assert (split_features(bst) >= 513).any()


# ------------------------------------------------------------------ histogram kernel variants through training
VARIANT_CODE = r"""
import sys, numpy as np
sys.path.insert(0, %(root)r)
from xgboost_ray_b200 import engine as E
d = np.load(%(data)r)
for F in %(widths)r:
    X, y = d["X%%d" %% F], d["y%%d" %% F]
    bst = E.train(%(params)r, E.DMatrix(X, label=y), num_boost_round=3, verbose_eval=False)
    np.savez(%(out)r %% F, **{"%%d_%%s" %% (i, k): v for i, t in enumerate(bst.get_trees()) for k, v in t.items()})
print("variant ok")
"""


class _Saved:
    def __init__(self, path):
        z = np.load(path)
        n = 1 + max(int(k.split("_", 1)[0]) for k in z.files)
        self.trees = [{k.split("_", 1)[1]: z[k] for k in z.files if int(k.split("_", 1)[0]) == i} for i in range(n)]

    def get_trees(self):
        return self.trees


def test_hist_variants_through_training(oracle, tmp_path):
    """The one-group-per-CTA kernels (256 / 512 threads), the two-groups-per-CTA kernel at an even (F = 1000) and an
    odd (F = 990) group count and the TMA-staged root level all train the oracle's trees at these widths."""
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5}
    widths = (1000, 990)
    arrays, ref = {}, {}
    for F in widths:
        X, rng = wide_X(12000, F, 400 + F, nan_frac=0.02)
        y, _ = wide_label(X, "reg:squarederror", rng)
        arrays["X%d" % F], arrays["y%d" % F] = X, y
        ref[F], _ = oracle.train(params, X, y, 3)
    data = str(tmp_path / "data.npz")
    np.savez(data, **arrays)
    for env in ({"B2_HIST_VARIANT": "0"}, {"B2_HIST_VARIANT": "1"}, {"B2_HIST_VARIANT": "2"}, {"B2_HIST_TMA": "1"}):
        tag = "_".join("%s%s" % kv for kv in env.items())
        out = str(tmp_path / (tag + "_%d.npz"))
        code = VARIANT_CODE % {"root": ROOT, "data": data, "widths": widths, "params": params, "out": out}
        r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0 and "variant ok" in r.stdout, (env, r.stdout[-500:], r.stderr[-1500:])
        for F in widths:
            assert_same_model(_Saved(out % F), ref[F])


# ------------------------------------------------------------------ two GPUs: feature-slot sharding at width
@pytest.mark.timeout(600)
@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_two_gpu_wide_identical(eng, oracle, exchange, monkeypatch):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import xgboost_ray_b200.main as M
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    M.shutdown_actors()                       # the exchange kind is read by the actor processes when they start
    if exchange == "nccl":
        monkeypatch.setenv("B2_EXCHANGE", "nccl")
    else:
        monkeypatch.delenv("B2_EXCHANGE", raising=False)
    F, n = 1000, 20001
    X, rng = wide_X(n, F, 500, nan_frac=0.03)
    y, _ = wide_label(X, "reg:squarederror", rng)
    params = {"objective": "reg:squarederror", "max_depth": 7, "eta": 0.3, "base_score": 0.5}
    b1 = train(params, RayDMatrix(X, y), num_boost_round=3, ray_params=RayParams(num_actors=1))
    b2 = train(params, RayDMatrix(X, y), num_boost_round=3, ray_params=RayParams(num_actors=2))
    assert b1.get_dump(dump_format="json", with_stats=True) == b2.get_dump(dump_format="json", with_stats=True)
    ob, _ = oracle.train(params, X, y, 3)
    for i, t in enumerate(b2.get_trees()):
        o = ob.tree(i)
        assert np.array_equal(t["split_feature"], o.split_feature) and np.array_equal(t["split_bin"], o.split_bin)
        leaf = o.split_feature < 0
        assert np.max(np.abs(t["value"][leaf] - o.value[leaf])) <= LEAF_TOL
    M.shutdown_actors()
