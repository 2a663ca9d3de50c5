"""The value domain on the H100: cuts, bins, trees and every raw-value prediction path at the edges of binary32 (+-inf,
+-FLT_MAX, subnormals, signed zeros, 1-ulp neighbours, values exactly on a split condition) and with a non-NaN
`missing`, against the CPU oracle, tests/shap_reference.py and exact known answers.  Training routes rows by bin,
prediction / leaf indices / SHAP / metrics by raw float (x < cond): the tests check that the two routes agree where
they are most likely not to.  The CPU half is tests/test_oracle_value_domain.py."""
import pickle

import numpy as np
import pytest

from tests import dart_reference as D
from tests import shap_reference as R
from tests.test_gpu_parity import assert_same_model

pytestmark = pytest.mark.gpu

F = np.float32
FLT_MAX = np.finfo(F).max
N = 70001                     # a multiple of neither the 64-row bin tile nor the 8-column extract batch
MISSINGS = [np.nan, 0.0, -999.0, np.inf]
MISSING_IDS = ["nan", "zero", "m999", "inf"]


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def _sprinkle(rng, col, values, frac):
    sel = rng.uniform(size=col.size) < frac
    col[sel] = rng.choice(np.asarray(values, F), size=int(sel.sum()))
    return col


def adversarial_block(n, seed, missing):
    """13 columns: +-inf among finite values, +-FLT_MAX, subnormals of both signs, mixed signed zeros, 1-ulp neighbours
    of 1.0, integers past 2^24, 255 / 256 / 257 distinct values, all-missing, only-sentinel missing, NaN holes, and a
    column holding the literal values 0, -0, -999 and +-inf (missing or not, depending on the sentinel)"""
    rng = np.random.RandomState(seed)
    u = lambda lo, hi: rng.uniform(lo, hi, size=n).astype(F)      # noqa: E731
    c0 = _sprinkle(rng, u(-5, 5), [np.inf, -np.inf], 0.05)
    c1 = _sprinkle(rng, u(-5, 5), [FLT_MAX, -FLT_MAX, np.nextafter(FLT_MAX, F(0))], 0.05)
    sub = rng.randint(1, 1 << 23, size=n).astype(np.uint32) | (rng.randint(0, 2, size=n).astype(np.uint32) << 31)
    c2 = _sprinkle(rng, sub.view(F).copy(), [0.0, -0.0], 0.2)
    c3 = rng.choice(np.array([-0.0, 0.0, 1.0, -1.0, 2.0], F), size=n)
    c4 = (np.uint32(0x3f800000) + rng.randint(-64, 65, size=n).astype(np.int64)).astype(np.uint32).view(F)
    c5 = (rng.randint(0, 1 << 26, size=n).astype(np.float64) + 2.0 ** 24).astype(F)
    bounds = []
    for m in (255, 256, 257):
        vals = (np.arange(m) * 0.5 - 30).astype(F)
        c = rng.choice(vals, size=n)
        c[:m] = vals
        bounds.append(c)
    c9 = np.full(n, np.nan, F)
    c10 = u(0, 10)
    c10[rng.uniform(size=n) < 0.07] = F(missing)
    c11 = u(0, 10)
    c11[rng.uniform(size=n) < 0.1] = np.nan
    c12 = _sprinkle(rng, rng.normal(size=n).astype(F), [0.0, -0.0, -999.0, np.inf, -np.inf], 0.1)
    return np.stack([c0, c1, c2, c3, c4, c5] + bounds + [c9, c10, c11, c12], axis=1).astype(F)


def adversarial(f, missing, n=N):
    assert f % 13 == 0
    return np.concatenate([adversarial_block(n, 17 + b, missing) for b in range(f // 13)], axis=1)


def labels(X, objective, seed=0):
    rng = np.random.RandomState(seed)
    c = lambda j: np.nan_to_num(np.clip(X[:, j].astype(np.float64), -6, 6))      # noqa: E731
    y = c(0) + (X[:, 3] > 0) + 0.5 * c(11) + np.sin(c(6)) + 0.3 * (X[:, 12] == 0) + rng.normal(scale=0.3, size=len(X))
    return (y > np.median(y)).astype(F) if objective == "binary:logistic" else y.astype(F)


def weights(X):
    w = np.random.RandomState(9).uniform(0.25, 4.0, size=len(X)).astype(F)
    extreme = (np.abs(X[:, 0]) == np.inf) | (np.abs(X[:, 1]) >= FLT_MAX / 2)
    w[extreme] = 0.0                                              # zero weights on the extremes
    return w


def assert_cuts_equal(dm, oc, X, missing):
    ptrs, vals, mins, hm = dm.get_cuts()
    assert np.array_equal(ptrs, oc.ptrs)
    assert np.array_equal(vals.view(np.uint32), oc.vals.view(np.uint32))
    assert np.array_equal(mins.view(np.uint32), oc.mins.view(np.uint32))
    assert np.array_equal(hm, oc.has_missing)
    assert np.array_equal(dm.get_bins(), oc.bin(X, missing))


# ------------------------------------------------------------------ cuts and bins
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("missing", MISSINGS, ids=MISSING_IDS)
@pytest.mark.parametrize("f", [13, 520])           # bin_tiled_kernel / bin_kernel
def test_cuts_and_bins_bit_exact(eng, oracle, f, missing, weighted):
    X = adversarial(f, missing)
    w = weights(X) if weighted else None
    oc = oracle.Cuts.from_data(X, 256, missing, weight=w)
    dm = eng.DMatrix(X, weight=w, missing=missing)
    dm._ensure_quantized(256, keep_raw=True)
    assert_cuts_equal(dm, oc, X, missing)
    assert oc.has_missing[9] and oc.has_missing[10] and oc.ptrs[10] - oc.ptrs[9] == 1


def test_weighted_rank_sums_past_2_pow_53(eng, oracle):
    """9M rows, most of them weighted near the largest quantised weight 2^30: the rank sums rmin + rmax that the prune
    compares in double pass 2^53, and some of them are rounded there.  Both sides must round them alike."""
    rng = np.random.RandomState(4)
    n = 9_000_000
    X = rng.randint(0, 5000, size=(n, 1)).astype(F)
    X[rng.uniform(size=n) < 0.01, 0] = np.nan
    # max w < 2, so wq = rint(w * 2^29).  A weight in [1, 2) quantises to a multiple of 64, which alone keeps every
    # sum exact in double; a tenth of the rows get odd quantised weights (odd * 2^-29), so the sums have odd bits
    w = rng.uniform(1.0, 2.0, size=n).astype(F)
    small = rng.uniform(size=n) < 0.1
    w[small] = (2 * rng.randint(0, 500, size=int(small.sum())) + 1).astype(np.float64) * 2.0 ** -29
    ok = ~np.isnan(X[:, 0])
    wq = np.rint(w[ok].astype(np.float64) * 2.0 ** 29).astype(np.int64)
    assert np.array_equal(wq.astype(np.float64), w[ok].astype(np.float64) * 2.0 ** 29)
    _, inv = np.unique(X[ok, 0], return_inverse=True)
    rmin = np.concatenate([[0], np.cumsum(np.bincount(inv, weights=wq))[:-1].astype(np.int64)])
    S = rmin + np.append(rmin[1:], wq.sum())                       # exact int64 rmin + rmax of every distinct value
    rounded = (S > 2 ** 53) & (S.astype(np.float64).astype(np.int64) != S)
    assert rounded.sum() > 100, int(rounded.sum())
    oc = oracle.Cuts.from_data(X, 256, weight=w)
    dm = eng.DMatrix(X, weight=w)
    dm._ensure_quantized(256, keep_raw=True)
    assert_cuts_equal(dm, oc, X, np.nan)


# ------------------------------------------------------------------ trees, and the training route against the raw route
def _train_both(eng, oracle, params, X, y, missing, rounds=3, **dm_kw):
    obst, _ = oracle.train(params, X, y, rounds, missing=missing, is_cat=dm_kw.pop("is_cat", None))
    dm = eng.DMatrix(X, label=y, missing=missing, **dm_kw)
    return eng.train(params, dm, num_boost_round=rounds, verbose_eval=False), obst, dm


def assert_routes_agree(eng, bst, dm, X, missing, **dm_kw):
    """the train margin (rows routed by bin while the trees grew) equals predict() on the raw floats, bit for bit"""
    train_margin = bst.predict(dm, output_margin=True, training=True)
    raw_margin = bst.predict(eng.DMatrix(X, missing=missing, **dm_kw), output_margin=True)
    assert np.array_equal(train_margin, raw_margin), float(np.max(np.abs(train_margin - raw_margin)))
    return raw_margin


@pytest.mark.parametrize("objective", ["reg:squarederror", "binary:logistic"])
@pytest.mark.parametrize("missing", MISSINGS, ids=MISSING_IDS)
def test_trees_identical_and_routes_agree(eng, oracle, missing, objective):
    X = adversarial(13, missing)
    y = labels(X, objective)
    params = {"objective": objective, "max_depth": 6, "eta": 0.3, "base_score": 0.5}
    bst, obst, dm = _train_both(eng, oracle, params, X, y, missing)
    assert_same_model(bst, obst)
    margin = assert_routes_agree(eng, bst, dm, X, missing)
    assert np.max(np.abs(margin - obst.predict_margin(X, missing)[:, 0])) <= 1e-5


def inf_split_case(n=20000, seed=3):
    """a column 0..19 with 19 replaced by FLT_MAX, a tenth NaN, label 5 * isnan(x): the root sends every real bin left
    and the missing rows right, so its condition is the last cut, FLT_MAX + FLT_MAX = +inf"""
    rng = np.random.RandomState(seed)
    x = rng.randint(0, 20, size=n).astype(F)
    x[x == 19] = FLT_MAX
    x[rng.uniform(size=n) < 0.1] = np.nan
    X = np.stack([x, rng.uniform(0, 10, size=n).astype(F), rng.normal(size=n).astype(F)], axis=1)
    y = (5.0 * np.isnan(x) + 0.3 * X[:, 1] + rng.normal(scale=0.1, size=n)).astype(F)
    return X, y


def test_inf_condition_grown_like_the_oracle(eng, oracle):
    X, y = inf_split_case()
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5}
    bst, obst, dm = _train_both(eng, oracle, params, X, y, np.nan)
    assert_same_model(bst, obst)
    t0 = bst.get_trees()[0]
    assert t0["split_feature"][0] == 0 and np.isposinf(t0["split_cond"][0]) and t0["default_left"][0] == 0
    assert_routes_agree(eng, bst, dm, X, np.nan)


def cat_case(missing=-999.0, n=30011, seed=6):
    rng = np.random.RandomState(seed)
    X = rng.uniform(0, 10, size=(n, 5)).astype(F)
    X[:, 3] = rng.randint(0, 21, size=n)
    X[:, 4] = rng.randint(0, 6, size=n)
    X[rng.uniform(size=n) < 0.1, 3] = F(missing)
    X[rng.uniform(size=n) < 0.05, 4] = F(missing)
    X[rng.uniform(size=n) < 0.05, 0] = F(missing)
    c3 = np.where(X[:, 3] == F(missing), 7, X[:, 3])
    y = (X[:, 1] + np.isin(c3, [2, 3, 5, 7, 11, 13, 17, 19]) * 3 + (X[:, 4] == 2) * 2
         + rng.normal(scale=0.2, size=n)).astype(F)
    kw = {"feature_types": ["q", "q", "q", "c", "c"], "enable_categorical": True}
    return X, y, kw, np.array([0, 0, 0, 1, 1], np.uint8)


@pytest.mark.parametrize("onehot", [4, 64])
def test_categorical_with_sentinel_identical(eng, oracle, onehot):
    X, y, kw, is_cat = cat_case()
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5, "max_cat_to_onehot": onehot}
    bst, obst, dm = _train_both(eng, oracle, params, X, y, -999.0, is_cat=is_cat, **kw)
    assert_same_model(bst, obst)
    assert any(t["split_type"].any() for t in bst.get_trees())
    assert_routes_agree(eng, bst, dm, X, -999.0, **kw)


def test_dart_routes_agree_and_pickled_inf_model_continues(eng):
    X, y = inf_split_case()
    params = {"objective": "reg:squarederror", "max_depth": 5, "eta": 0.3, "base_score": 0.5, "booster": "dart",
              "rate_drop": 0.4, "skip_drop": 0.0, "seed": 3}
    dm = eng.DMatrix(X, label=y)
    bst = eng.train(params, dm, num_boost_round=5, verbose_eval=False)
    trees, w = bst.get_trees(), bst.get_tree_weights()
    assert np.isposinf(trees[0]["split_cond"][0])
    # predict(training=True) of DART is the margin of the next round's drop set, which dart_margins_kernel rebuilds
    # from the bins: it equals the reference walk of the same bins, and every tree's bin route equals its raw route
    bins, hm = dm.get_bins(), dm.get_cuts()[3]
    nxt = D.drop_set(w, 5, seed=3, rate_drop=0.4, skip_drop=0.0)
    want = D.margins(trees, w, bins, hm, np.full((len(X), 1), 0.5, F), skip=nxt)
    assert bst.predict(dm, output_margin=True, training=True).tobytes() == want.reshape(-1).tobytes()
    raw_leaf = bst.predict(eng.DMatrix(X), pred_leaf=True)
    for j, t in enumerate(trees):
        assert np.array_equal(D.leaves_on_bins(t, bins, hm), raw_leaf[:, j]), j
    b2 = pickle.loads(pickle.dumps(bst))
    assert np.isposinf(b2.get_trees()[0]["split_cond"][0])
    more = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=2, xgb_model=b2, verbose_eval=False)
    assert more.num_boosted_rounds() == 7
    for a, b in zip(bst.get_trees(), more.get_trees()[:5]):
        assert np.array_equal(a["split_cond"].view(np.uint32), b["split_cond"].view(np.uint32))


def test_borrowed_numeric_cuts_route_alike(eng, oracle):
    rng = np.random.RandomState(8)
    X1 = rng.uniform(0, 10, size=(20000, 4)).astype(F)              # no missing values: has_missing = 0
    X2 = rng.uniform(-5, 15, size=(30011, 4)).astype(F)             # beyond the borrowed range, with NaN
    X2[rng.uniform(size=X2.shape) < 0.1] = np.nan
    y = (np.nan_to_num(X2[:, 0], nan=20) + np.nan_to_num(X2[:, 1]) * 0.5 + rng.normal(size=len(X2))).astype(F)
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5}
    d1 = eng.DMatrix(X1)
    dm = eng.DMatrix(X2, label=y, ref=d1)
    bst = eng.train(params, dm, num_boost_round=3, verbose_eval=False)
    obst, _ = oracle.train(params, X2, y, 3, cuts=oracle.Cuts.from_data(X1, 256))
    assert_same_model(bst, obst)
    assert_routes_agree(eng, bst, dm, X2, np.nan)


# ------------------------------------------------------------------ probe rows from the model's own nodes
CAT_PROBES = [-1.0, -0.0, 2.5, 254.9, 255.0, 256.0, 1e9, np.inf, -np.inf, np.nan]


def probe_rows(trees, X, missing, seed=0, max_trees=3):
    rng = np.random.RandomState(seed)
    rows = []
    for t in trees[:max_trees]:
        for nid in np.nonzero(t["split_feature"] >= 0)[0]:
            f = int(t["split_feature"][nid])
            if t["split_type"][nid]:
                cats = [b for b in range(256) if (int(t["cat_bits"][nid][b >> 5]) >> (b & 31)) & 1]
                vals = cats[:3] + [c for c in range(8) if c not in cats][:3] + CAT_PROBES + [missing]
            else:
                c = F(t["split_cond"][nid])
                vals = [c, np.nextafter(c, F(-np.inf)), np.nextafter(c, F(np.inf)), np.inf, -np.inf, np.nan, missing]
                if c == 0:
                    vals.append(-0.0)
            for v in vals:
                r = X[rng.randint(len(X))].copy()
                r[f] = F(v)
                rows.append(r)
    return np.asarray(rows, F)


def _base_value(bst):
    bs = float(bst.params.get("base_score", 0.5))
    return float(-np.log(1.0 / bs - 1.0)) if bst.params.get("objective") == "binary:logistic" else bs


def _probe_model(eng, oracle, case):
    if case == "inf_cond":
        X, y = inf_split_case()
        return _train_both(eng, oracle, {"objective": "reg:squarederror", "max_depth": 6, "base_score": 0.5}, X, y,
                           np.nan) + (X, np.nan, {})
    if case == "sentinel":
        X = adversarial(13, -999.0, n=20011)
        y = labels(X, "binary:logistic")
        return _train_both(eng, oracle, {"objective": "binary:logistic", "max_depth": 6, "base_score": 0.5}, X, y,
                           -999.0) + (X, -999.0, {})
    X, y, kw, is_cat = cat_case()
    return _train_both(eng, oracle, {"objective": "reg:squarederror", "max_depth": 6, "base_score": 0.5}, X, y,
                       -999.0, is_cat=is_cat, **kw) + (X, -999.0, kw)


@pytest.mark.parametrize("case", ["inf_cond", "sentinel", "categorical"])
def test_probe_rows_every_raw_path(eng, oracle, case, tmp_path):
    bst, obst, _, X, missing, kw = _probe_model(eng, oracle, case)
    assert_same_model(bst, obst)
    trees = bst.get_trees()
    P = probe_rows(trees, X, missing)
    d = eng.DMatrix(P, missing=missing, **kw)
    leaf = bst.predict(d, pred_leaf=True)
    assert np.array_equal(leaf, R.leaf_index(trees, P, missing))
    margin = bst.predict(d, output_margin=True)
    assert np.max(np.abs(margin - obst.predict_margin(P, missing)[:, 0])) <= 1e-5
    phi = bst.predict(d, pred_contribs=True)
    ref = R.shap_contribs(trees, P, missing=missing, base_value=_base_value(bst))[:, 0]
    tol = 1e-5 * np.maximum(1.0, np.abs(margin))[:, None]
    assert np.all(np.abs(phi - ref) <= tol), float(np.max(np.abs(phi - ref)))
    sub = P[:50]
    ds = eng.DMatrix(sub, missing=missing, **kw)
    inter = bst.predict(ds, pred_interactions=True)
    iref = R.shap_contribs(trees, sub, missing=missing, interactions=True, base_value=_base_value(bst))[:, 0]
    assert np.all(np.abs(inter - iref) <= tol[:50, :, None]), float(np.max(np.abs(inter - iref)))
    f = str(tmp_path / "m.json")
    bst.save_model(f)
    for other in (eng.Booster(model_file=f), pickle.loads(pickle.dumps(bst))):
        assert np.array_equal(other.predict(d, pred_leaf=True), leaf)
        assert np.array_equal(other.predict(d, output_margin=True), margin)
        assert np.array_equal(other.predict(d, pred_contribs=True), phi)
        assert np.array_equal(other.predict(ds, pred_interactions=True), inter)


# ------------------------------------------------------------------ eval metrics on a sentinel-missing matrix
@pytest.mark.parametrize("objective,metric", [("reg:squarederror", "rmse"), ("binary:logistic", "logloss")])
def test_eval_metric_with_sentinel(eng, oracle, objective, metric):
    X = adversarial(13, -999.0, n=20011)
    Xe = adversarial_block(7001, 99, -999.0)
    y, ye = labels(X, objective), labels(Xe, objective, seed=1)
    params = {"objective": objective, "max_depth": 6, "base_score": 0.5, "eval_metric": metric}
    obst, _ = oracle.train(params, X, y, 3, missing=-999.0)
    res = {}
    de = eng.DMatrix(Xe, label=ye, missing=-999.0)
    bst2 = eng.train(params, eng.DMatrix(X, label=y, missing=-999.0), num_boost_round=3, evals=[(de, "eval")],
                     evals_result=res, verbose_eval=False)
    assert_same_model(bst2, obst)
    want = obst.metric(metric, obst.predict_margin(Xe, -999.0), ye)
    assert abs(res["eval"][metric][-1] - want) <= 1e-5 * max(1.0, abs(want)), (res["eval"][metric][-1], want)


# ------------------------------------------------------------------ public API
def _ngpu():
    from xgboost_ray_b200 import engine
    return engine.device_count()


@pytest.mark.timeout(600)
def test_public_api_sentinel_one_actor(oracle):
    from xgboost_ray_b200 import RayDMatrix, RayParams, predict, train
    from xgboost_ray_b200.sklearn import RayXGBRegressor
    X = adversarial(13, -999.0, n=20011)
    y = labels(X, "reg:squarederror")
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5}
    ob, _ = oracle.train(params, X, y, 3, missing=-999.0)
    bst = train(params, RayDMatrix(X, y, missing=-999.0), num_boost_round=3, ray_params=RayParams(num_actors=1))
    assert_same_model(bst, ob)
    p = predict(bst, RayDMatrix(X, missing=-999.0), ray_params=RayParams(num_actors=1))
    assert np.max(np.abs(p - ob.predict(X, missing=-999.0))) <= 1e-5
    reg = RayXGBRegressor(n_estimators=3, max_depth=6, learning_rate=0.3, base_score=0.5, missing=-999.0)
    reg.fit(X, y, ray_params=RayParams(num_actors=1))
    assert_same_model(reg.get_booster(), ob)
    assert np.max(np.abs(reg.predict(X, ray_params=RayParams(num_actors=1)) - ob.predict(X, missing=-999.0))) <= 1e-5


@pytest.mark.timeout(600)
def test_public_api_sentinel_two_actors_identical_to_one():
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    X = adversarial(13, -999.0, n=20011)
    y = labels(X, "reg:squarederror")
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5}
    b1 = train(params, RayDMatrix(X, y, missing=-999.0), num_boost_round=3, ray_params=RayParams(num_actors=1))
    b2 = train(params, RayDMatrix(X, y, missing=-999.0), num_boost_round=3, ray_params=RayParams(num_actors=2))
    assert b1.get_dump(dump_format="json", with_stats=True) == b2.get_dump(dump_format="json", with_stats=True)


# ------------------------------------------------------------------ borrowed cuts and categories they do not know
def _borrowed_cat(rng, n, codes, missing_frac=0.0):
    X = np.stack([rng.uniform(0, 10, size=n), rng.choice(np.asarray(codes, F), size=n)], axis=1).astype(F)
    X[:len(codes), 1] = codes
    if missing_frac:
        X[rng.uniform(size=n) < missing_frac, 1] = np.nan
    return X


CAT_KW = {"feature_types": ["q", "c"], "enable_categorical": True}


@pytest.mark.parametrize("bad,match", [(7.0, "category code 7 is above the largest code 5"),
                                       (-1.0, "got -1"), (2.5, "got 2.5"), (-np.inf, "got -inf"),
                                       (1e9, r"got 1e\+09")])
@pytest.mark.parametrize("path", ["ref", "frozen"])
def test_borrowed_cuts_refuse_unknown_categories(eng, bad, match, path):
    rng = np.random.RandomState(2)
    d1 = eng.DMatrix(_borrowed_cat(rng, 5000, range(6)), **CAT_KW)
    d1._ensure_quantized(256, keep_raw=True)
    X2 = _borrowed_cat(rng, 8000, range(6))
    X2[4321, 1] = bad
    y = rng.normal(size=len(X2)).astype(F)
    with pytest.raises(eng.XGBoostError, match="categorical feature 1: .*" + match):
        if path == "ref":
            eng.train({"max_depth": 3}, eng.DMatrix(X2, label=y, ref=d1, **CAT_KW), num_boost_round=1, verbose_eval=False)
        else:
            eng.DMatrix(X2, label=y, **CAT_KW)._ensure_quantized(256, cuts=d1.get_cuts())


def test_borrowed_cuts_refuse_missing_that_collides_with_category_255(eng):
    rng = np.random.RandomState(4)
    d1 = eng.DMatrix(_borrowed_cat(rng, 5000, range(256)), **CAT_KW)          # codes 0..255, no missing
    d1._ensure_quantized(256, keep_raw=True)
    X2 = _borrowed_cat(rng, 6000, range(256), missing_frac=0.05)
    with pytest.raises(eng.XGBoostError, match="categorical feature 1: .*missing sentinel"):
        eng.DMatrix(X2, ref=d1, **CAT_KW)._ensure_quantized(256)


def test_borrowed_cuts_with_known_categories_identical_and_route_alike(eng, oracle):
    """the borrowed cuts have no missing values, the training matrix has NaN in the categorical feature: both sides
    mark it has_missing (DESIGN.md §2 item 6), grow the same trees, and training routes NaN as predict() does"""
    rng = np.random.RandomState(5)
    X1 = _borrowed_cat(rng, 5000, range(10))
    d1 = eng.DMatrix(X1, **CAT_KW)
    X2 = _borrowed_cat(rng, 20011, range(0, 10, 2), missing_frac=0.05)       # a subset of the codes, and NaN
    y = (np.isin(X2[:, 1], [2, 6]) * 3 + X2[:, 0] * 0.2 + rng.normal(scale=0.1, size=len(X2))).astype(F)
    params = {"objective": "reg:squarederror", "max_depth": 4, "base_score": 0.5}
    dm = eng.DMatrix(X2, label=y, ref=d1, **CAT_KW)
    bst = eng.train(params, dm, num_boost_round=3, verbose_eval=False)
    borrowed = oracle.Cuts.from_data(X1, 256, is_cat=[0, 1])
    assert list(borrowed.has_missing) == [0, 0]
    obst, _ = oracle.train(params, X2, y, 3, cuts=borrowed)
    assert list(dm.get_cuts()[3]) == list(obst.cuts.has_missing) == [0, 1]
    assert_same_model(bst, obst)
    assert any(t["split_type"].any() for t in bst.get_trees())
    margin = assert_routes_agree(eng, bst, dm, X2, np.nan, **CAT_KW)
    assert np.max(np.abs(margin - obst.predict_margin(X2)[:, 0])) <= 1e-5
