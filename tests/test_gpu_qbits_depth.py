"""The fixed-point histogram path across hist_qbits 8-24 and trees of depth 13-14, against the CPU oracle.

hist_qbits sets both the size of a quantised gradient (|q| <= 2^qbits) and the overflow-guard window of the int32
shared-memory cells (2^(30 - qbits) rows add at most 2^30).  At 22-24 bits the window is 256, 128 or 64 rows and the
chunk shrinks to it; at 8 bits it is 2^22 rows and gains are coarse, so exact ties decide splits.  Depth 13-14 runs
the split scan, the level decision and the gathering leaf path at 4,096-8,192 nodes per level with node ids up to
32,766.  The quantiser's own edges (tiny and subnormal maxima of hessians and weights) close the file.

Tolerance: trees are compared exactly (topology, splits, default directions, loss_chg); leaf values, margins and
predictions within 1e-5, except where a test says bit for bit.  Device memory: depth 14 keeps 2 GiB of level
histograms per feature group, so every deep case uses at most 16 features (one group)."""
import numpy as np
import pytest

from tests.test_gpu_parity import LEAF_TOL, assert_same_model, make_data, run_both
from tests.test_oracle_quantisation import (binade_bounds, grow_tiny_hessian, quantise_case, reference_quantise,
                                          three_bit_weights, tiny_hessian_case)

pytestmark = pytest.mark.gpu

F = np.float32


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


# ------------------------------------------------------------------ histogram kernel at the window edges (a10)
def window_edge_cases(f):
    """(label, bins, qg, qh, ridx, window, chunk) of f features at qbits 22-24: |q| = 2^qbits exactly, and on the
    constant feature 0 a run of window rows of +2^qbits (cell exactly 2^30 at the window boundary), a run of
    2^qbits - 1 that leaves the cell just below 2^30 at the check followed by a full window of +2^qbits (the cell
    reaches 2^31 - window), and the same runs negated"""
    for qbits in (22, 23, 24):
        window = 1 << (30 - qbits)
        top = 1 << qbits
        rng = np.random.RandomState(qbits)
        n = 9 * window + 3000
        bins = rng.randint(0, 256, size=(n, f)).astype(np.uint8)
        bins[:, 0] = 7
        bins[:, 1] &= 1
        bins[:, 2] = 255
        runs = [np.full(window, top), np.full(window, top - 1), np.full(window, top), np.full(window, -top),
                np.full(window, -(top - 1)), np.full(window, -top), np.full(3 * window, top)]
        qg = np.concatenate(runs + [np.where(rng.uniform(size=3000) < 0.5, top, -top)]).astype(np.int32)
        qh = np.full(n, top, np.int32)
        qh[n - 3000:] = rng.choice([0, 1, top - 1, top], size=3000)
        sel = np.sort(rng.choice(n, n // 2, replace=False)).astype(np.int32)
        for ridx in (None, sel, rng.permutation(n).astype(np.int32)):
            for chunk in (window, window // 2):
                yield (qbits, chunk, None if ridx is None else ridx.size), bins, qg, qh, ridx, window, chunk


@pytest.mark.parametrize("f", [37, 530])   # 2 groups (one group-pair CTA type); 17 groups (one group per CTA)
def test_hist_window_edges_bit_exact(eng, oracle, f):
    for label, bins, qg, qh, ridx, window, chunk in window_edge_cases(f):
        ref = oracle.hist_int(bins, qg, qh, ridx)
        assert ref[0, 7, 0] == int(qg.astype(np.int64)[ridx if ridx is not None else slice(None)].sum())
        got, _ = eng.hist_build_raw(bins, qg, qh, ridx=ridx, window_rows=window, chunk_rows=chunk)
        assert np.array_equal(ref, got), label


def test_hist_qbits8_window_of_four_million_rows(eng, oracle):
    """qbits 8: the window is 2^22 rows.  One node of 2^22 + 2^18 rows whose first 2^22 rows all add +2^8 to the
    constant feature's cell, so it reaches 2^30 exactly as the first window closes, then keeps growing."""
    window = 1 << 22
    n, f = window + (1 << 18), 4
    rng = np.random.RandomState(8)
    bins = rng.randint(0, 256, size=(n, f)).astype(np.uint8)
    bins[:, 0] = 3
    qg = np.full(n, 256, np.int32)
    qg[window:] = np.where(rng.uniform(size=n - window) < 0.8, 256, -256)
    qh = np.full(n, 256, np.int32)
    ref = oracle.hist_int(bins, qg, qh)
    assert ref[0, 3, 0] > 2 ** 30 and ref[0, 3, 1] == 256 * n
    for chunk in (8192, 2048):
        got, _ = eng.hist_build_raw(bins, qg, qh, window_rows=window, chunk_rows=chunk)
        assert np.array_equal(ref, got), chunk


# ------------------------------------------------------------------ whole trees at hist_qbits 8-24 (a9-a14)
QBITS = [8, 12, 22, 23, 24]


def regression(n, f, seed, nan_frac=0.0):
    X = make_data(n, f, seed, "uniform", nan_frac=nan_frac)
    rng = np.random.RandomState(seed + 1)
    x = np.nan_to_num(X, nan=5.0)
    y = x[:, : min(f, 6)].sum(axis=1) + np.sin(x[:, 0]) * 3 + rng.normal(scale=0.5, size=n)
    return X, (y - y.mean()).astype(F)


def check_margins(ebst, obst, dm, X_test=None, dm_test=None):
    m = ebst.predict(dm, output_margin=True, training=True)
    assert np.max(np.abs(m - obst.margin[:, 0])) <= LEAF_TOL
    if X_test is not None:
        assert np.max(np.abs(ebst.predict(dm_test, output_margin=True) - obst.predict(X_test, output_margin=True))) <= LEAF_TOL


@pytest.mark.parametrize("qbits", QBITS)
@pytest.mark.parametrize("objective", ["reg:squarederror", "binary:logistic"])
def test_trees_identical_at_qbits(eng, oracle, qbits, objective):
    X, y = regression(20000, 16, 31)
    if objective == "binary:logistic":
        y = (y > np.median(y)).astype(F)
    params = {"objective": objective, "max_depth": 8, "eta": 0.3, "base_score": 0.5, "hist_qbits": qbits}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 4)     # rounds 2+ replay the captured graph
    assert_same_model(ebst, obst)
    check_margins(ebst, obst, dm)


@pytest.mark.parametrize("qbits", QBITS)
def test_trees_identical_at_qbits_missing_and_weights(eng, oracle, qbits):
    n, f = 15000, 12
    X = make_data(n, f, 5, "mixed", nan_frac=0.15)
    rng = np.random.RandomState(qbits)
    y = (np.nan_to_num(X[:, 0]) + np.nan_to_num(X[:, 3]) + rng.normal(scale=0.5, size=n) > 0).astype(F)
    w = rng.uniform(0.5, 2.0, size=n).astype(F)
    params = {"objective": "binary:logistic", "max_depth": 8, "base_score": 0.5, "min_child_weight": 0.5,
              "hist_qbits": qbits}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 3, weight=w)
    assert_same_model(ebst, obst)
    check_margins(ebst, obst, dm)


@pytest.mark.parametrize("qbits", QBITS)
def test_categorical_trees_identical_at_qbits(eng, oracle, qbits):
    from tests.test_gpu_parity import make_cat_data, run_both_cat
    X, score, rng = make_cat_data(20000, 41, 0.05)
    y = score + rng.normal(scale=0.3, size=len(score)).astype(F)
    params = {"objective": "reg:squarederror", "max_depth": 8, "eta": 0.3, "base_score": 0.5, "hist_qbits": qbits}
    ebst, obst, dm = run_both_cat(eng, oracle, params, X, y, 3)
    assert_same_model(ebst, obst)
    check_margins(ebst, obst, dm)


def test_trees_identical_qbits24_million_rows(eng, oracle):
    """2^20 + 4097 rows at 24 bits: the root histogram runs 64-row chunks (one window each) over the whole grid."""
    X, y = regression((1 << 20) + 4097, 8, 17)
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5, "hist_qbits": 24}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 2)
    assert_same_model(ebst, obst)
    check_margins(ebst, obst, dm)


def test_chunk_override_clamped_to_window(eng, oracle):
    """hist_chunk_rows above the 64-row window of 24 bits is clamped at every level, the root included."""
    X, y = regression(30000, 10, 23)
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5, "hist_qbits": 24}
    ebst, obst, dm = run_both(eng, oracle, dict(params, hist_chunk_rows=4096), X, y, 3)
    plain = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=3, verbose_eval=False)
    assert ebst.get_dump(dump_format="json", with_stats=True) == plain.get_dump(dump_format="json", with_stats=True)
    assert_same_model(ebst, obst)
    check_margins(ebst, obst, dm)


# ------------------------------------------------------------------ depth 13 and 14
DEEP_ROWS = 1 << 18


def node_depths(t):
    d = np.zeros(len(t["left"]), np.int32)
    for nid in range(1, len(d)):       # a child's id is larger than its parent's
        d[nid] = d[t["parent"][nid]] + 1
    return d


def leaf_walk(t, X):
    """node id of the leaf each row reaches, numeric splits only (x < cond goes left, NaN takes the default)"""
    n = X.shape[0]
    nid = np.zeros(n, np.int64)
    rows = np.arange(n)
    while True:
        feat = t["split_feature"][nid]
        inner = feat >= 0
        if not inner.any():
            return nid
        x = X[rows, np.maximum(feat, 0)]
        left = np.where(np.isnan(x), t["default_left"][nid] != 0, x < t["split_cond"][nid])
        nid = np.where(inner, np.where(left, t["left"][nid], t["right"][nid]), nid)


def deep_case(seed, nan_frac=0.0):
    X = make_data(DEEP_ROWS, 16, seed, "uniform", nan_frac=nan_frac)
    rng = np.random.RandomState(seed + 7)
    x = np.nan_to_num(X, nan=5.0)
    y = x[:, :8].sum(axis=1) + np.sin(x[:, 0] * 2) * 3 + rng.normal(scale=2.0, size=DEEP_ROWS)
    if nan_frac:
        # NaN rows lean one way on feature 0 and the other way on feature 1: both default directions win somewhere
        y += np.where(np.isnan(X[:, 0]), 6.0, 0.0) - np.where(np.isnan(X[:, 1]), 6.0, 0.0)
    # centred: with labels far from base_score, the binary32 loss_chg of a deep split rounds away and growth stops
    return X, (y - y.mean()).astype(F)


def check_deep(ebst, obst, dm, depth, X_test=None, dm_test=None, walk=True):
    assert_same_model(ebst, obst)
    t0 = ebst.get_trees()[0]
    d = node_depths(t0)
    assert d.max() == depth
    deep_splits = int(((t0["split_feature"] >= 0) & (d >= 12)).sum())
    assert deep_splits > 2000, deep_splits                     # the deep levels really fill
    check_margins(ebst, obst, dm, X_test, dm_test)
    if walk:
        leaf = ebst.predict(dm_test, pred_leaf=True)
        trees = ebst.get_trees()
        want = np.stack([leaf_walk(t, X_test) for t in trees], axis=1)
        assert np.array_equal(np.asarray(leaf).reshape(want.shape).astype(np.int64), want)


@pytest.mark.parametrize("depth,objective", [(14, "reg:squarederror"), (14, "binary:logistic"), (13, "reg:squarederror")])
def test_deep_trees_identical(eng, oracle, depth, objective):
    X, y = deep_case(3)
    if objective == "binary:logistic":
        y = (y > np.median(y)).astype(F)
    params = {"objective": objective, "max_depth": depth, "eta": 0.3, "base_score": 0.5, "min_child_weight": 0.0}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 2)
    Xt, _ = deep_case(4)
    Xt = Xt[:20000]
    check_deep(ebst, obst, dm, depth, Xt, eng.DMatrix(Xt))


def test_deep_trees_missing_both_directions(eng, oracle):
    X, y = deep_case(5, nan_frac=0.1)
    params = {"objective": "reg:squarederror", "max_depth": 13, "eta": 0.3, "base_score": 0.5, "min_child_weight": 0.0}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 2)
    t0 = ebst.get_trees()[0]
    dl = t0["default_left"][t0["split_feature"] >= 0]
    assert dl.any() and not dl.all()
    Xt, _ = deep_case(6, nan_frac=0.1)
    Xt = Xt[:20000]
    check_deep(ebst, obst, dm, 13, Xt, eng.DMatrix(Xt))


def test_deep_trees_colsample_bynode(eng, oracle):
    X, y = deep_case(7)
    params = {"objective": "reg:squarederror", "max_depth": 14, "eta": 0.3, "base_score": 0.5, "min_child_weight": 0.0,
              "colsample_bynode": 0.5, "seed": 11}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 2)
    Xt = X[:20000]
    check_deep(ebst, obst, dm, 14, Xt, eng.DMatrix(Xt))


def test_deep_trees_categorical(eng, oracle):
    """Categorical features at thousands of nodes per level: stored siblings and eval_cat_splits."""
    rng = np.random.RandomState(9)
    n = DEEP_ROWS
    Xn = rng.uniform(0, 10, size=(n, 12))
    cards = (3, 20, 100, 200)
    Xc = np.column_stack([rng.randint(0, c, size=n) for c in cards])
    X = np.column_stack([Xn, Xc]).astype(F)
    y = (Xn[:, :6].sum(axis=1) + (Xc[:, 1] % 3 == 0) * 2.0 + (Xc[:, 2] % 7 < 3) * 1.5 + (Xc[:, 3] % 5) * 0.7
         + rng.normal(scale=2.0, size=n))
    y = (y - y.mean()).astype(F)
    is_cat = [0] * 12 + [1] * 4
    types = ["q"] * 12 + ["c"] * 4
    params = {"objective": "reg:squarederror", "max_depth": 13, "eta": 0.3, "base_score": 0.5, "min_child_weight": 0.0}
    obst, _ = oracle.train(params, X, y, 2, is_cat=is_cat)
    dm = eng.DMatrix(X, label=y, feature_types=types, enable_categorical=True)
    ebst = eng.train(params, dm, num_boost_round=2, verbose_eval=False)
    t0 = ebst.get_trees()[0]
    st = t0["split_type"][(t0["split_feature"] >= 0) & (node_depths(t0) >= 10)]
    assert st.sum() > 100                                      # categorical splits deep in the tree
    Xt = X[:20000]
    check_deep(ebst, obst, dm, 13, Xt, eng.DMatrix(Xt, feature_types=types, enable_categorical=True), walk=False)


# ------------------------------------------------------------------ the quantiser's edges on the GPU
@pytest.mark.parametrize("qbits", [8, 18, 24])
def test_quantize_kernel_every_binade(eng, oracle, qbits):
    """quant_exponent_kernel + quantize_kernel against oracle.quantize and rint(v * 2^(qbits - e)) in float64, with
    max |g| at both ends of every binade from 2^-149 to 2^127 and max |h| in the mirrored binade (so every subnormal
    binade is met by both)"""
    rng = np.random.RandomState(qbits)
    for b in range(-149, 128):
        for i, gmax in enumerate(binade_bounds(b)):
            g = quantise_case(gmax, rng, negative_max=(b % 2 == 0))
            h = np.abs(quantise_case(binade_bounds(-22 - b)[1 - i], rng, negative_max=False))
            qg, qh, es = eng.quantize_raw(g, h, qbits)
            for v, q, e in ((g, qg, es[0]), (h, qh, es[1])):
                want, we = reference_quantise(v, qbits)
                oq, oe = oracle.quantize(v, qbits)
                assert e == we == oe, (qbits, b, float(np.max(np.abs(v))), e, we)
                assert np.array_equal(q, oq) and np.array_equal(q.astype(np.float64), want), (qbits, b)
    qg, qh, es = eng.quantize_raw(np.zeros(5, F), np.full(5, -0.0, F), qbits)
    assert es == (0, 0) and not qg.any() and not qh.any()


def subnormal_pairs(y):
    """gradients y * 2^-60 and hessians in [2^-128, 2^-126) with full mantissas: max |h| is subnormal, and its
    quantised values (unlike those of a few-bit hessian) change when the exponent is off by one"""
    y64 = np.asarray(y, np.float64)
    frac = np.modf(np.abs(y64) * 7.3)[0]
    return (y64 * 2.0 ** -60).astype(F), ((0.25 + 0.75 * frac) * 2.0 ** -126).astype(F)


def subnormal_obj(pred, d):
    return subnormal_pairs(d.get_label())


SUBNORMAL_PARAMS = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5, "lambda": 0.0,
                    "min_child_weight": 0.0}


@pytest.mark.parametrize("qbits", [8, 12])
def test_subnormal_hessian_trees_match_oracle(eng, oracle, qbits):
    """lambda 0, so H is not negligible and the quantised hessians decide gains, splits and every node's sum_hess"""
    X, y = regression(20000, 8, 51)
    g, h = subnormal_pairs(y)
    assert np.max(h) < np.float32(2.0 ** -126) and np.unique(h).size > 10000
    params = dict(SUBNORMAL_PARAMS, hist_qbits=qbits)
    ebst = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=2, obj=subnormal_obj, verbose_eval=False)
    cuts = oracle.Cuts.from_data(X, 256)
    bins = cuts.bin(X)
    obst = oracle.Booster(params, cuts)
    obst.init_margin(X.shape[0])
    for _ in range(2):
        obst.boost(bins, y, None, custom_g=g, custom_h=h)
    assert_same_model(ebst, obst, leaf_tol=0.0)
    for i, t in enumerate(ebst.get_trees()):
        assert len(t["left"]) > 15
        assert np.array_equal(t["sum_hess"], obst.tree(i).sum_hess), i


@pytest.mark.parametrize("qbits", [8, 18, 24])
def test_tiny_hessian_custom_objective(eng, oracle, qbits):
    """hessians (1 + j/8) * 2^-k, lambda 1, min_child_weight 0: the model must not depend on k, down to subnormal
    hessians (k = 140), and must equal the oracle's bit for bit"""
    X, y, hunit = tiny_hessian_case()
    ref = None
    for k in (100, 106, 112, 122, 126, 140):
        h = (hunit.astype(np.float64) * 2.0 ** -k).astype(F)

        def obj(pred, d, h=h):
            return (np.asarray(pred, F).reshape(-1) - d.get_label()).astype(F), h

        params = {"objective": "reg:squarederror", "max_depth": 5, "eta": 0.3, "base_score": 0.5, "lambda": 1.0,
                  "min_child_weight": 0.0, "hist_qbits": qbits}
        dm = eng.DMatrix(X, label=y)
        ebst = eng.train(params, dm, num_boost_round=2, obj=obj, verbose_eval=False)
        obst = grow_tiny_hessian(oracle, X, y, hunit, k, qbits)
        assert_same_model(ebst, obst, leaf_tol=0.0)
        m = ebst.predict(dm, output_margin=True, training=True)
        assert np.array_equal(np.asarray(m, F).view(np.uint32), obst.margin[:, 0].view(np.uint32)), k
        trees = [(t["split_feature"].tolist(), t["split_bin"].tolist(), t["value"].view(np.uint32).tolist())
                 for t in ebst.get_trees()]
        if ref is None:
            ref = trees
            assert len(trees[0][0]) > 15
        assert trees == ref, k


def test_weighted_cuts_invariant_under_power_of_two_scale(eng, oracle):
    rng = np.random.RandomState(12)
    n, f = 20000, 4
    X = rng.normal(size=(n, f)).astype(F)
    X[:, 1] = np.round(X[:, 1] * 3)
    X[rng.uniform(size=X.shape) < 0.1] = np.nan
    w = three_bit_weights(rng, n)
    assert np.signbit(w[w == 0]).any()                          # -0.0 weights must not pass for the maximum
    base = None
    for k in (0, -140, -126, -99, -98, -40, 60, 100):
        wk = (w.astype(np.float64) * 2.0 ** k).astype(F)
        dm = eng.DMatrix(X, weight=wk)
        dm._ensure_quantized(256, keep_raw=True)
        got = [a.view(np.uint32) if a.dtype == F else a for a in dm.get_cuts()] + [dm.get_bins()]
        if base is None:
            base = got
            oc = oracle.Cuts.from_data(X, 256, weight=w)
            assert np.array_equal(got[0], oc.ptrs) and np.array_equal(got[1], oc.vals.view(np.uint32))
            assert np.array_equal(got[4], oc.bin(X))
        for a, b in zip(got, base):
            assert np.array_equal(a, b), k


# ------------------------------------------------------------------ two GPUs
def _ngpu():
    from xgboost_ray_b200 import engine
    return engine.device_count()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_two_gpu_subnormal_hessians_identical_to_one_gpu(exchange, monkeypatch):
    """The peer-memory exchange takes the quantisation exponents from its own kernel: with a subnormal max |h| its
    sum_hess (in the dump's cover) must equal one GPU's"""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    import xgboost_ray_b200.main as M
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    M.shutdown_actors()
    if exchange == "nccl":
        monkeypatch.setenv("B2_EXCHANGE", "nccl")
    else:
        monkeypatch.delenv("B2_EXCHANGE", raising=False)
    X, y = regression(20000, 8, 51)
    params = dict(SUBNORMAL_PARAMS, hist_qbits=8)
    b1 = train(params, RayDMatrix(X, y), num_boost_round=2, obj=subnormal_obj, ray_params=RayParams(num_actors=1))
    b2 = train(params, RayDMatrix(X, y), num_boost_round=2, obj=subnormal_obj, ray_params=RayParams(num_actors=2))
    M.shutdown_actors()
    assert b1.get_dump(dump_format="json", with_stats=True) == b2.get_dump(dump_format="json", with_stats=True)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
@pytest.mark.parametrize("depth,qbits", [(14, 24), (6, 8)])
def test_two_gpu_identical_to_one_gpu(exchange, depth, qbits, monkeypatch):
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    import xgboost_ray_b200.main as M
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    M.shutdown_actors()                       # the exchange kind is read by the actor processes when they start
    if exchange == "nccl":
        monkeypatch.setenv("B2_EXCHANGE", "nccl")
    else:
        monkeypatch.delenv("B2_EXCHANGE", raising=False)
    X, y = deep_case(13)
    X = X[: 1 << 17]
    y = y[: 1 << 17]
    params = {"objective": "reg:squarederror", "max_depth": depth, "eta": 0.3, "base_score": 0.5,
              "min_child_weight": 0.0, "hist_qbits": qbits}
    b1 = train(params, RayDMatrix(X, y), num_boost_round=2, ray_params=RayParams(num_actors=1))
    b2 = train(params, RayDMatrix(X, y), num_boost_round=2, ray_params=RayParams(num_actors=2))
    M.shutdown_actors()
    assert b1.get_dump(dump_format="json", with_stats=True) == b2.get_dump(dump_format="json", with_stats=True)
