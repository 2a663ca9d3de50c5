"""GPU checks of the scalar objectives' gradient kernels (gradient_scalar_kernel, gradient_param_kernel,
gradient_multi_target_kernel): the pairs read back with B2_BoosterGetGradients equal tests/objective_reference.py bit
for bit on the edge grids of tests/test_objective_gradient_edges.py, fed through base_margin; a pair that is not finite
fails the round and keeps the model's trees; the fused |g|, |h| maxima (T <= 16) and absmax_kernel (T > 16, or
subsample < 1) give the oracle's trees; and a NaN or infinite label is refused before any tree is grown."""
import ctypes as C

import numpy as np
import pytest

from tests import multi_target_reference as MT
from tests import objective_reference as R
from tests.test_gpu_parity import assert_same_model
from tests.test_objective_gradient_edges import all_cases, case_id, edge_grid, param_sets

pytestmark = pytest.mark.gpu
F = np.float32
ROWS_PER_PASS = 132 * 16 * 256          # grid_for's cap on an H100 (132 SMs, 16 CTAs of 256 threads each)


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def get_gradients(eng, bst, n):
    g = np.zeros(n, np.float32)
    h = np.zeros(n, np.float32)
    eng._check(eng.lib().B2_BoosterGetGradients(bst.handle, g.ctypes.data_as(C.POINTER(C.c_float)),
                                                  h.ctypes.data_as(C.POINTER(C.c_float)), n))
    return g, h


def features(n, seed=0):
    return np.random.RandomState(seed).uniform(0, 10, size=(n, 2)).astype(F)


def resize(a, n, shift=0):
    """a rotated by `shift` and tiled or cut to n rows."""
    if a is None:
        return None
    a = np.roll(a, shift, axis=0)
    reps = -(-n // len(a))
    return np.ascontiguousarray(np.concatenate([a] * reps, axis=0)[:n])


def one_round(eng, params, X, y, m, w, **dm_kw):
    """One update from margin m (base_margin) with base_score fixed; (booster, error text or None)."""
    dm = eng.DMatrix(X, label=y, weight=w, base_margin=m, **dm_kw)
    bst = eng.Booster(dict(params, max_depth=1, base_score=0.5), cache=[dm])
    try:
        bst.update(dm, 0)
        return bst, None
    except eng.XGBoostError as e:
        return bst, str(e)


@pytest.mark.parametrize("n", ["grid", 1, 255, 257, 2 * ROWS_PER_PASS + 1])
@pytest.mark.parametrize("case", all_cases(), ids=case_id)
def test_gradients_bit_equal_to_reference(eng, case, n):
    """Every edge row, weighted and not, at row counts around one warp-block and past two grid-stride passes."""
    params, weighted = case
    p, y, w = edge_grid(params, weighted)
    if n != "grid":
        p, y, w = resize(p, n, 7), resize(y, n, 7), resize(w, n, 7)
    n = len(p)
    bst, err = one_round(eng, params, features(n), y, p, w)
    rg, rh, bad = R.gradients(params, p, y, w)
    if bad:
        assert err is not None and "not finite" in err and params["objective"] in err, err
    else:
        assert err is None, err
    g, h = get_gradients(eng, bst, n)
    assert same_bits(g, rg), np.nonzero(g.view(np.uint32) != rg.view(np.uint32))[0][:10]
    assert same_bits(h, rh), np.nonzero(h.view(np.uint32) != rh.view(np.uint32))[0][:10]


@pytest.mark.parametrize("obj", R.CHECKS_FINITE)
def test_nonfinite_pair_fails_the_round_and_keeps_the_trees(eng, obj):
    """Without its overflowing rows the grid trains; with them the next round fails with the existing error and the
    model keeps its trees."""
    params = dict(param_sets(obj)[-1], objective=obj, eta=0.1)
    p, y, w = edge_grid(params, True)
    over = np.array([R.gradients(params, p[i:i + 1], y[i:i + 1], w[i:i + 1])[2] > 0 for i in range(len(p))])
    assert over.any()
    X = features(len(p), 3)
    ok = eng.DMatrix(X[~over], label=y[~over], weight=w[~over], base_margin=p[~over])
    bad_dm = eng.DMatrix(X, label=y, weight=w, base_margin=p)
    bst = eng.Booster(dict(params, max_depth=2, base_score=0.5), cache=[ok])
    bst.update(ok, 0)
    assert bst.num_trees() == 1
    before = [t["value"].copy() for t in bst.get_trees()]
    # the margin of the failing round is base_margin plus the kept tree: the reference confirms a row still overflows
    m1 = bst.predict(bad_dm, output_margin=True)
    assert R.gradients(params, m1, y, w)[2] > 0
    with pytest.raises(eng.XGBoostError, match="%s: a gradient or hessian is not finite" % obj):
        bst.update(bad_dm, 1)
    assert bst.num_trees() == 1
    assert all(np.array_equal(a["value"], b) for a, b in zip(bst.get_trees(), before))


def multi_target_grid(params, T, weighted):
    """(margin, label) [n][T] with the objective's edge rows in every column (rotated per column), weight [n]."""
    p, y, w = edge_grid(params, weighted)
    M = np.stack([np.roll(p, 5 * k) for k in range(T)], axis=1).astype(F)
    Y = np.stack([np.roll(y, 5 * k) for k in range(T)], axis=1).astype(F)
    if params["objective"] not in R.CHECKS_FINITE:   # as in edge_grid: no row whose pair overflows in some column
        g, h, _ = R.gradients_multi_target(params, M, Y, w)
        keep = np.all(np.isfinite(g) & np.isfinite(h), axis=0)
        M, Y, w = M[keep], Y[keep], None if w is None else w[keep]
    return M, Y, w


@pytest.mark.parametrize("T", [1, 16, 17])
@pytest.mark.parametrize("obj", MT.MULTI_TARGET_OBJECTIVES)
@pytest.mark.parametrize("weighted", [False, True])
def test_multi_target_gradients_bit_equal(eng, obj, T, weighted):
    for extra in param_sets(obj):
        params = dict(extra, objective=obj)
        M, Y, w = multi_target_grid(params, T, weighted)
        n = len(M)
        bst, err = one_round(eng, params, features(n, T), Y if T > 1 else Y[:, 0], M if T > 1 else M[:, 0], w,
                             multi_target=T > 1)
        rg, rh, bad = R.gradients_multi_target(params, M, Y, w)
        if bad:
            assert err is not None and "not finite" in err, err
        else:
            assert err is None, err
        g, h = get_gradients(eng, bst, n * T)
        assert same_bits(g, rg.reshape(-1)) and same_bits(h, rh.reshape(-1)), (params, T)


def finite_edge_data(obj, T, n=3000, seed=0):
    """Edge-heavy data whose pairs are all finite at the base margin: margins at the clamps and on both sides of zero,
    labels at 0, 1 and its neighbours, weights from 2^-149 to 1e4 (the last sets |g|, |h| maxima far above the rest)."""
    rng = np.random.RandomState(seed)
    X = features(n, seed)
    margins = np.array([0.0, -0.0, 2.0 ** -149, 1e-8, -1e-8, 1.0, -1.0, 16.6, -16.6, 88.7, -88.7], F)
    if obj in R.LOGISTIC:
        labels = np.array([0.0, 1.0, 0.99999994, 0.5], F)
    else:
        labels = np.array([0.0, 1.0, 0.99999994, 1.0000001, 3.0, -0.5], F)
    M = margins[rng.randint(0, len(margins), size=(n, T))] + (X[:, :1] > 5).astype(F)
    Y = labels[rng.randint(0, len(labels), size=(n, T))]
    w = np.array([1.0, 0.5, 2.0 ** -149, 1e-30, 2.0], F)[rng.randint(0, 5, n)]
    w[rng.randint(0, n, 30)] = F(1e4)
    return X, M.astype(F), Y.astype(F), w


@pytest.mark.parametrize("subsample", [1.0, 0.7])
@pytest.mark.parametrize("T", [1, 16, 17])
@pytest.mark.parametrize("obj", ["reg:squarederror", "binary:logistic", "reg:pseudohubererror"])
def test_quantisation_scale_gives_the_oracles_trees(eng, oracle, obj, T, subsample):
    """One round at depth 2: the |g|, |h| maxima set each tree's fixed-point exponent, so a wrong maximum (the fused
    one for T <= 16 at subsample 1, absmax_kernel otherwise) changes the leaves."""
    X, M, Y, w = finite_edge_data(obj, T, seed=T)
    params = {"objective": obj, "max_depth": 2, "eta": 1.0, "base_score": 0.5, "subsample": subsample, "seed": 3}
    g, h, bad = R.gradients_multi_target(params, M, Y, w)
    assert bad == 0 and np.isfinite(g).all() and np.isfinite(h).all()
    if T == 1:
        dm = eng.DMatrix(X, label=Y[:, 0], weight=w, base_margin=M[:, 0])
        ref = R.train(oracle, params, X, Y[:, 0], 1, weight=w, base_margin_rows=M)
    else:
        dm = eng.DMatrix(X, label=Y, weight=w, base_margin=M, multi_target=True)
        ref = MT.train(oracle, params, X, Y, 1, weight=w, base_margin=M)
    bst = eng.train(params, dm, num_boost_round=1, verbose_eval=False)
    assert_same_model(bst, ref)


NONFINITE_OBJECTIVES = ["reg:squarederror", "reg:linear", "binary:logistic", "reg:pseudohubererror"]


@pytest.mark.parametrize("obj", NONFINITE_OBJECTIVES)
@pytest.mark.parametrize("bad_label", [np.nan, np.inf, -np.inf])
@pytest.mark.parametrize("base_score", [0.5, None])
@pytest.mark.parametrize("T,strategy", [(1, None), (3, "one_output_per_tree"), (3, "multi_output_tree")])
def test_nonfinite_labels_are_refused(eng, obj, bad_label, base_score, T, strategy):
    n = 500
    X = features(n, 5)
    Y = (np.random.RandomState(5).uniform(size=(n, T)) > 0.5).astype(F)
    Y[123, T - 1] = bad_label
    params = {"objective": obj, "max_depth": 2}
    if base_score is not None:
        params["base_score"] = base_score
    if strategy is not None:
        params["multi_strategy"] = strategy
    lab = Y if T > 1 else Y[:, 0]
    bad_dm = eng.DMatrix(X, label=lab, multi_target=T > 1)
    bst = eng.Booster(params, cache=[bad_dm])
    with pytest.raises(eng.XGBoostError, match="label must be finite for %s" % obj):
        bst.update(bad_dm, 0)
    assert bst.num_trees() == 0
    Y[123, T - 1] = 1.0
    ok = eng.DMatrix(X, label=Y if T > 1 else Y[:, 0], multi_target=T > 1)
    bst.update(ok, 0)
    assert bst.num_trees() == (1 if strategy == "multi_output_tree" else T)
