"""GPU checks of multi:softprob / multi:softmax on both sides of the fused class-count limit KF (16 today): gradients
bit-equal to the oracle's, trees identical to the oracle (graph replay at K <= KF, direct launches above), mlogloss /
merror against a float64 reference of the kernel's binary32 sequence, the softmax transform and argmax, SHAP
contributions in each shared-memory branch of the contributions kernel, label validation, save / load / continuation
and two GPUs."""
import ctypes as C
import math
import re

import numpy as np
import pytest

from tests import shap_reference as R
from tests.objective_reference import expf_
from tests.test_gpu_parity import assert_same_model, make_data

pytestmark = pytest.mark.gpu
F32 = np.float32
LABEL_MSG = r"label must be in \[0, num_class\)"
# class counts, resolved against the library's fused limit KF at run time: both sides of it stay covered if it moves
K_SPECS = ["2", "3", "KF", "KF+1", "40"]


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def classes(eng, spec):
    kf = eng.lib().b2_gradient_fused_max_classes()
    return {"KF": kf, "KF+1": kf + 1}.get(spec) or int(spec)


def get_gradients(eng, bst, n):
    g = np.zeros(n, np.float32)
    h = np.zeros(n, np.float32)
    eng._check(eng.lib().B2_BoosterGetGradients(bst.handle, g.ctypes.data_as(C.POINTER(C.c_float)),
                                                  h.ctypes.data_as(C.POINTER(C.c_float)), n))
    return g, h


def eval_metric(eng, bst, d, name):
    """The metric as a double (the eval string prints 6 decimals)."""
    if d is not bst._train:
        d._ensure_raw()
    out = C.c_double(0)
    eng._check(eng.lib().B2_BoosterEvalSet(bst.handle, d.handle, name.encode(), C.byref(out)))
    return out.value


def raises_with(pattern, fn):
    """fn() raises, and the message of the exception or of one of its causes (the public train() reports a failed
    actor and chains the actor's error) matches pattern."""
    with pytest.raises(Exception) as ei:
        fn()
    msgs, e = [], ei.value
    while e is not None:
        msgs.append(str(e))
        e = e.__cause__
    assert any(re.search(pattern, m) for m in msgs), msgs


def class_labels(X, K):
    """K classes from the first two features (NaN counts as 0)."""
    x = np.nan_to_num(X.astype(np.float64))
    return ((np.floor(x[:, 0] * K / 10.0) + (x[:, 1] > 5) * (K // 3 + 1)) % K).astype(np.float32)


def softmax_ref(m):
    """or_transform / transform_kernel in binary32: mx, e_k = expf(m_k - mx), s = sum e_k in class order, p = e / s."""
    m = np.asarray(m, F32)
    e = expf_(m - m.max(axis=1, keepdims=True))
    s = np.zeros(len(m), F32)
    for k in range(m.shape[1]):
        s = s + e[:, k]
    return (e / s[:, None]).astype(F32)


def metric_rows(m, y):
    """Per-row mlogloss terms (float64 of the binary32 p of the true class, clamped at 1e-16f) and merror flags
    (first index of the maximum), the sequence of metric_kernel."""
    m = np.asarray(m, F32)
    n, K = m.shape
    mx = m.max(axis=1)
    s = np.zeros(n, F32)
    for k in range(K):
        s = s + expf_(m[:, k] - mx)
    yi = y.astype(np.int64)
    p = expf_(m[np.arange(n), yi] - mx) / s
    p = np.maximum(p, F32(1e-16))
    return -np.log(p.astype(np.float64)), (np.argmax(m, axis=1) != yi).astype(np.float64)


def weighted_mean(v, w):
    w = np.ones(len(v)) if w is None else w.astype(np.float64)
    return math.fsum(v * w) / math.fsum(w), float(np.sum(np.abs(v * w))) / math.fsum(w)


def check_metric(got, v, w, n, exact=False):
    want, scale = weighted_mean(v, w)
    if exact:
        assert got == want, (got, want)
    else:   # two summation orders of the same doubles (the GPU sums with atomics), then one division
        assert abs(got - want) <= 4 * n * 2.0 ** -53 * scale + 2.0 ** -52 * abs(want), (got, want)


class Reordered:
    """An oracle model grown as num_parallel_tree successive custom-gradient rounds (class order inside each) seen in the
    engine's order (the parallel trees of a class next to each other)."""

    def __init__(self, bst, K, npt):
        self.bst, self.K, self.npt = bst, K, npt
        self.num_trees = bst.num_trees
        self.margin = bst.margin

    def tree(self, i):
        r, rem = divmod(i, self.K * self.npt)
        k, j = divmod(rem, self.npt)
        return self.bst.tree(r * self.K * self.npt + j * self.K + k)

    def predict(self, X):
        return self.bst.predict(X)


def oracle_train(oracle, params, X, y, rounds, weight=None):
    """The oracle's model; num_parallel_tree > 1 grows npt trees per class and round from the round's gradients with
    eta / npt, as the engine does (the oracle has no num_parallel_tree of its own)."""
    npt = int(params.get("num_parallel_tree", 1))
    if npt == 1:
        return oracle.train(params, X, y, rounds, weight=weight)[0]
    K = int(params["num_class"])
    op = {k: v for k, v in params.items() if k != "num_parallel_tree"}
    op["eta"] = float(F32(params.get("eta", 0.3)) / F32(npt))
    cuts = oracle.Cuts.from_data(X, int(params.get("max_bin", 256)), weight=weight)
    bins = cuts.bin(X)
    bst = oracle.Booster(op, cuts)
    bst.init_margin(X.shape[0])
    for _ in range(rounds):
        g, h = oracle.gradients("multi:softprob", bst.margin, y, weight, num_class=K)
        for _ in range(npt):
            bst.boost(bins, y, weight, custom_g=g, custom_h=h)
    return Reordered(bst, K, npt)


# ------------------------------------------------------------------ gradients
@pytest.mark.parametrize("kspec", K_SPECS + ["100"])
def test_gradients_bit_equal_to_oracle(eng, oracle, kspec):
    """Margin rows with ties for the maximum, a leader far enough ahead that the others' p underflow to 0, values near
    +-80 and +-0.0; labels 0, K-1 and K-1 + 0.5; weights 0, 1e-3, 1, 1e3; n = 40,009 (a partial last grid stride)."""
    K = classes(eng, kspec)
    n = 40009
    rng = np.random.RandomState(K)
    M = rng.normal(scale=3.0, size=(n, K)).astype(F32)
    kind = np.arange(n) % 6
    rows = np.arange(n)
    M[kind == 1] = rng.normal(size=(int(np.sum(kind == 1)), 1)).astype(F32)              # all equal: p = 1/K
    sel = rows[kind == 2]                                                                   # the maximum twice
    a, b = rng.randint(0, K, len(sel)), rng.randint(0, K, len(sel))
    M[sel, a] = F32(9.5)
    M[sel, b] = F32(9.5)
    sel = rows[kind == 3]                                                                   # the rest underflow
    M[sel, rng.randint(0, K, len(sel))] = F32(130.0)                                        # > 104 ahead
    sel = rows[kind == 4]                                                                   # near +-80
    M[sel] = (np.where(rng.uniform(size=(len(sel), K)) < 0.5, -80.0, 80.0)
              + rng.uniform(-0.5, 0.5, size=(len(sel), K))).astype(F32)
    sel = rows[kind == 5]                                                                   # +-0.0
    M[sel] = np.where(rng.uniform(size=(len(sel), K)) < 0.5, F32(-0.0), F32(0.0))
    y = np.choose(rng.randint(0, 3, n), [0.0, K - 1.0, K - 0.5]).astype(F32)
    w = np.choose(rng.randint(0, 4, n), [0.0, 1e-3, 1.0, 1e3]).astype(F32)
    X = make_data(n, 3, 2, "uniform")
    dm = eng.DMatrix(X, label=y, weight=w, base_margin=M)
    bst = eng.Booster({"objective": "multi:softprob", "num_class": K, "max_depth": 2}, cache=[dm])
    bst.update(dm, 0)
    g, h = get_gradients(eng, bst, n * K)
    rg, rh = oracle.gradients("multi:softprob", M, y, w, num_class=K)
    g, h = g.reshape(K, n).T, h.reshape(K, n).T          # the engine is class-major [K][n]
    rg, rh = rg.reshape(n, K), rh.reshape(n, K)
    assert np.array_equal(g.view(np.uint32), rg.view(np.uint32)), np.argwhere(g.view(np.uint32) != rg.view(np.uint32))[:10]
    assert np.array_equal(h.view(np.uint32), rh.view(np.uint32)), np.argwhere(h.view(np.uint32) != rh.view(np.uint32))[:10]
    under = (kind == 3) & (w == 1.0)                       # the underflow branch was reached: g in {0, -1}, h clamped
    assert np.all(np.isin(g[under], [0.0, -1.0, 1.0])) and np.all(h[under] == F32(1e-16))


# ------------------------------------------------------------------ trees
@pytest.mark.parametrize("variant", ["plain", "missing_weights", "sampling", "npt2"])
@pytest.mark.parametrize("kspec", ["KF", "KF+1", "40"])
def test_trees_identical_to_oracle(eng, oracle, kspec, variant):
    """At K = KF the class trees replay as a CUDA graph (fused |g|, |h| maxima); above it each class tree runs its own
    absmax pass and direct launches."""
    K = classes(eng, kspec)
    n, f = 20000, 12
    X = make_data(n, f, 40 + K, "uniform", nan_frac=0.1 if variant == "missing_weights" else 0.0)
    y = class_labels(X, K)
    w = np.random.RandomState(K).uniform(0.2, 3.0, n).astype(F32) if variant == "missing_weights" else None
    params = {"objective": "multi:softprob", "num_class": K, "max_depth": 5, "eta": 0.3}
    if variant == "sampling":
        params.update(subsample=0.7, colsample_bynode=0.8, seed=9)
    if variant == "npt2":
        params["num_parallel_tree"] = 2
    obst = oracle_train(oracle, params, X, y, 3, weight=w)
    dm = eng.DMatrix(X, label=y, weight=w)
    ebst = eng.train(params, dm, num_boost_round=3, verbose_eval=False)
    assert ebst.num_trees() == 3 * K * int(params.get("num_parallel_tree", 1))
    assert_same_model(ebst, obst)
    m = ebst.predict(dm, output_margin=True, training=True).reshape(n, K)
    assert np.max(np.abs(m - obst.margin)) <= 1e-5
    if variant in ("plain", "npt2"):
        Xt = make_data(2000, f, 77, "uniform")
        assert np.max(np.abs(ebst.predict(eng.DMatrix(Xt)) - obst.predict(Xt))) <= 1e-5


def test_iteration_range_with_parallel_trees(eng):
    """Tree t adds to class (t / npt) % K: the margin of every iteration range equals the sum of the leaves reached."""
    K = classes(eng, "KF+1")
    X = make_data(4000, 6, 11, "uniform")
    y = class_labels(X, K)
    bst = eng.train({"objective": "multi:softprob", "num_class": K, "max_depth": 3, "num_parallel_tree": 2,
                     "subsample": 0.8, "seed": 1}, eng.DMatrix(X, label=y), 3, verbose_eval=False)
    trees = bst.get_trees()
    Xt = make_data(500, 6, 12, "uniform")
    d = eng.DMatrix(Xt)
    per_round = 2 * K
    for it in ((0, 1), (1, 2), (1, 3), (0, 3)):
        tr = (it[0] * per_round, it[1] * per_round)
        leaves = R.leaf_index(trees, Xt, tree_range=tr).astype(np.int64)
        want = np.full((len(Xt), K), 0.5, F32)
        for j, t in enumerate(range(*tr)):
            want[:, (t // 2) % K] += trees[t]["value"][leaves[:, j]]
        got = bst.predict(d, output_margin=True, iteration_range=it)
        assert np.max(np.abs(got - want)) <= 1e-5, it
        assert np.array_equal(bst.predict(d, iteration_range=it).view(np.uint32), softmax_ref(got).view(np.uint32))


# ------------------------------------------------------------------ metrics
def forced_margins(yv, K, rng):
    """base_margin of a validation matrix: rows 0..199 put the true class 300 below the others (its p underflows, the row
    adds -log(1e-16f)); rows 200..399 tie two classes at 1e9 (the trees' leaves vanish in its ulp of 64), the label
    on the second one for the odd rows: the first index wins the argmax."""
    n = len(yv)
    bm = np.zeros((n, K), F32)
    bm[np.arange(200), yv[:200].astype(np.int64)] = F32(-300.0)
    a = rng.randint(0, K - 1, 200)
    b = a + 1 + (rng.randint(0, K, 200) % (K - 1 - a))
    rows = np.arange(200, 400)
    bm[rows, a] = F32(1e9)
    bm[rows, b] = F32(1e9)
    yv[rows] = np.where(rows % 2 == 1, b, a).astype(F32)
    return bm, a, b


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("kspec", K_SPECS)
def test_metrics_against_float64_reference(eng, kspec, weighted):
    K = classes(eng, kspec)
    rng = np.random.RandomState(3 + K)
    n, nv, f = 20000, 3000, 8
    X = make_data(n, f, 50 + K, "uniform")
    y = class_labels(X, K)
    Xv = make_data(nv, f, 60 + K, "uniform")
    yv = class_labels(Xv, K)
    bm, a, b = forced_margins(yv, K, rng)
    w = rng.uniform(0.5, 2.0, n).astype(F32) if weighted else None
    wv = rng.uniform(0.5, 2.0, nv).astype(F32) if weighted else None
    dm = eng.DMatrix(X, label=y, weight=w)
    dv = eng.DMatrix(Xv, label=yv, weight=wv, base_margin=bm)
    params = {"objective": "multi:softprob", "num_class": K, "max_depth": 4, "eta": 0.3}
    res = {}
    bst = eng.train(params, dm, 2, evals=[(dm, "train"), (dv, "valid")], evals_result=res, verbose_eval=False)
    assert list(res["train"]) == ["mlogloss"]                           # the default metric of multi-class
    for d, lab, ww, m in ((dm, y, w, bst.predict(dm, output_margin=True, training=True)),
                          (dv, yv, wv, bst.predict(dv, output_margin=True))):
        v, e = metric_rows(m, lab)
        check_metric(eval_metric(eng, bst, d, "mlogloss"), v, ww, len(lab))
        check_metric(eval_metric(eng, bst, d, "merror"), e, ww, len(lab), exact=not weighted)
    mv = bst.predict(dv, output_margin=True)
    v, e = metric_rows(mv, yv)
    assert np.all(v[:200] == -np.log(np.float64(F32(1e-16))))         # the underflow rows were reached
    assert np.all(mv[np.arange(200, 400), a] == mv[np.arange(200, 400), b])
    assert np.array_equal(e[200:400], (np.arange(200, 400) % 2 == 1).astype(np.float64))
    # a matrix of underflow rows only: mlogloss is -log(1e-16f)
    du = eng.DMatrix(Xv[:200], label=yv[:200], base_margin=bm[:200])
    vu = -np.log(np.float64(F32(1e-16)))
    assert abs(eval_metric(eng, bst, du, "mlogloss") - vu) <= 4 * 200 * 2.0 ** -53 * vu


# ------------------------------------------------------------------ transform and predict
@pytest.mark.parametrize("kspec", K_SPECS)
def test_transform_and_softmax_argmax(eng, kspec):
    K = classes(eng, kspec)
    rng = np.random.RandomState(70 + K)
    X = make_data(5000, 6, 71, "uniform")
    y = class_labels(X, K)
    Xv = make_data(1000, 6, 72, "uniform")
    yv = class_labels(Xv, K)
    bm, a, b = forced_margins(yv, K, rng)
    bm[400:500] = rng.uniform(-90, 90, size=(100, K)).astype(F32)      # wide margins: exp near both ends
    params = {"objective": "multi:softprob", "num_class": K, "max_depth": 4}
    bst = eng.train(params, eng.DMatrix(X, label=y), 2, verbose_eval=False)
    sm = eng.train(dict(params, objective="multi:softmax"), eng.DMatrix(X, label=y), 2, verbose_eval=False)
    for d in (eng.DMatrix(Xv), eng.DMatrix(Xv, base_margin=bm)):
        m = bst.predict(d, output_margin=True)
        p = bst.predict(d)
        assert np.array_equal(p.view(np.uint32), softmax_ref(m).view(np.uint32))
        ms = sm.predict(d, output_margin=True)
        cls = sm.predict(d)
        assert np.array_equal(cls, np.argmax(ms, axis=1).astype(F32))
    rows = np.arange(200, 400)
    assert np.all(ms[rows, a] == ms[rows, b]) and np.array_equal(cls[rows], a.astype(F32))   # the first index wins


# ------------------------------------------------------------------ SHAP
@pytest.mark.parametrize("kspec,f,depth,rounds,rows", [("KF+1", 10, 5, 3, 200),     # 8 warps in shared memory
                                                       ("32", 100, 4, 2, 100),       # 4 warps
                                                       ("32", 800, 3, 2, 64)])      # global scratch
def test_contribs_at_large_class_counts(eng, kspec, f, depth, rounds, rows):
    """The kernel keeps warps * K * (F+1) doubles in <= 200 KiB of shared memory: K (F+1) = 187 fits 8 warps, 3,232
    fits 4, 25,632 does not fit one and the rows accumulate in global scratch."""
    K = classes(eng, kspec)
    X = make_data(3000, f, 80 + f, "uniform", nan_frac=0.05)
    y = class_labels(X, K)
    bst = eng.train({"objective": "multi:softprob", "num_class": K, "max_depth": depth}, eng.DMatrix(X, label=y),
                    rounds, verbose_eval=False)
    xs = X[:rows]
    d = eng.DMatrix(xs)
    phi = bst.predict(d, pred_contribs=True, strict_shape=True)
    ref = R.shap_contribs(bst.get_trees(), xs, num_class=K, npt=1, base_value=0.5)
    margin = bst.predict(d, output_margin=True).reshape(rows, K)
    tol = 1e-5 * np.maximum(1.0, np.abs(margin))[:, :, None]
    assert phi.shape == (rows, K, f + 1)
    assert np.all(np.abs(phi - ref) <= tol), float(np.max(np.abs(phi - ref)))
    assert np.all(np.abs(phi.astype(np.float64).sum(axis=2) - margin) <= tol[:, :, 0])
    if kspec == "KF+1":
        leaf = bst.predict(d, pred_leaf=True)
        assert np.array_equal(leaf, R.leaf_index(bst.get_trees(), xs))


# ------------------------------------------------------------------ label validation
@pytest.mark.parametrize("kspec", ["3", "KF+1"])
def test_labels_outside_the_classes_fail(eng, kspec):
    K = classes(eng, kspec)
    n = 3000
    X = make_data(n, 4, 90, "uniform")
    y = class_labels(X, K)
    params = {"objective": "multi:softprob", "num_class": K, "max_depth": 3}
    E = eng.XGBoostError
    for bad in (K, -1.0, -0.5, np.nan):
        for row in (0, n - 1):
            yb = y.copy()
            yb[row] = bad
            with pytest.raises(E, match=LABEL_MSG + " for multi:softprob, num_class = %d" % K):
                eng.train(params, eng.DMatrix(X, label=yb), 1, verbose_eval=False)
    with pytest.raises(E, match=LABEL_MSG + " for multi:softmax"):
        eng.train(dict(params, objective="multi:softmax"), eng.DMatrix(X, label=np.where(y == 0, K, y).astype(F32)), 1,
                  verbose_eval=False)
    # K - 0.1 truncates to class K - 1, as xgboost does: the same gradients bit for bit
    grads = []
    for last in (K - 0.1, K - 1.0):
        yl = y.copy()
        yl[::7] = last
        dm = eng.DMatrix(X, label=yl)
        bst = eng.Booster(params, cache=[dm])
        bst.update(dm, 0)
        grads.append(get_gradients(eng, bst, n * K))
    assert all(np.array_equal(u.view(np.uint32), v.view(np.uint32)) for u, v in zip(*grads))
    # an evaluation matrix with one bad label fails the evaluation, training stays possible, a valid matrix evaluates
    Xv = make_data(500, 4, 91, "uniform")
    yv = class_labels(Xv, K)
    dm = eng.DMatrix(X, label=y)
    for bad in (K, -1.0, np.nan):
        for row in (0, 499):
            ybv = yv.copy()
            ybv[row] = bad
            dbad = eng.DMatrix(Xv, label=ybv)
            for metric in ("mlogloss", "merror"):
                with pytest.raises(E, match=LABEL_MSG):
                    eng.train(dict(params, eval_metric=metric), dm, 1, evals=[(dbad, "v")], verbose_eval=False)
    bst = eng.train(params, dm, 2, verbose_eval=False)
    with pytest.raises(E, match=LABEL_MSG):
        bst.eval(dbad)
    good = eng.DMatrix(Xv, label=yv)
    v, _ = metric_rows(bst.predict(good, output_margin=True), yv)
    check_metric(eval_metric(eng, bst, good, "mlogloss"), v, None, len(yv))


def test_labels_outside_the_classes_fail_public_api(eng):
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    X = make_data(2000, 4, 92, "uniform")
    y = class_labels(X, 4)
    y[1234] = 4.0
    raises_with(LABEL_MSG, lambda: train({"objective": "multi:softprob", "num_class": 4}, RayDMatrix(X, y),
                                         num_boost_round=1, ray_params=RayParams(num_actors=1)))


# ------------------------------------------------------------------ save / load and continuation
def test_save_load_and_continuation(eng, oracle, tmp_path):
    K = classes(eng, "KF+1")
    X = make_data(6000, 8, 95, "uniform", nan_frac=0.05)
    y = class_labels(X, K)
    params = {"objective": "multi:softprob", "num_class": K, "max_depth": 4}
    bst = eng.train(params, eng.DMatrix(X, label=y), 2, verbose_eval=False)
    path = str(tmp_path / "m.json")
    bst.save_model(path)
    loaded = eng.Booster(model_file=path)
    Xt = eng.DMatrix(make_data(1000, 8, 96, "uniform", nan_frac=0.05))
    for kw in ({}, {"output_margin": True}):
        assert np.array_equal(bst.predict(Xt, **kw).view(np.uint32), loaded.predict(Xt, **kw).view(np.uint32))
    cont = eng.train(params, eng.DMatrix(X, label=y), 2, xgb_model=path, verbose_eval=False)
    full = eng.train(params, eng.DMatrix(X, label=y), 4, verbose_eval=False)
    assert cont.num_trees() == full.num_trees() == 4 * K
    assert_same_model(cont, oracle.train(params, X, y, 4)[0])
    for u, v in zip(cont.get_trees(), full.get_trees()):
        assert np.array_equal(u["split_feature"], v["split_feature"]) and np.array_equal(u["split_bin"], v["split_bin"])
        assert np.max(np.abs(u["value"] - v["value"])) <= 1e-6


# ------------------------------------------------------------------ two GPUs
@pytest.mark.timeout(300)
def test_two_gpu_model_byte_identical(eng):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, RayShardingMode, train
    K = classes(eng, "KF+1")
    X = make_data(20001, 10, 97, "uniform", nan_frac=0.05)
    y = class_labels(X, K)
    params = {"objective": "multi:softprob", "num_class": K, "max_depth": 5}
    mode = RayShardingMode.INTERLEAVED
    b1 = train(params, RayDMatrix(X, y, sharding=mode), num_boost_round=3, ray_params=RayParams(num_actors=1))
    b2 = train(params, RayDMatrix(X, y, sharding=mode), num_boost_round=3, ray_params=RayParams(num_actors=2))
    assert bytes(b1.save_raw()) == bytes(b2.save_raw())


@pytest.mark.timeout(300)
def test_two_gpu_bad_label_on_rank_1_fails(eng):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, RayShardingMode, train
    K = classes(eng, "KF+1")
    X = make_data(4001, 6, 98, "uniform")
    y = class_labels(X, K)
    params = {"objective": "multi:softprob", "num_class": K, "max_depth": 3}
    mode = RayShardingMode.INTERLEAVED
    yb = y.copy()
    yb[3] = K          # an odd row: INTERLEAVED gives it to rank 1 only
    raises_with(LABEL_MSG, lambda: train(params, RayDMatrix(X, yb, sharding=mode), num_boost_round=1,
                                         ray_params=RayParams(num_actors=2)))
    dv = RayDMatrix(X, yb, sharding=mode)     # the same row in an evaluation matrix: the count travels with the sums
    raises_with(LABEL_MSG, lambda: train(params, RayDMatrix(X, y, sharding=mode), num_boost_round=1, evals=[(dv, "v")],
                                         ray_params=RayParams(num_actors=2)))
