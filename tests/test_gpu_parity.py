"""GPU parity tests: the sm_90a engine (through the C-ABI, via xgboost_ray_b200.engine) against the
CPU oracle on the same seeded inputs.  Integer / index results are bit-exact; leaf values are
compared with the tolerance BASELINE.json's north_star states (1e-5)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LEAF_TOL = 1e-5


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def make_data(n, f, seed, kind="uniform", nan_frac=0.0):
    rng = np.random.RandomState(seed)
    if kind == "uniform":
        X = rng.uniform(0, 10, size=(n, f)).astype(np.float32)
    elif kind == "lowcard":
        X = rng.randint(0, 5, size=(n, f)).astype(np.float32)
    elif kind == "mixed":
        X = rng.normal(size=(n, f)).astype(np.float32)
        X[:, ::3] = np.round(X[:, ::3] * 2)          # heavy ties
        X[:, 1] = 3.0                                 # constant feature
        if f > 2:
            X[:, 2] = (X[:, 2] > 0).astype(np.float32)  # binary feature
    if nan_frac > 0:
        X[rng.uniform(size=X.shape) < nan_frac] = np.nan
    return X


# ------------------------------------------------------------------ histogram kernel (a10)
# with B2_HIST_NARROW=1 F = 32 a + r, 0 < r <= 16 puts the r leftover features into a NARROW last group (one lane per row,
# pow2ceil(r) steps, 32 / w shared-memory replicas): widths 1, 2, 4, 8, 16 alone and behind full groups are all covered
@pytest.mark.parametrize("narrow", [0, 1])
@pytest.mark.parametrize("n,f", [(1, 1), (17, 3), (1000, 28), (5000, 100), (3000, 50), (2000, 200), (4097, 33),
                                 (3001, 2), (2500, 34), (3000, 12), (777, 16), (2000, 48), (1500, 7), (6000, 104),
                                 (1500, 800)])   # more groups than the pair plan holds: one group per CTA
def test_hist_kernel_bit_exact(eng, oracle, n, f, narrow):
    rng = np.random.RandomState(n + f)
    bins = rng.randint(0, 256, size=(n, f)).astype(np.uint8)
    qg = rng.randint(-(1 << 18), 1 << 18, size=n).astype(np.int32)
    qh = rng.randint(0, 1 << 18, size=n).astype(np.int32)
    ref = oracle.hist_int(bins, qg, qh)
    got, _ = eng.hist_build_raw(bins, qg, qh, window_rows=4096, chunk_rows=512, narrow=narrow)
    assert np.array_equal(ref, got)


def test_hist_kernel_adversarial_and_windows(eng, oracle):
    n, f = 20000, 37
    rng = np.random.RandomState(7)
    bins = rng.randint(0, 256, size=(n, f)).astype(np.uint8)
    bins[:, 0] = 9          # constant feature: every row hits the same cell
    bins[:, 1] = bins[:, 1] & 1   # binary feature
    bins[:, 2] = 255
    qg = np.full(n, (1 << 18), np.int32)     # extreme values: the guard interval for 18 bits is 2^12 rows
    qg[::2] = -(1 << 18)
    qg[: n // 2] = (1 << 18)                 # long same-sign runs on the constant feature: its cell saturates
    qh = np.full(n, (1 << 18), np.int32)
    ref = oracle.hist_int(bins, qg, qh)
    for window, chunk in ((4096, 512), (1024, 256), (4096, 4096), (4096, 8192)):
        got, _ = eng.hist_build_raw(bins, qg, qh, window_rows=window, chunk_rows=chunk)
        assert np.array_equal(ref, got), (window, chunk)


def test_hist_kernel_gather(eng, oracle):
    n, f = 30000, 100
    rng = np.random.RandomState(11)
    bins = rng.randint(0, 256, size=(n, f)).astype(np.uint8)
    qg = rng.randint(-1000, 1000, size=n).astype(np.int32)
    qh = rng.randint(0, 1000, size=n).astype(np.int32)
    for nsel in (0, 1, 15, 16, 17, 4999, 30000):
        ridx = rng.permutation(n)[:nsel].astype(np.int32)
        ref = oracle.hist_int(bins, qg, qh, ridx) if nsel else np.zeros((f, 256, 2), np.int64)
        got, _ = eng.hist_build_raw(bins, qg, qh, ridx=ridx, window_rows=4096, chunk_rows=1024)
        assert np.array_equal(ref, got), nsel


def test_hist_kernel_variants_bit_exact(oracle):
    """Every kernel variant (TMA-staged rows; 3x8 / 2x16 warps with one group per CTA; 32 warps with two groups
    per CTA) produces the same integers."""
    import os
    import subprocess
    import sys
    code = (
        "import numpy as np, sys; sys.path.insert(0, %r)\n"
        "from xgboost_ray_b200 import engine as E\n"
        "from oracle import oracle as O\n"
        "rng = np.random.RandomState(3); n = 70001\n"
        "qg = rng.randint(-(1 << 18), 1 << 18, size=n).astype(np.int32); qh = rng.randint(0, 1 << 18, size=n).astype(np.int32)\n"
        "sel = np.sort(rng.choice(n, 33333, replace=False)).astype(np.int32)\n"
        "for f in (100, 70, 17, 96, 105, 112):\n"   # 4, 3 (odd: a half-empty CTA in the two-group variant) and 1 feature groups; 96..112: the all-groups-per-CTA kernel
        "    bins = rng.randint(0, 256, size=(n, f)).astype(np.uint8)\n"
        "    for ridx in (None, sel):\n"
        "        ref = O.hist_int(bins, qg, qh, ridx); got, _ = E.hist_build_raw(bins, qg, qh, ridx=ridx, window_rows=4096, chunk_rows=2048)\n"
        "        assert np.array_equal(ref, got), (f, ridx is None)\n"
        "print('variant ok')\n") % os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for env in ({"B2_HIST_TMA": "1"}, {"B2_HIST_VARIANT": "0"}, {"B2_HIST_VARIANT": "1"}, {"B2_HIST_VARIANT": "2"},
                {"B2_HIST_VARIANT": "3"}, {"B2_HIST_VARIANT": "4"}, {"B2_HIST_ALIGNED": "1"}, {"B2_HIST_NARROW": "1"},
                {"B2_HIST_NARROW": "1", "B2_HIST_ALIGNED": "1"}, {"B2_HIST_VARIANT": "2", "B2_HIST_NARROW": "1"}):
        r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=300)
        assert r.returncode == 0 and "variant ok" in r.stdout, (env, r.stdout[-500:], r.stderr[-1500:])


# ------------------------------------------------------------------ cuts and bins (a7, a8)
@pytest.mark.parametrize("kind,nan_frac,n,f", [("uniform", 0.0, 5000, 7), ("lowcard", 0.0, 3000, 5),
                                               ("mixed", 0.0, 4000, 9), ("mixed", 0.1, 4000, 9),
                                               ("uniform", 0.3, 700, 33), ("uniform", 0.0, 200, 3)])
def test_cuts_and_bins_bit_exact(eng, oracle, kind, nan_frac, n, f):
    X = make_data(n, f, 3, kind, nan_frac)
    if nan_frac > 0:
        X[:, -1] = np.nan  # all-missing feature
    oc = oracle.Cuts.from_data(X, 256)
    dm = eng.DMatrix(X)
    dm._ensure_quantized(256, keep_raw=True)
    ptrs, vals, mins, hm = dm.get_cuts()
    assert np.array_equal(ptrs, oc.ptrs)
    assert np.array_equal(vals.view(np.uint32), oc.vals.view(np.uint32))
    assert np.array_equal(mins.view(np.uint32), oc.mins.view(np.uint32))
    assert np.array_equal(hm, oc.has_missing)
    assert np.array_equal(dm.get_bins(), oc.bin(X))


def test_cuts_small_max_bin(eng, oracle):
    X = make_data(6000, 4, 5, "uniform")
    for mb in (2, 16, 64):
        oc = oracle.Cuts.from_data(X, mb)
        dm = eng.DMatrix(X)
        dm._ensure_quantized(mb)
        ptrs, vals, mins, hm = dm.get_cuts()
        assert np.array_equal(ptrs, oc.ptrs)
        assert np.array_equal(vals.view(np.uint32), oc.vals.view(np.uint32))


# ------------------------------------------------------------------ whole trees (a9-a14)
def assert_same_model(eng_bst, or_bst, leaf_tol=LEAF_TOL):
    trees = eng_bst.get_trees()
    assert len(trees) == or_bst.num_trees
    for i, t in enumerate(trees):
        o = or_bst.tree(i)
        assert len(t["left"]) == o.n_nodes, "tree %d node count" % i
        assert np.array_equal(t["left"], o.left) and np.array_equal(t["right"], o.right), "tree %d topology" % i
        assert np.array_equal(t["split_feature"], o.split_feature), "tree %d split features" % i
        assert np.array_equal(t["split_bin"], o.split_bin), "tree %d split bins" % i
        assert np.array_equal(t["default_left"], o.default_left), "tree %d default directions" % i
        nanc = np.isnan(o.split_cond)      # partition-based categorical splits store NaN
        assert np.array_equal(np.isnan(t["split_cond"]), nanc), "tree %d NaN conds" % i
        assert np.array_equal(t["split_cond"][~nanc].view(np.uint32), o.split_cond[~nanc].view(np.uint32)), "tree %d conds" % i
        assert np.array_equal(t["split_type"], o.split_type), "tree %d split types" % i
        assert np.array_equal(t["cat_bits"], o.cat_bits), "tree %d category sets" % i
        leaf = o.split_feature < 0
        assert np.max(np.abs(t["value"][leaf] - o.value[leaf])) <= leaf_tol, "tree %d leaf values" % i
        assert np.allclose(t["loss_chg"], o.loss_chg, rtol=0, atol=0), "tree %d loss_chg" % i


def run_both(eng, oracle, params, X, y, rounds, weight=None, base_margin=None):
    obst, _ = oracle.train(params, X, y, rounds, weight=weight, base_margin=base_margin)
    dm = eng.DMatrix(X, label=y, weight=weight, base_margin=base_margin)
    ebst = eng.train(params, dm, num_boost_round=rounds, verbose_eval=False)
    return ebst, obst, dm


@pytest.mark.parametrize("objective", ["reg:squarederror", "binary:logistic"])
@pytest.mark.parametrize("n,f,depth", [(2000, 10, 4), (20000, 28, 6), (50000, 100, 8)])
def test_trees_identical(eng, oracle, objective, n, f, depth):
    X = make_data(n, f, 21, "uniform")
    rng = np.random.RandomState(4)
    lin = X[:, : min(f, 5)].sum(axis=1) + np.sin(X[:, 0]) + rng.normal(scale=0.5, size=n)
    y = lin.astype(np.float32) if objective == "reg:squarederror" else (lin > np.median(lin)).astype(np.float32)
    params = {"objective": objective, "max_depth": depth, "eta": 0.3, "base_score": 0.5, "hist_qbits": 18}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 5)
    assert_same_model(ebst, obst)
    # margin cache == oracle margin cache
    m = ebst.predict(dm, output_margin=True, training=True)
    assert np.max(np.abs(m - obst.margin[:, 0])) <= 1e-5
    # predict on raw floats == oracle predict
    Xt = make_data(3000, f, 99, "uniform")
    pe = ebst.predict(eng.DMatrix(Xt))
    po = obst.predict(Xt)
    assert np.max(np.abs(pe - po)) <= 1e-5


def test_trees_identical_missing_and_weights(eng, oracle):
    n, f = 8000, 12
    X = make_data(n, f, 5, "mixed", nan_frac=0.15)
    rng = np.random.RandomState(1)
    y = (np.nan_to_num(X[:, 0]) + np.nan_to_num(X[:, 3]) > 0).astype(np.float32)
    w = rng.uniform(0.5, 2.0, size=n).astype(np.float32)
    params = {"objective": "binary:logistic", "max_depth": 5, "base_score": 0.5, "min_child_weight": 2.0,
              "lambda": 0.5, "gamma": 0.01}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 6, weight=w)
    assert_same_model(ebst, obst)
    assert any((t["default_left"] == 1).any() for t in ebst.get_trees()), "test data should exercise default-left"
    Xt = make_data(1000, f, 77, "mixed", nan_frac=0.2)
    assert np.max(np.abs(ebst.predict(eng.DMatrix(Xt)) - obst.predict(Xt))) <= 1e-5


def test_trees_identical_multiclass(eng, oracle):
    n, f, K = 6000, 8, 4
    X = make_data(n, f, 8, "uniform")
    y = (np.floor(X[:, 0] / 2.5).astype(int) % K).astype(np.float32)
    params = {"objective": "multi:softprob", "num_class": K, "max_depth": 4, "base_score": 0.5}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 3)
    assert ebst.num_trees() == 3 * K
    assert_same_model(ebst, obst)
    pe = ebst.predict(eng.DMatrix(X))
    assert pe.shape == (n, K)
    assert np.max(np.abs(pe - obst.predict(X))) <= 1e-5


def test_toy_matrix_known_answers(eng, oracle):
    """Ported relational known-answers of xgboost_ray/tests/test_end_to_end.py:72-139."""
    x = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 1], [0, 0, 1, 0]] * 8, np.float32)
    y = np.array([0, 1, 2, 3] * 8, np.float32)
    params = {"max_depth": 2, "objective": "multi:softmax", "num_class": 4, "nthread": 1, "booster": "gbtree"}
    bst = eng.train(params, eng.DMatrix(x, label=y), num_boost_round=2, verbose_eval=False)
    assert list(bst.predict(eng.DMatrix(x))) == list(y)
    test_x = eng.DMatrix(np.array([[0, 0, 1, 1], [0, 0, 1, 0]], np.float32))
    b1 = eng.train(params, eng.DMatrix(x[::2], label=y[::2]), num_boost_round=2, verbose_eval=False)
    assert list(b1.predict(test_x)) == [2, 2]
    b2 = eng.train(params, eng.DMatrix(x[1::2], label=y[1::2]), num_boost_round=2, verbose_eval=False)
    assert list(b2.predict(test_x)) == [3, 3]


def test_metrics_match_oracle(eng, oracle):
    n, f = 5000, 6
    X = make_data(n, f, 2, "uniform")
    y = (X[:, 0] > 5).astype(np.float32)
    params = {"objective": "binary:logistic", "max_depth": 3, "base_score": 0.5, "eval_metric": ["logloss", "error"]}
    dm = eng.DMatrix(X, label=y)
    Xv = make_data(1000, f, 3, "uniform")
    yv = (Xv[:, 0] > 5).astype(np.float32)
    dv = eng.DMatrix(Xv, label=yv)
    res = {}
    ebst = eng.train(params, dm, num_boost_round=4, evals=[(dm, "train"), (dv, "valid")], evals_result=res,
                     verbose_eval=False)
    obst, _ = oracle.train(params, X, y, 4)
    assert abs(res["train"]["logloss"][-1] - obst.metric("logloss", obst.margin, y)) < 1e-6
    assert abs(res["train"]["error"][-1] - obst.metric("error", obst.margin, y)) < 1e-9
    mv = obst.predict_margin(Xv)
    assert abs(res["valid"]["logloss"][-1] - obst.metric("logloss", mv, yv)) < 1e-6
    assert len(res["valid"]["logloss"]) == 4
    # metrics see the transformed prediction: rmse / mae of a logistic model compare the PROBABILITY with the label,
    # error / logloss of a squared-error model use the raw value (test_end_to_end.py:449 asks for "error" there)
    res2 = {}
    eng.train(dict(params, eval_metric=["rmse", "mae"]), dm, num_boost_round=2, evals=[(dm, "train")], evals_result=res2,
              verbose_eval=False)
    ob2, _ = oracle.train(params, X, y, 2)
    p = ob2.predict(X)
    assert abs(res2["train"]["rmse"][-1] - float(np.sqrt(np.mean((p - y) ** 2)))) < 1e-6
    assert abs(res2["train"]["mae"][-1] - float(np.mean(np.abs(p - y)))) < 1e-6
    assert abs(res2["train"]["rmse"][-1] - ob2.metric("rmse", ob2.margin, y)) < 1e-7
    res3 = {}
    reg = {"objective": "reg:squarederror", "max_depth": 3, "base_score": 0.5, "eval_metric": ["rmse", "error"]}
    eng.train(reg, dm, num_boost_round=2, evals=[(dm, "train")], evals_result=res3, verbose_eval=False)
    ob3, _ = oracle.train(reg, X, y, 2)
    raw = ob3.predict(X)
    assert abs(res3["train"]["error"][-1] - float(np.mean((raw > 0.5) != (y > 0.5)))) < 1e-9
    with pytest.raises(eng.XGBoostError, match="does not fit"):
        eng.train(dict(reg, eval_metric="mlogloss"), dm, num_boost_round=1, evals=[(dm, "train")], verbose_eval=False)


def test_custom_objective_and_continuation(eng, oracle):
    n, f = 4000, 5
    X = make_data(n, f, 12, "uniform")
    y = (X[:, 1] * 0.5 + X[:, 2]).astype(np.float32)
    params = {"objective": "reg:squarederror", "max_depth": 4, "base_score": 0.5}

    def sq(pred, d):
        return pred - d.get_label(), np.ones_like(pred)

    a = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=4, verbose_eval=False)
    b = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=4, obj=sq, verbose_eval=False)
    ta, tb = a.get_trees(), b.get_trees()
    for u, v in zip(ta, tb):
        assert np.array_equal(u["split_feature"], v["split_feature"]) and np.array_equal(u["split_bin"], v["split_bin"])
    # 2 + 2 continued == 4 uninterrupted (test_fault_tolerance.py:401-444 relational known-answer)
    c = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=2, verbose_eval=False)
    d = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=2, xgb_model=c, verbose_eval=False)
    assert d.num_trees() == 4
    for u, v in zip(ta, d.get_trees()):
        assert np.array_equal(u["split_feature"], v["split_feature"]) and np.array_equal(u["split_bin"], v["split_bin"])
        assert np.max(np.abs(u["value"] - v["value"])) <= 1e-6
    # pickle round trip predicts identically (model object must be picklable, main.py:619)
    import pickle
    e = pickle.loads(pickle.dumps(a))
    dmx = eng.DMatrix(X)
    assert np.array_equal(a.predict(dmx), e.predict(dmx))
    assert a.get_dump(dump_format="json") == e.get_dump(dump_format="json")


def test_errors_surface(eng):
    X = make_data(100, 3, 1)
    with pytest.raises(eng.XGBoostError):
        eng.train({"objective": "rank:pairwise"}, eng.DMatrix(X, label=X[:, 0]), 1, verbose_eval=False)
    with pytest.raises(eng.XGBoostError):
        eng.train({"objective": "reg:squarederror"}, eng.DMatrix(X), 1, verbose_eval=False)  # no labels
    with pytest.raises(eng.XGBoostError):
        eng.train({"max_bin": 1000}, eng.DMatrix(X, label=X[:, 0]), 1, verbose_eval=False)


# ------------------------------------------------------------------ edge cases of the device-driven level loop
@pytest.mark.parametrize("case", ["constant_label", "depth1", "tiny", "wide200", "small_bins", "multiclass_missing",
                                  "deep_sparse_tree"])
def test_edge_cases_identical(eng, oracle, case):
    rng = np.random.RandomState(17)
    w = None
    if case == "constant_label":          # no split is ever valid: every tree is a single leaf
        X = make_data(3000, 6, 1); y = np.full(3000, 2.5, np.float32)
        params = {"objective": "reg:squarederror", "max_depth": 5, "base_score": 0.5}
    elif case == "depth1":
        X = make_data(5000, 9, 2); y = (X[:, 4] > 3).astype(np.float32)
        params = {"objective": "binary:logistic", "max_depth": 1, "base_score": 0.5}
    elif case == "tiny":                  # fewer rows than one warp iteration / one stage
        X = make_data(13, 3, 3); y = X[:, 0].astype(np.float32)
        params = {"objective": "reg:squarederror", "max_depth": 4, "base_score": 0.5, "min_child_weight": 0.0}
    elif case == "wide200":               # 7 feature groups
        X = make_data(6000, 200, 4); y = (X[:, 150] + X[:, 7] * 0.5 + rng.normal(size=6000)).astype(np.float32)
        params = {"objective": "reg:squarederror", "max_depth": 4, "base_score": 0.5}
    elif case == "small_bins":
        X = make_data(8000, 10, 5); y = (np.sin(X[:, 0]) + X[:, 1]).astype(np.float32)
        params = {"objective": "reg:squarederror", "max_depth": 6, "base_score": 0.5, "max_bin": 16}
    elif case == "multiclass_missing":
        X = make_data(5000, 7, 6, "mixed", nan_frac=0.2); y = rng.randint(0, 3, size=5000).astype(np.float32)
        w = rng.uniform(0.1, 3.0, size=5000).astype(np.float32)
        params = {"objective": "multi:softprob", "num_class": 3, "max_depth": 5, "base_score": 0.5, "alpha": 0.1}
    else:                                  # gamma prunes most branches: ragged trees, many early leaves
        X = make_data(20000, 8, 7); y = (X[:, 0] > 9.5).astype(np.float32) * 5 + rng.normal(scale=0.05, size=20000).astype(np.float32)
        params = {"objective": "reg:squarederror", "max_depth": 10, "base_score": 0.5, "gamma": 5.0, "eta": 0.5}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 3, weight=w)
    assert_same_model(ebst, obst)
    K = int(params.get("num_class", 1))
    m = ebst.predict(dm, output_margin=True, training=True).reshape(len(X), K)
    assert np.max(np.abs(m - obst.margin)) <= 1e-5
    if case == "constant_label":
        assert all(len(t["left"]) == 1 for t in ebst.get_trees())
    if case == "deep_sparse_tree":
        assert any(1 < len(t["left"]) < 2 ** 11 - 1 for t in ebst.get_trees())


def test_config_c2_shape_higgs_like(eng, oracle):
    """BASELINE config C2 at test size: 28 fp32 features (21 N(0,1) + 7 heavy-tailed exp(N)), binary:logistic,
    256 bins, depth 6, one GPU -- one feature group, heavy ties in none, long tails in some cuts."""
    rng = np.random.RandomState(1234)
    n = 200_000
    X = rng.normal(size=(n, 28)).astype(np.float32)
    X[:, 21:] = np.exp(X[:, 21:])
    wv = rng.normal(size=8).astype(np.float32)
    logit = X[:, :8] @ wv + 0.5 * X[:, 0] * X[:, 1]
    y = (rng.uniform(size=n) < 1.0 / (1.0 + np.exp(-logit))).astype(np.float32)
    params = {"objective": "binary:logistic", "max_depth": 6, "eta": 0.3, "base_score": 0.5, "max_bin": 256,
              "eval_metric": ["logloss", "error"]}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 8)
    assert_same_model(ebst, obst)
    p = ebst.predict(eng.DMatrix(X[:5000]))
    assert np.max(np.abs(p - obst.predict(X[:5000]))) <= 1e-5
    assert np.mean((p > 0.5) == (y[:5000] > 0.5)) > 0.7


# ------------------------------------------------------------------ categorical features (A.2 / A.6 / A.8, config C5)
CAT_TYPES = ["q", "q", "q", "c", "c", "c"]
IS_CAT = [0, 0, 0, 1, 1, 1]


def make_cat_data(n, seed, nan_frac=0.0):
    rng = np.random.RandomState(seed)
    Xn = rng.uniform(0, 10, size=(n, 3))
    X = np.column_stack([Xn, rng.randint(0, 3, size=n), rng.randint(0, 20, size=n), rng.randint(0, 200, size=n)]).astype(np.float32)
    score = (Xn[:, 0] > 5) * 1.0 + (X[:, 3] == 2) * 1.5 + (X[:, 4] % 3 == 0) * 2.0 + (X[:, 5] % 7 < 2) * 1.0
    if nan_frac > 0:
        X[rng.uniform(size=X.shape) < nan_frac] = np.nan
    return X, score.astype(np.float32), rng


def run_both_cat(eng, oracle, params, X, y, rounds):
    obst, _ = oracle.train(params, X, y, rounds, is_cat=IS_CAT)
    dm = eng.DMatrix(X, label=y, feature_types=CAT_TYPES, enable_categorical=True)
    ebst = eng.train(params, dm, num_boost_round=rounds, verbose_eval=False)
    return ebst, obst, dm


@pytest.mark.parametrize("nan_frac", [0.0, 0.1])
def test_categorical_cuts_and_bins_bit_exact(eng, oracle, nan_frac):
    X, _, _ = make_cat_data(20000, 31, nan_frac)
    cuts = oracle.Cuts.from_data(X, 256, is_cat=IS_CAT)
    dm = eng.DMatrix(X, feature_types=CAT_TYPES, enable_categorical=True)
    dm._ensure_quantized(256)
    ptrs, vals, mins, hm = dm.get_cuts()
    assert np.array_equal(ptrs, cuts.ptrs) and np.array_equal(vals.view(np.uint32), cuts.vals.view(np.uint32))
    assert np.array_equal(hm, cuts.has_missing)
    assert np.array_equal(dm.get_bins(), cuts.bin(X))


@pytest.mark.parametrize("objective,extra", [
    ("reg:squarederror", {}), ("reg:squarederror", {"max_cat_to_onehot": 1}), ("reg:squarederror", {"max_cat_threshold": 8}),
    ("reg:squarederror", {"max_cat_to_onehot": 32, "min_child_weight": 50}), ("binary:logistic", {}),
])
@pytest.mark.parametrize("nan_frac", [0.0, 0.08])
def test_categorical_trees_identical(eng, oracle, objective, extra, nan_frac):
    X, score, rng = make_cat_data(30000, 33, nan_frac)
    y = score + rng.normal(scale=0.3, size=len(score)).astype(np.float32)
    if objective == "binary:logistic":
        y = (y > 2.5).astype(np.float32)
    params = dict({"objective": objective, "max_depth": 6, "eta": 0.3, "base_score": 0.5}, **extra)
    ebst, obst, dm = run_both_cat(eng, oracle, params, X, y, 5)
    assert_same_model(ebst, obst)
    types = np.concatenate([t["split_type"][t["split_feature"] >= 0] for t in ebst.get_trees()])
    assert types.any() and not types.all()                      # both numeric and categorical splits were chosen
    assert np.max(np.abs(ebst.predict(dm, output_margin=True) - obst.predict(X, output_margin=True))) <= LEAF_TOL


def test_categorical_multiclass_and_model_io(eng, oracle, tmp_path):
    import pickle
    X, score, rng = make_cat_data(20000, 35, 0.05)
    y = np.clip(np.round(score), 0, 4).astype(np.float32)
    params = {"objective": "multi:softprob", "num_class": 5, "max_depth": 5, "eta": 0.4}
    ebst, obst, dm = run_both_cat(eng, oracle, params, X, y, 3)
    assert_same_model(ebst, obst)
    Xt = X[:500].copy()
    Xt[:50, 4] = 150.0           # categories the training data never had in this column
    Xt[50:60, 5] = 231.0
    dt = eng.DMatrix(Xt, feature_types=CAT_TYPES, enable_categorical=True)
    want = obst.predict(Xt)
    got = ebst.predict(dt)
    assert np.max(np.abs(got - want)) <= LEAF_TOL
    # JSON model round trip (categories / categories_nodes / categories_segments / categories_sizes / split_type)
    f = str(tmp_path / "cat.json")
    ebst.save_model(f)
    import json
    tr = json.load(open(f))["learner"]["gradient_booster"]["model"]["trees"]
    assert any(t["categories_nodes"] for t in tr) and all(len(t["split_type"]) == len(t["left_children"]) for t in tr)
    for t in tr:
        assert sum(t["categories_sizes"]) == len(t["categories"]) and sum(t["split_type"]) == len(t["categories_nodes"])
    b2 = eng.Booster(model_file=f)
    assert np.array_equal(b2.predict(dt), got)
    b3 = pickle.loads(pickle.dumps(ebst))
    assert np.array_equal(b3.predict(dt), got)
    assert b3.get_dump(dump_format="json") == ebst.get_dump(dump_format="json")
    assert any(":{" in d for d in ebst.get_dump())              # text dump lists the category set


def test_categorical_pandas_category_dtype(eng, oracle):
    import pandas as pd
    X, score, rng = make_cat_data(5000, 37, 0.0)
    df = pd.DataFrame({"a": X[:, 0], "b": X[:, 1], "c": X[:, 2],
                       "k3": pd.Categorical(X[:, 3].astype(int)), "k20": pd.Categorical(X[:, 4].astype(int)),
                       "k200": pd.Categorical(X[:, 5].astype(int))})
    with pytest.raises(eng.XGBoostError):
        eng.DMatrix(df, label=score)
    codes = np.column_stack([X[:, :3]] + [df[c].cat.codes.to_numpy() for c in ("k3", "k20", "k200")]).astype(np.float32)
    params = {"objective": "reg:squarederror", "max_depth": 4, "eta": 0.5}
    obst, _ = oracle.train(params, codes, score, 3, is_cat=IS_CAT)
    ebst = eng.train(params, eng.DMatrix(df, label=score, enable_categorical=True), num_boost_round=3, verbose_eval=False)
    assert_same_model(ebst, obst)


def test_categorical_invalid_codes_error(eng):
    X = np.array([[0.0, 1.0], [1.0, 2.5]], np.float32)
    dm = eng.DMatrix(X, label=[0, 1], feature_types=["q", "c"], enable_categorical=True)
    with pytest.raises(eng.XGBoostError, match="category codes"):
        dm._ensure_quantized(256)
    with pytest.raises(eng.XGBoostError, match="enable_categorical"):
        eng.DMatrix(X, feature_types=["q", "c"])


@pytest.mark.parametrize("extra", [{"scale_pos_weight": 4.0}, {"max_delta_step": 0.7}, {"max_delta_step": 1.5, "alpha": 0.5},
                                   {"scale_pos_weight": 0.25, "max_delta_step": 0.3, "min_child_weight": 3.0}])
def test_trees_identical_scale_pos_weight_and_max_delta_step(eng, oracle, extra):
    X = make_data(20000, 20, 61, "uniform", nan_frac=0.03)
    rng = np.random.RandomState(62)
    y = ((np.nan_to_num(X[:, 0]) + np.nan_to_num(X[:, 3]) + rng.normal(size=len(X))) > 13).astype(np.float32)   # ~10 % positives
    params = dict({"objective": "binary:logistic", "max_depth": 5, "eta": 0.3, "base_score": 0.5}, **extra)
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 4)
    assert_same_model(ebst, obst)


def test_unsupported_parameters_fail_loudly(eng):
    X = make_data(100, 3, 1)
    dm = eng.DMatrix(X, label=X[:, 0])
    for bad in ({"sampling_method": "gradient_based"}, {"grow_policy": "lossguide"}, {"max_leaves": 8},
                {"monotone_constraints": "(1,0,0)"}, {"max_bin": 1024}):
        with pytest.raises(eng.XGBoostError, match="not supported"):
            eng.train(dict({"objective": "reg:squarederror"}, **bad), dm, num_boost_round=1, verbose_eval=False)


@pytest.mark.parametrize("nan_frac", [0.0, 0.1])
@pytest.mark.parametrize("max_bin", [16, 256])
def test_weighted_sketch_cuts_bit_exact(eng, oracle, nan_frac, max_bin):
    X = make_data(30000, 12, 71, "mixed", nan_frac)
    rng = np.random.RandomState(72)
    w = rng.gamma(2.0, 1.0, size=len(X)).astype(np.float32)
    w[::13] = 0.0                                               # zero-weight rows stay in the summary with no mass
    cuts = oracle.Cuts.from_data(X, max_bin, weight=w)
    dm = eng.DMatrix(X, weight=w)
    dm._ensure_quantized(max_bin)
    ptrs, vals, mins, hm = dm.get_cuts()
    assert np.array_equal(ptrs, cuts.ptrs) and np.array_equal(vals.view(np.uint32), cuts.vals.view(np.uint32))
    assert np.array_equal(mins.view(np.uint32), cuts.mins.view(np.uint32)) and np.array_equal(hm, cuts.has_missing)
    assert np.array_equal(dm.get_bins(), cuts.bin(X))
    unweighted = oracle.Cuts.from_data(X, max_bin)
    assert max_bin == 256 or not np.array_equal(unweighted.vals, cuts.vals)   # the weights matter
    bad = w.copy(); bad[5] = -2.0
    with pytest.raises(eng.XGBoostError, match="weights"):
        eng.DMatrix(X, weight=bad)._ensure_quantized(max_bin)


# ------------------------------------------------------------------ row / column sampling (sampling.cuh)
@pytest.mark.parametrize("extra", [
    {"subsample": 0.5, "seed": 7}, {"colsample_bytree": 0.5}, {"colsample_bylevel": 0.4, "seed": 3},
    {"colsample_bynode": 0.3, "seed": 11}, {"subsample": 0.8, "colsample_bytree": 0.7, "colsample_bylevel": 0.7,
                                           "colsample_bynode": 0.5, "seed": 2024},
])
def test_trees_identical_with_sampling(eng, oracle, extra):
    X = make_data(20000, 40, 81, "uniform", nan_frac=0.02)
    rng = np.random.RandomState(82)
    y = (np.nan_to_num(X[:, :8]).sum(axis=1) + rng.normal(size=len(X))).astype(np.float32)
    params = dict({"objective": "reg:squarederror", "max_depth": 5, "eta": 0.3, "base_score": 0.5}, **extra)
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 4)
    assert_same_model(ebst, obst)
    plain, _ = oracle.train({k: v for k, v in params.items() if k in ("objective", "max_depth", "eta", "base_score")}, X, y, 1)
    assert not np.array_equal(plain.tree(0).split_feature, obst.tree(0).split_feature) or "subsample" in extra


def test_sampling_with_categorical_and_multiclass(eng, oracle):
    X, score, rng = make_cat_data(20000, 83, 0.03)
    y = np.clip(np.round(score), 0, 4).astype(np.float32)
    params = {"objective": "multi:softprob", "num_class": 5, "max_depth": 4, "eta": 0.4, "subsample": 0.7,
              "colsample_bynode": 0.5, "seed": 5}
    ebst, obst, dm = run_both_cat(eng, oracle, params, X, y, 2)
    assert_same_model(ebst, obst)


def test_feature_weights_known_answer(eng, oracle):
    """test_end_to_end.py:429-467: feature_weights = 0..9 with colsample_bynode=0.1 -> f0 never splits, f9 most often."""
    rng = np.random.RandomState(1994)
    X = rng.randn(1000, 10).astype(np.float32)
    y = rng.randn(1000).astype(np.float32)
    fw = np.arange(10, dtype=np.float32)
    params = {"objective": "reg:squarederror", "colsample_bynode": 0.1, "max_depth": 6}
    dm = eng.DMatrix(X, label=y)
    dm.set_info(feature_weights=fw)
    ebst = eng.train(params, dm, num_boost_round=60, verbose_eval=False)
    fmap = ebst.get_fscore()
    assert fmap.get("f0") is None and max(fmap.values()) == fmap.get("f9")
    obst, _ = oracle.train(params, X, y, 60, feature_weights=fw)
    assert_same_model(ebst, obst)


@pytest.mark.parametrize("objective", ["reg:squarederror", "binary:logistic"])
def test_base_score_estimated_when_not_given(eng, oracle, objective, tmp_path):
    """A.3: without base_score the engine estimates it from the labels (all ranks) like xgboost >= 2.0 and keeps it
    with the model."""
    X = make_data(20000, 8, 91, "uniform", nan_frac=0.02)
    rng = np.random.RandomState(92)
    y = np.nan_to_num(X[:, 0]) * 2 + rng.normal(size=len(X))
    y = (y > 14).astype(np.float32) if objective == "binary:logistic" else y.astype(np.float32)
    w = rng.uniform(0.5, 2.0, size=len(X)).astype(np.float32)
    params = {"objective": objective, "max_depth": 4, "eta": 0.3}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 3, weight=w)
    assert np.float32(ebst.params["base_score"]) == np.float32(obst.params["base_score"]) != np.float32(0.5)
    assert_same_model(ebst, obst)
    assert np.max(np.abs(ebst.predict(dm) - obst.predict(X))) <= LEAF_TOL
    f = str(tmp_path / "m.json")
    ebst.save_model(f)
    assert np.array_equal(eng.Booster(model_file=f).predict(eng.DMatrix(X)), ebst.predict(dm))


def test_custom_objective_known_answer_single_process(eng):
    """test_xgboost_api.py:77-102, single process: squared-log-error objective, rounded predictions == labels."""
    from tests.fault_injection import rmsle, squared_log
    x = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 1], [0, 0, 1, 0]] * 8, np.float32)
    y = np.array([0, 1, 0, 1] * 8, np.float32)
    dm = eng.DMatrix(x, label=y)
    res = {}
    bst = eng.train({"tree_method": "hist", "max_depth": 2, "seed": 1000}, dm, num_boost_round=10, obj=squared_log, feval=rmsle,
                    evals=[(dm, "dtrain")], evals_result=res, verbose_eval=False)
    assert list(np.round(bst.predict(eng.DMatrix(x)))) == list(y)
    assert len(res["dtrain"]["PyRMSLE"]) == 10 and res["dtrain"]["PyRMSLE"][-1] < res["dtrain"]["PyRMSLE"][0]
    assert eng.collective.allreduce([1.0, 2.0]).tolist() == [1.0, 2.0]      # no communicator: identity


def _auc_ref(p, y, w=None):
    """xgboost BinaryROCAUC: descending predictions, ties form one step, trapezoids."""
    p = np.asarray(p, np.float64); y = np.asarray(y, np.float64)
    w = np.ones_like(y) if w is None else np.asarray(w, np.float64)
    order = np.argsort(-p, kind="stable")
    p, y, w = p[order], y[order], w[order]
    tp = np.cumsum(y * w); fp = np.cumsum((1 - y) * w)
    ends = np.nonzero(np.append(p[1:] != p[:-1], True))[0]
    tp_e, fp_e = np.concatenate([[0.0], tp[ends]]), np.concatenate([[0.0], fp[ends]])
    area = np.sum((fp_e[1:] - fp_e[:-1]) * (tp_e[1:] + tp_e[:-1]) * 0.5)
    return area / (fp[-1] * tp[-1])


@pytest.mark.parametrize("weighted", [False, True])
def test_auc_metric(eng, weighted):
    """`auc` (SURVEY.md A.10; the metric of the reference's ranking / sklearn tests): equals the trapezoid AUC of the
    transformed predictions, with ties and sample weights; early stopping maximises it."""
    rng = np.random.RandomState(4)
    n, f = 30000, 8
    X = np.round(rng.uniform(0, 10, size=(n, f)), 1).astype(np.float32)        # coarse values: many tied predictions
    y = (X[:, 0] + X[:, 1] + rng.normal(scale=3.0, size=n) > 10).astype(np.float32)
    w = rng.gamma(2.0, 1.0, size=n).astype(np.float32) if weighted else None
    params = {"objective": "binary:logistic", "max_depth": 3, "eta": 0.3, "base_score": 0.5, "eval_metric": ["logloss", "auc"]}
    dm = eng.DMatrix(X, label=y, weight=w)
    Xv, yv = X[: n // 3] + np.float32(0.05), y[: n // 3]
    dv = eng.DMatrix(Xv, label=yv, weight=None if w is None else w[: n // 3])
    res = {}
    bst = eng.train(params, dm, num_boost_round=5, evals=[(dm, "train"), (dv, "valid")], evals_result=res, verbose_eval=False)
    assert abs(res["train"]["auc"][-1] - _auc_ref(bst.predict(eng.DMatrix(X)), y, w)) < 2e-6
    assert abs(res["valid"]["auc"][-1] - _auc_ref(bst.predict(eng.DMatrix(Xv)), yv, None if w is None else w[: n // 3])) < 2e-6
    assert res["train"]["auc"][-1] > res["train"]["auc"][0] > 0.5
    one = eng.DMatrix(X[:100], label=np.ones(100, np.float32))
    assert abs(float(bst.eval(one).split("auc:")[-1]) - 0.5) < 1e-9            # a single class: 0.5
    bst2 = eng.train(dict(params, eval_metric="auc"), dm, num_boost_round=50, evals=[(dv, "valid")], early_stopping_rounds=3,
                     verbose_eval=False)
    assert bst2.best_iteration is not None and bst2.best_score >= 0.5


def test_num_parallel_tree_known_answers(eng, tmp_path):
    """num_parallel_tree (random forests; xgboost_ray/tests/test_sklearn.py:277-286 `num_parallel_tree` dump length):
    n trees per class and round from the SAME gradients, leaf values scaled by eta / n.  Without sampling the n trees of a
    round are identical and their sum is the single tree of an ordinary round -- bit for bit (n is a power of two)."""
    rng = np.random.RandomState(8)
    n, f = 20000, 10
    X = rng.uniform(0, 10, size=(n, f)).astype(np.float32)
    y = (X[:, 0] * 2 + np.sin(X[:, 1]) * 3 + rng.normal(scale=0.3, size=n)).astype(np.float32)
    base = {"objective": "reg:squarederror", "max_depth": 4, "eta": 0.5, "base_score": 0.5}
    b1 = eng.train(base, eng.DMatrix(X, label=y), num_boost_round=3, verbose_eval=False)
    b4 = eng.train(dict(base, num_parallel_tree=4), eng.DMatrix(X, label=y), num_boost_round=3, verbose_eval=False)
    assert b4.num_trees() == 12 and b4.num_boosted_rounds() == 3 and len(b4.get_dump()) == 12
    t1, t4 = b1.get_trees(), b4.get_trees()
    for r in range(3):
        for j in range(4):
            assert np.array_equal(t4[4 * r + j]["split_feature"], t1[r]["split_feature"])
            assert np.array_equal(t4[4 * r + j]["split_bin"], t1[r]["split_bin"])
            leaf = t1[r]["split_feature"] < 0
            if r == 0:   # same gradients: exactly a quarter of the single tree's leaves (after round 0 the margins are
                #          sums of four quarters, which differ from one whole in the last bit)
                assert np.array_equal(t4[j]["value"][leaf] * np.float32(4.0), t1[0]["value"][leaf])
            assert np.allclose(t4[4 * r + j]["value"][leaf] * np.float32(4.0), t1[r]["value"][leaf], rtol=1e-5, atol=1e-6)
    assert np.allclose(b4.predict(eng.DMatrix(X)), b1.predict(eng.DMatrix(X)), rtol=1e-5, atol=1e-5)
    assert np.allclose(b4.predict(eng.DMatrix(X), iteration_range=(0, 2)), b1.predict(eng.DMatrix(X), iteration_range=(0, 2)),
                       rtol=1e-5, atol=1e-5)
    assert np.allclose(b4.predict(eng.DMatrix(X), iteration_range=(0, 1)), b1.predict(eng.DMatrix(X), iteration_range=(0, 1)),
                       rtol=1e-6, atol=1e-6)
    f_ = str(tmp_path / "rf.json")
    b4.save_model(f_)
    b4l = eng.Booster(model_file=f_)
    assert b4l.num_parallel_tree == 4 and b4l.num_boosted_rounds() == 3
    assert np.array_equal(b4l.predict(eng.DMatrix(X)), b4.predict(eng.DMatrix(X)))
    # 3 classes x 2 parallel trees: trees of a class sit next to each other (tree_info 0 0 1 1 2 2)
    yc = (X[:, 0] // 3.4).astype(np.float32)
    m1 = eng.train({"objective": "multi:softprob", "num_class": 3, "max_depth": 3, "eta": 0.5}, eng.DMatrix(X, label=yc), 2, verbose_eval=False)
    m2 = eng.train({"objective": "multi:softprob", "num_class": 3, "max_depth": 3, "eta": 0.5, "num_parallel_tree": 2},
                   eng.DMatrix(X, label=yc), 2, verbose_eval=False)
    assert m2.num_trees() == 12 and np.allclose(m2.predict(eng.DMatrix(X)), m1.predict(eng.DMatrix(X)), atol=1e-6)
    # a forest proper: one round, row and column sampling -> different trees, averaged leaves, sane fit
    rf = eng.train(dict(base, eta=1.0, num_parallel_tree=16, subsample=0.8, colsample_bynode=0.8, seed=3, max_depth=6),
                   eng.DMatrix(X, label=y), num_boost_round=1, verbose_eval=False)
    ts = rf.get_trees()
    assert len(ts) == 16 and any(not np.array_equal(ts[0]["split_feature"], t["split_feature"]) or
                                 not np.array_equal(ts[0]["split_bin"], t["split_bin"]) for t in ts[1:])
    assert np.mean((rf.predict(eng.DMatrix(X)) - y) ** 2) < 0.25 * np.var(y)
