"""scipy.sparse input on the GPU: a CSR DMatrix against its dense twin (the same matrix with NaN in every absent cell).

The device keeps the CSR and densifies tiles of it for the kernels that read raw rows, and keys the sketch straight
from it.  Cuts, bins, models, evaluation logs and every prediction output must be bit-identical to the twin's, at the
density, feature-count, tile-boundary and value edges, for every objective and training mode."""
import ctypes as C
import json

import numpy as np
import pytest
import scipy.sparse as sp

from tests.test_gpu_parity import assert_same_model

pytestmark = pytest.mark.gpu

FLT_MAX = np.finfo(np.float32).max


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def twin(X):
    c = sp.coo_matrix(X)
    out = np.full(c.shape, np.nan, np.float32)
    out[c.row, c.col] = c.data.astype(np.float32)
    return out


def rand_csr(n, f, density, seed, lo=-5.0, hi=5.0):
    rng = np.random.RandomState(seed)
    X = sp.random(n, f, density=density, random_state=rng, format="csr", dtype=np.float32,
                  data_rvs=lambda k: np.round(rng.uniform(lo, hi, size=k), 2))
    return X


def target(X, seed, kind="reg"):
    rng = np.random.RandomState(seed)
    T = np.nan_to_num(twin(X), nan=0.0)
    z = T[:, : min(T.shape[1], 6)].sum(axis=1) + rng.normal(scale=0.3, size=T.shape[0])
    if kind == "reg":
        return z.astype(np.float32)
    return (z > np.median(z)).astype(np.float32)


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def check_same(eng, params, X, rounds=4, eval_X=None, interactions=None, info=None, eval_info=None, **dm_kw):
    """Train on the CSR and on its twin; everything must be identical.  info / eval_info: set_info keyword arguments."""
    info, eval_info = info or {}, eval_info or {}
    eval_X = X[: min(X.shape[0], 1500)] if eval_X is None else eval_X
    runs = []
    for conv in (lambda A: A, twin):
        dtrain = eng.DMatrix(conv(X), **dm_kw)
        dtrain.set_info(**info)
        deval = eng.DMatrix(conv(eval_X), **dm_kw)
        deval.set_info(**eval_info)
        res = {}
        bst = eng.train(params, dtrain, rounds, evals=[(dtrain, "train"), (deval, "eval")], evals_result=res,
                        verbose_eval=False)
        runs.append((dtrain, deval, bst, res))
    (ds, es, bs, rs), (dd, ed, bd, rd) = runs
    assert json.dumps(rs) == json.dumps(rd), "evals_result"   # NaN-aware: a NaN metric must be NaN on both
    assert bs.save_raw() == bd.save_raw(), "model"
    ps, pd_ = ds.get_cuts(), dd.get_cuts()
    assert np.array_equal(ps[0], pd_[0]) and np.array_equal(u32(ps[1]), u32(pd_[1]))
    assert np.array_equal(u32(ps[2]), u32(pd_[2])) and np.array_equal(ps[3], pd_[3])
    if X.shape[0] * X.shape[1] <= 4 * 10 ** 7:
        assert np.array_equal(ds.get_bins(), dd.get_bins())
    for a, b in ((es, ed), (ds, dd)):   # the train matrices were quantised without their raw values: re-uploaded here
        assert np.array_equal(u32(bs.predict(a, output_margin=True)), u32(bd.predict(b, output_margin=True)))
        assert np.array_equal(u32(bs.predict(a)), u32(bd.predict(b)))
        assert np.array_equal(u32(bs.predict(a, pred_leaf=True)), u32(bd.predict(b, pred_leaf=True)))
    if not bs.is_vector_leaf:
        assert np.array_equal(u32(bs.predict(es, pred_contribs=True)), u32(bd.predict(ed, pred_contribs=True)))
        if interactions or (interactions is None and X.shape[1] <= 40):
            sl = eval_X[:200]
            assert np.array_equal(u32(bs.predict(eng.DMatrix(sl, **dm_kw), pred_interactions=True)),
                                  u32(bd.predict(eng.DMatrix(twin(sl), **dm_kw), pred_interactions=True)))
    return bs, bd, ds, dd


REG = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5, "eval_metric": ["rmse", "mae"]}
BIN = {"objective": "binary:logistic", "max_depth": 6, "eta": 0.3, "eval_metric": ["logloss", "auc"]}


@pytest.mark.parametrize("density", [0.0, 0.001, 0.05, 0.6, 1.0])
def test_density(eng, density):
    X = rand_csr(4000, 32, density, 1)
    check_same(eng, REG, X, info={"label": target(X, 2)}, eval_info={"label": target(X[:1500], 2)})


@pytest.mark.parametrize("f", [1, 32, 33, 100, 513, 1000])
def test_feature_counts(eng, f):
    X = rand_csr(3000, f, min(1.0, 4.0 / f + 0.02), 3)
    y = target(X, 4, "bin")
    check_same(eng, BIN, X, info={"label": y}, eval_info={"label": y[:1500]})


@pytest.mark.timeout(900)
@pytest.mark.parametrize("k,delta", [(1, -1), (1, 1), (2, 1)])
def test_tile_boundaries(eng, k, delta):
    """Row counts around whole tiles: several densified tiles per consumer, a last tile of one row."""
    f = 1000
    n = k * eng.raw_tile_rows(f) + delta
    X = rand_csr(n, f, 0.005, 5)
    y = target(X, 6)
    p = dict(REG, max_depth=5)
    check_same(eng, p, X, rounds=2, eval_X=X, interactions=False, info={"label": y}, eval_info={"label": y})


@pytest.mark.parametrize("full_row", [False, True])
def test_row_structure(eng, full_row):
    """Empty rows, all-absent trailing columns, a row with every column stored."""
    n, f = 2000, 40
    X = rand_csr(n, f - 5, 0.1, 7).tolil()
    X.resize((n, f))
    X[10:60, :] = 0          # lil: assigning 0 removes the entries -> empty rows
    X = X.tocsr()
    X.eliminate_zeros()
    assert X.shape == (n, f) and X[:, f - 5:].nnz == 0 and X[20].nnz == 0
    if full_row:
        full = np.arange(1, f + 1, dtype=np.float32)
        X = sp.vstack([X[:100], sp.csr_matrix(full[None, :]), X[100:]]).tocsr()
        assert X[100].nnz == f
    check_same(eng, REG, X, info={"label": target(X, 8)}, eval_info={"label": target(X[:1500], 8)})


@pytest.mark.parametrize("missing", [None, 0.0, -999.0])
def test_value_edges(eng, missing):
    n, f = 3000, 12
    X = rand_csr(n, f, 0.3, 9)
    rng = np.random.RandomState(10)
    special = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, FLT_MAX, -FLT_MAX, 1e-45, -1e-45, 1e-40, -999.0],
                       np.float32)
    y = target(X, 11)
    pick = rng.uniform(size=X.nnz) < 0.3
    X.data[pick] = special[rng.randint(0, special.size, size=int(pick.sum()))]
    kw = {} if missing is None else {"missing": missing}
    check_same(eng, REG, X, info={"label": y}, eval_info={"label": y[:1500]}, **kw)


@pytest.mark.parametrize("n_codes", [3, 12])   # one-hot / partition splits (max_cat_to_onehot = 4)
def test_categorical_with_absent_codes(eng, n_codes):
    n, f = 4000, 8
    rng = np.random.RandomState(12)
    X = rand_csr(n, f, 0.4, 13).tolil()
    for j in (1, 4):   # categorical columns: stored codes, absent = missing category
        col = rng.randint(0, n_codes, size=n).astype(np.float32)
        col[rng.uniform(size=n) < 0.4] = 0   # removed below: absent codes
        X[:, j] = col[:, None]
    X = X.tocsr()
    X.eliminate_zeros()
    types = ["c" if j in (1, 4) else "q" for j in range(f)]
    y = target(X, 14, "bin")
    check_same(eng, dict(BIN, max_cat_to_onehot=4), X, info={"label": y}, eval_info={"label": y[:1500]},
               feature_types=types, enable_categorical=True)


def test_weights_and_base_margin(eng):
    X = rand_csr(5000, 20, 0.1, 15)
    rng = np.random.RandomState(16)
    y = target(X, 17, "bin")
    w = rng.uniform(0.2, 3.0, size=5000).astype(np.float32)
    bm = rng.normal(size=5000).astype(np.float32)
    check_same(eng, BIN, X, info={"label": y, "weight": w, "base_margin": bm},
               eval_info={"label": y[:1500], "weight": w[:1500], "base_margin": bm[:1500]})


def test_softprob(eng):
    X = rand_csr(5000, 30, 0.1, 18)
    y = np.random.RandomState(19).randint(0, 5, size=5000).astype(np.float32)
    check_same(eng, {"objective": "multi:softprob", "num_class": 5, "max_depth": 5, "eval_metric": ["mlogloss", "merror"]},
               X, info={"label": y}, eval_info={"label": y[:1500]})


def test_rank_ndcg(eng):
    X = rand_csr(4000, 25, 0.1, 20)
    rng = np.random.RandomState(21)
    qid = np.sort(rng.randint(0, 200, size=4000))
    y = rng.randint(0, 4, size=4000).astype(np.float32)
    check_same(eng, {"objective": "rank:ndcg", "max_depth": 5, "eval_metric": ["ndcg@5", "map"]}, X,
               info={"label": y, "qid": qid}, eval_info={"label": y[:1500], "qid": qid[:1500]})


def test_survival_aft(eng):
    X = rand_csr(4000, 15, 0.2, 22)
    rng = np.random.RandomState(23)
    lo = rng.uniform(1, 10, size=4000).astype(np.float32)
    hi = np.where(rng.uniform(size=4000) < 0.3, np.inf, lo * 1.5).astype(np.float32)
    check_same(eng, {"objective": "survival:aft", "max_depth": 4, "eval_metric": ["aft-nloglik"]}, X,
               info={"label_lower_bound": lo, "label_upper_bound": hi},
               eval_info={"label_lower_bound": lo[:1500], "label_upper_bound": hi[:1500]})


def test_quantile_two_alphas(eng):
    X = rand_csr(4000, 20, 0.15, 24)
    y = target(X, 25)
    check_same(eng, {"objective": "reg:quantileerror", "quantile_alpha": [0.2, 0.8], "max_depth": 5,
                     "eval_metric": ["quantile"]}, X, info={"label": y}, eval_info={"label": y[:1500]})


@pytest.mark.parametrize("strategy", ["one_output_per_tree", "multi_output_tree"])
def test_multi_target(eng, strategy):
    X = rand_csr(4000, 20, 0.15, 26)
    Y = np.stack([target(X, 27 + t) for t in range(3)], axis=1)
    check_same(eng, {"objective": "reg:squarederror", "multi_strategy": strategy, "max_depth": 5, "eval_metric": ["rmse"]},
               X, info={"label": Y}, eval_info={"label": Y[:1500]}, multi_target=True)


def test_dart(eng):
    X = rand_csr(4000, 20, 0.15, 30)
    y = target(X, 31)
    check_same(eng, {"booster": "dart", "rate_drop": 0.3, "objective": "reg:squarederror", "max_depth": 5, "seed": 3},
               X, rounds=6, info={"label": y}, eval_info={"label": y[:1500]})


def test_colsample_bynode_depth8(eng):
    X = rand_csr(6000, 60, 0.1, 32)
    y = target(X, 33)
    check_same(eng, {"objective": "reg:squarederror", "max_depth": 8, "colsample_bynode": 0.5, "seed": 4}, X,
               info={"label": y}, eval_info={"label": y[:1500]})


def test_refresh_and_continuation(eng):
    """process_type=update and xgb_model continuation read the train matrix's raw rows (re-uploaded CSR)."""
    X = rand_csr(5000, 20, 0.2, 34)
    y, y2 = target(X, 35), target(X, 36)
    out = []
    for conv in (lambda A: A, twin):
        base = eng.train(REG, eng.DMatrix(conv(X), label=y), 3, verbose_eval=False)
        cont = eng.train(REG, eng.DMatrix(conv(X), label=y2), 2, xgb_model=base, verbose_eval=False)
        upd = eng.train(dict(REG, process_type="update", updater="refresh"), eng.DMatrix(conv(X), label=y2), 3,
                        xgb_model=base, verbose_eval=False)
        out.append((cont.save_raw(), upd.save_raw(), u32(upd.predict(eng.DMatrix(conv(X))))))
    assert out[0][0] == out[1][0] and out[0][1] == out[1][1] and np.array_equal(out[0][2], out[1][2])


@pytest.mark.timeout(1200)
def test_two_million_rows_depth14(eng):
    X = rand_csr(2_000_000, 50, 0.05, 37)
    y = target(X, 38)
    check_same(eng, {"objective": "reg:squarederror", "max_depth": 14, "eta": 0.3}, X, rounds=2, eval_X=X[:100000],
               interactions=False, info={"label": y}, eval_info={"label": y[:100000]})


@pytest.mark.parametrize("shape", [(6000, 33, 0.05), (5000, 100, 0.2)])
def test_oracle_parity(eng, oracle, shape):
    n, f, density = shape
    X = rand_csr(n, f, density, 39)
    y = target(X, 40, "bin")
    params = {"objective": "binary:logistic", "max_depth": 6, "eta": 0.3, "base_score": 0.5}
    obst, _ = oracle.train(params, twin(X), y, 4)
    ebst = eng.train(params, eng.DMatrix(X, label=y), 4, verbose_eval=False)
    assert_same_model(ebst, obst)
    Xt = rand_csr(2000, f, density, 41)
    assert np.max(np.abs(ebst.predict(eng.DMatrix(Xt)) - obst.predict(twin(Xt)))) <= 1e-5


# ---------------------------------------------------------------------------------------------- the C ABI
def _create(eng, indptr, indices, values, n, f):
    indptr = np.ascontiguousarray(indptr, np.int64)
    indices = np.ascontiguousarray(indices, np.int32)
    values = np.ascontiguousarray(values, np.float32)
    h = eng._H(0)
    rc = eng.lib().B2_MatrixCreateFromCSR(indptr.ctypes.data_as(eng._LP), eng._ip(indices), eng._fp(values), n, f,
                                           indices.size, float("nan"), 0, C.byref(h))
    if rc == 0:
        eng.lib().B2_MatrixFree(h.value)
        return None
    return eng.lib().B2_GetLastError().decode()


def test_abi_refuses_malformed_csr_naming_the_row(eng):
    ok = ([0, 2, 3, 3], [0, 2, 1], [1.0, 2.0, 3.0])
    assert _create(eng, *ok, 3, 4) is None
    assert "row 1: column 4 is outside [0, 4)" in _create(eng, [0, 2, 3, 3], [0, 2, 4], [1, 2, 3], 3, 4)
    assert "row 0: column -1" in _create(eng, [0, 2, 3, 3], [-1, 2, 1], [1, 2, 3], 3, 4)
    assert "row 1: indptr decreases" in _create(eng, [0, 2, 1, 3], [0, 2, 1], [1, 2, 3], 3, 4)
    assert "row 2: indptr[3] = 2, must equal nnz = 3" in _create(eng, [0, 1, 2, 2], [0, 2, 1], [1, 2, 3], 3, 4)
    assert "row 0: indptr[0] = 1" in _create(eng, [1, 2, 3, 3], [0, 2, 1], [1, 2, 3], 3, 4)
    assert "row 0: column 2 is stored twice" in _create(eng, [0, 2, 3, 3], [2, 2, 1], [1, 2, 3], 3, 4)
    assert "row 0: column 0 follows column 2" in _create(eng, [0, 2, 3, 3], [2, 0, 1], [1, 2, 3], 3, 4)


def test_device_bytes(eng):
    n, f = 20000, 300
    X = rand_csr(n, f, 0.01, 42)
    y = target(X, 43)
    ds, dd = eng.DMatrix(X, label=y), eng.DMatrix(twin(X), label=y)
    info = dd.device_bytes() - 4 * n * f
    assert ds.device_bytes() == 8 * (n + 1) + 8 * X.nnz + info
    ds._ensure_quantized(256)
    dd._ensure_quantized(256)
    assert ds.device_bytes() == dd.device_bytes() < 4 * n * f
    ds._ensure_raw()
    assert ds.device_bytes() == dd.device_bytes() + 8 * (n + 1) + 8 * X.nnz


# ---------------------------------------------------------------------------------------------- public API
def _rd_params():
    return {"objective": "binary:logistic", "max_depth": 5, "eta": 0.3, "eval_metric": ["logloss"]}


@pytest.mark.timeout(900)
def test_ray_one_actor_equals_engine(eng):
    from xgboost_ray_b200 import RayDMatrix, RayParams, predict, train
    X = rand_csr(20000, 40, 0.05, 44)
    y = target(X, 45, "bin")
    rb = train(_rd_params(), RayDMatrix(X, y), num_boost_round=4, ray_params=RayParams(num_actors=1))
    eb = eng.train(_rd_params(), eng.DMatrix(X, label=y), 4, verbose_eval=False)
    for a, b in zip(rb.get_trees(), eb.get_trees()):
        for k in ("left", "right", "split_feature", "split_bin", "default_left"):
            assert np.array_equal(a[k], b[k])
        assert np.array_equal(u32(a["value"]), u32(b["value"]))
    pr = predict(rb, RayDMatrix(X), ray_params=RayParams(num_actors=1))
    assert np.array_equal(u32(pr), u32(eb.predict(eng.DMatrix(X))))


@pytest.mark.timeout(900)
def test_ray_two_actors_equal_one(eng):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, RayShardingMode, predict, train
    X = rand_csr(20000, 40, 0.05, 46)
    y = target(X, 47, "bin")
    one = train(_rd_params(), RayDMatrix(X, y), num_boost_round=4, ray_params=RayParams(num_actors=1))
    for mode in (RayShardingMode.INTERLEAVED, RayShardingMode.BATCH):
        two = train(_rd_params(), RayDMatrix(X, y, sharding=mode), num_boost_round=4, ray_params=RayParams(num_actors=2))
        assert two.save_raw() == one.save_raw()
        p2 = predict(two, RayDMatrix(X, sharding=mode), ray_params=RayParams(num_actors=2))
        assert np.array_equal(u32(p2), u32(predict(one, RayDMatrix(X), ray_params=RayParams(num_actors=1))))


@pytest.mark.timeout(900)
def test_sklearn_on_csr_equals_twin(eng):
    from xgboost_ray_b200 import RayParams
    from xgboost_ray_b200.sklearn import RayXGBClassifier
    X = rand_csr(8000, 30, 0.1, 48)
    y = np.random.RandomState(49).randint(0, 3, size=8000)
    rp = RayParams(num_actors=1)
    outs = []
    for data in (X, twin(X)):
        clf = RayXGBClassifier(n_estimators=4, max_depth=4).fit(data, y, ray_params=rp)
        outs.append((u32(clf.predict_proba(data, ray_params=rp)), u32(clf.apply(data, ray_params=rp))))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
