"""A CSR matrix quantised, evaluated and predicted from its stored entries only, against its dense twin (the same
matrix with NaN in every absent cell).

The sketch keys and sorts the stored entries of a batch of features (a budget of entries per batch), and the tree
walks of predict, pred_leaf, the evaluation margins and the refresh updater look a row's value up in its stored
entries.  Cuts, bins, models, evaluation logs and predictions must be bit-identical to the twin's and to the oracle's
cuts, at the column, value, weight, categorical, batch-boundary and row-count edges."""
import json

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

FLT_MAX = np.finfo(np.float32).max
FLT_TRUE_MIN = np.float32(1e-45)
BATCH_ENTRIES = 1 << 24   # kSketchBatchEntries (matrix.cu): valid entries of one sketch batch


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


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def bernoulli_csr(n, f, density, seed, values=None):
    """n x f CSR whose cells are stored independently with probability `density` (no sort, no duplicates): the gaps
    between stored cells of the flattened matrix are geometric.  values(k, rng) -> k float32 values (default U[-5, 5)
    rounded to 2 digits, so that there are ties)."""
    rng = np.random.default_rng(seed)
    cells = n * f
    pos = np.cumsum(rng.geometric(density, size=int(cells * density * 1.2) + 64)) - 1 if density > 0 else np.zeros(0, np.int64)
    pos = pos[pos < cells]
    rows, cols = pos // f, (pos % f).astype(np.int32)
    vals = (values(pos.size, rng) if values else np.round(rng.uniform(-5, 5, size=pos.size), 2)).astype(np.float32)
    indptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(rows, minlength=n), out=indptr[1:])
    return sp.csr_matrix((vals, cols, indptr), shape=(n, f))


def csr_from_columns(cols, n):
    """CSR from {column: (rows, values)} with explicitly stored entries (NaN and zeros stay stored)."""
    f = max(cols) + 1
    r = np.concatenate([np.asarray(v[0], np.int64) for v in cols.values()])
    c = np.concatenate([np.full(len(v[0]), k, np.int32) for k, v in cols.items()])
    v = np.concatenate([np.asarray(v[1], np.float32) for v in cols.values()])
    o = np.lexsort((c, r))
    indptr = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(r, minlength=n), out=indptr[1:])
    return sp.csr_matrix((v[o], c[o], indptr), shape=(n, f))


def assert_cuts_equal(a, b):
    assert np.array_equal(a[0], b[0]), "ptrs"
    assert np.array_equal(u32(a[1]), u32(b[1])), "cut values"
    assert np.array_equal(u32(a[2]), u32(b[2])), "mins"
    assert np.array_equal(a[3], b[3]), "has_missing"


def check_cuts(eng, oracle, X, max_bin=256, missing=np.nan, weight=None, is_cat=None, bins=True, **kw):
    """cuts and bins of the CSR == the twin's == oracle.Cuts.from_data(twin)"""
    T = twin(X)
    out = []
    for data in (X, T):
        dm = eng.DMatrix(data, missing=missing, weight=weight, **kw)
        dm._ensure_quantized(max_bin, keep_raw=True)
        out.append((dm.get_cuts(), dm.get_bins() if bins else None))
    (cs, bs), (cd, bd) = out
    assert_cuts_equal(cs, cd)
    oc = oracle.Cuts.from_data(T, max_bin, missing=missing, is_cat=is_cat, weight=weight)
    assert_cuts_equal(cs, (oc.ptrs, oc.vals, oc.mins, oc.has_missing))
    if bins:
        assert np.array_equal(bs, bd)
        if is_cat is None:
            assert np.array_equal(bs, oc.bin(T, missing=missing))
    return cs


def edge_matrix(n, missing=np.nan):
    """columns: 0 no stored entry, 1 stored in every row, 2 all stored NaN, 3 all stored `missing` (when not NaN),
    4 float edges (+-0, +-inf, +-FLT_MAX, subnormals), 5 heavy ties, 6 random, 7 a single entry"""
    rng = np.random.default_rng(0)
    rows = np.arange(n)
    edges = np.array([0.0, -0.0, np.inf, -np.inf, FLT_MAX, -FLT_MAX, FLT_TRUE_MIN, -FLT_TRUE_MIN, 1e-40, -1e-40, 1.0, -1.0],
                     np.float32)
    half = rows[rng.random(n) < 0.5]
    cols = {
        1: (rows, np.round(rng.uniform(0, 3, n), 1)),
        2: (rows[::3], np.full(len(rows[::3]), np.nan)),
        3: (rows[1::4], np.full(len(rows[1::4]), np.float32(missing) if not np.isnan(missing) else 7.0)),
        4: (half, edges[rng.integers(0, edges.size, half.size)]),
        5: (rows[::2], np.where(rng.random(len(rows[::2])) < 0.9, 2.5, rng.integers(0, 4, len(rows[::2]))).astype(np.float32)),
        6: (rows[rng.random(n) < 0.3], None),
        7: (rows[n // 2:n // 2 + 1], np.array([3.0], np.float32)),
    }
    cols[6] = (cols[6][0], rng.normal(size=cols[6][0].size).astype(np.float32))
    return csr_from_columns(cols, n)


@pytest.mark.parametrize("max_bin", [2, 16, 256])
@pytest.mark.parametrize("missing", [np.nan, 7.0])
def test_cuts_at_column_and_value_edges(eng, oracle, max_bin, missing):
    X = edge_matrix(3000, missing)
    assert X[:, 0].nnz == 0 and X[:, 1].nnz == X.shape[0]
    cs = check_cuts(eng, oracle, X, max_bin=max_bin, missing=missing)
    assert cs[3][0] == 1 and cs[3][1] == 0 and cs[3][2] == 1   # absent / stored-missing columns have missing values
    if not np.isnan(missing):
        assert cs[3][3] == 1


@pytest.mark.parametrize("scale_exp", [0, 7, -20])
def test_weighted_cuts(eng, oracle, scale_exp):
    X = bernoulli_csr(5000, 12, 0.3, 1)
    w = np.random.default_rng(2).uniform(0, 3, 5000).astype(np.float32)
    w[::7] = 0.0
    w = (w * np.float32(2.0 ** scale_exp)).astype(np.float32)
    cs = check_cuts(eng, oracle, X, weight=w)
    ref = check_cuts(eng, oracle, X, weight=(w / np.float32(2.0 ** scale_exp)).astype(np.float32), bins=False)
    assert_cuts_equal(cs, ref)   # integer weights are scale-free


def test_categorical_columns_mixed_in(eng, oracle):
    n, f = 4000, 8
    rng = np.random.default_rng(3)
    X = bernoulli_csr(n, f, 0.4, 4).tolil()
    for j in (2, 5):   # stored codes, some rows absent (missing category)
        col = rng.integers(1, 9, n).astype(np.float32)
        col[rng.random(n) < 0.3] = 0
        X[:, j] = col[:, None]
    X = X.tocsr()
    X.eliminate_zeros()
    types = ["c" if j in (2, 5) else "q" for j in range(f)]
    is_cat = np.array([t == "c" for t in types], np.uint8)
    cs = check_cuts(eng, oracle, X, is_cat=is_cat, feature_types=types, enable_categorical=True)
    assert cs[3][2] == 1 and cs[3][5] == 1


@pytest.mark.parametrize("n", [1, 2, 50])
def test_tiny_and_empty_rows(eng, oracle, n):
    X = bernoulli_csr(n, 6, 0.5, 5 + n).tolil()
    X[n // 2, :] = 0
    X = X.tocsr()
    X.eliminate_zeros()
    check_cuts(eng, oracle, X)
    check_cuts(eng, oracle, sp.csr_matrix((n, 6), dtype=np.float32))   # no entry at all


@pytest.mark.timeout(900)
@pytest.mark.parametrize("f", [3, 4, 5])
def test_batch_boundary(eng, oracle, f):
    """Columns 0-3 store every one of 2^22 rows, so the first batch is full exactly at F = 4; column 4 has a few entries
    and starts a second batch."""
    n = BATCH_ENTRIES // 4
    rng = np.random.default_rng(6)
    cols = {j: (np.arange(n), np.round(rng.uniform(0, 100, n), 1)) for j in range(min(f, 4))}
    if f == 5:
        cols[4] = (np.arange(0, n, 4096), rng.normal(size=n // 4096))
    X = csr_from_columns(cols, n)
    check_cuts(eng, oracle, X, max_bin=64)


@pytest.mark.timeout(1200)
def test_wide_matrix_spans_batches(eng, oracle):
    """2M x 20,000 at 0.05 % (20M entries, two batches): every feature's cuts are those of the same columns sketched
    alone.  The twin (160 GB) cannot be built: each narrow block is checked against its own twin and the oracle."""
    n, f = 2_000_000, 20_000
    X = bernoulli_csr(n, f, 0.0005, 7)
    counts = np.bincount(X.indices, minlength=f)
    assert X.nnz > BATCH_ENTRIES
    edge = int(np.searchsorted(np.cumsum(counts), BATCH_ENTRIES, side="right"))   # first feature of the second batch
    dm = eng.DMatrix(X)
    dm._ensure_quantized(256)
    ptrs, vals, mins, hm = dm.get_cuts()
    for a in (0, edge - 12, f - 24):
        b = a + 24
        Xb = X[:, a:b]
        T = twin(Xb)
        oc = oracle.Cuts.from_data(T, 256)
        for data in (Xb, T):
            d = eng.DMatrix(data)
            d._ensure_quantized(256)
            p2, v2, m2, h2 = d.get_cuts()
            sub = (ptrs[a:b + 1] - ptrs[a], vals[ptrs[a]:ptrs[b]], mins[a:b], hm[a:b])
            assert_cuts_equal(sub, (p2, v2, m2, h2))
        assert_cuts_equal(sub, (oc.ptrs, oc.vals, oc.mins, oc.has_missing))


# ---------------------------------------------------------------------------------------------- tree walks
def train_both(eng, params, X, y, Xe, ye, rounds, info=None, eval_info=None, **kw):
    info, eval_info = info or {}, eval_info or {}
    runs = []
    for conv in (lambda A: A, twin):
        dt = eng.DMatrix(conv(X), label=y, **kw)
        dt.set_info(**info)
        de = eng.DMatrix(conv(Xe), label=ye, **kw)
        de.set_info(**eval_info)
        res = {}
        bst = eng.train(params, dt, rounds, evals=[(dt, "train"), (de, "eval")], evals_result=res, verbose_eval=False)
        runs.append((bst, dt, de, res))
    (bs, ds, es, rs), (bd, dd, ed, rd) = runs
    assert json.dumps(rs) == json.dumps(rd), "evaluation log"
    assert bs.save_raw() == bd.save_raw(), "model"
    for ir in ((0, 0), (1, rounds)):
        for a, b in ((es, ed), (ds, dd)):
            assert np.array_equal(u32(bs.predict(a, output_margin=True, iteration_range=ir)),
                                  u32(bd.predict(b, output_margin=True, iteration_range=ir)))
            assert np.array_equal(u32(bs.predict(a, iteration_range=ir)), u32(bd.predict(b, iteration_range=ir)))
            assert np.array_equal(u32(bs.predict(a, pred_leaf=True, iteration_range=ir)),
                                  u32(bd.predict(b, pred_leaf=True, iteration_range=ir)))
    return bs


def data(seed, n=6000, f=40, density=0.1):
    X = bernoulli_csr(n, f, density, seed)
    T = np.nan_to_num(twin(X), nan=0.0)
    y = (T[:, :8].sum(axis=1) + np.random.default_rng(seed).normal(scale=0.3, size=n)).astype(np.float32)
    return X, y


MODES = {
    "scalar": ({"objective": "reg:squarederror", "max_depth": 6, "eval_metric": ["rmse", "mae"]}, {}),
    "softprob5": ({"objective": "multi:softprob", "num_class": 5, "max_depth": 5, "eval_metric": ["mlogloss", "merror"]}, {}),
    "vector_leaf3": ({"objective": "reg:squarederror", "multi_strategy": "multi_output_tree", "max_depth": 5,
                      "eval_metric": ["rmse"]}, {}),
    "dart": ({"booster": "dart", "rate_drop": 0.3, "objective": "reg:squarederror", "max_depth": 5, "seed": 3}, {}),
    "categorical": ({"objective": "binary:logistic", "max_depth": 5, "max_cat_to_onehot": 4,
                     "eval_metric": ["logloss", "auc"]}, {}),
    "base_margin": ({"objective": "reg:squarederror", "max_depth": 6}, {}),
    "quantile2": ({"objective": "reg:quantileerror", "quantile_alpha": [0.2, 0.8], "max_depth": 5,
                   "eval_metric": ["quantile"]}, {}),
}


@pytest.mark.parametrize("mode", sorted(MODES))
def test_eval_log_and_predictions(eng, mode):
    params, kw = MODES[mode]
    X, y = data(10)
    Xe, ye = data(11, n=3000)
    info, eval_info = {}, {}
    if mode == "softprob5":
        y, ye = (np.abs(y) * 3).astype(np.int64) % 5, (np.abs(ye) * 3).astype(np.int64) % 5
        y, ye = y.astype(np.float32), ye.astype(np.float32)
    elif mode == "vector_leaf3":
        y = np.stack([y, -y, y * 0.5], axis=1)
        ye = np.stack([ye, -ye, ye * 0.5], axis=1)
        kw = {"multi_target": True}
    elif mode == "categorical":
        rng = np.random.default_rng(12)
        X, Xe = X.tolil(), Xe.tolil()
        for A in (X, Xe):
            for j in (3, 7):
                col = rng.integers(0, 12, A.shape[0]).astype(np.float32)
                col[rng.random(A.shape[0]) < 0.3] = 0
                A[:, j] = col[:, None]
        X, Xe = X.tocsr(), Xe.tocsr()
        X.eliminate_zeros()
        Xe.eliminate_zeros()
        y, ye = (y > np.median(y)).astype(np.float32), (ye > np.median(ye)).astype(np.float32)
        kw = {"feature_types": ["c" if j in (3, 7) else "q" for j in range(X.shape[1])], "enable_categorical": True}
    elif mode == "base_margin":
        info = {"base_margin": np.linspace(-1, 1, X.shape[0]).astype(np.float32)}
        eval_info = {"base_margin": np.linspace(1, -1, Xe.shape[0]).astype(np.float32)}
    train_both(eng, params, X, y, Xe, ye, 5, info=info, eval_info=eval_info, **kw)


def test_large_model_walks(eng):
    """200 trees of depth 8 on rows of 10 % density: many lookups per row."""
    X, y = data(13, n=20000, f=100)
    Xe, ye = data(14, n=5000, f=100)
    train_both(eng, {"objective": "reg:squarederror", "max_depth": 8, "eta": 0.1}, X, y, Xe, ye, 200)


def test_refresh_model_file(eng):
    X, y = data(15)
    y2 = (y * 0.5 + 1).astype(np.float32)
    out = []
    for conv in (lambda A: A, twin):
        base = eng.train({"objective": "reg:squarederror", "max_depth": 6}, eng.DMatrix(conv(X), label=y), 4,
                         verbose_eval=False)
        upd = eng.train({"objective": "reg:squarederror", "max_depth": 6, "process_type": "update", "updater": "refresh"},
                        eng.DMatrix(conv(X), label=y2), 4, xgb_model=base, verbose_eval=False)
        out.append(upd.save_raw())
    assert out[0] == out[1]


# ---------------------------------------------------------------------------------------------- two ranks
@pytest.mark.timeout(900)
@pytest.mark.parametrize("weighted", [False, True])
def test_two_ranks_equal_one_and_oracle(eng, oracle, weighted):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from tests.test_gpu_parity import assert_same_model
    from xgboost_ray_b200 import RayDMatrix, RayParams, RayShardingMode, train
    X, y = data(16, n=20000, f=60, density=0.08)
    yb = (y > np.median(y)).astype(np.float32)
    w = np.random.default_rng(17).uniform(0, 2, X.shape[0]).astype(np.float32) if weighted else None
    params = {"objective": "binary:logistic", "max_depth": 5, "eta": 0.3, "base_score": 0.5}
    one = train(params, RayDMatrix(X, yb, weight=w), num_boost_round=4, ray_params=RayParams(num_actors=1))
    for mode in (RayShardingMode.INTERLEAVED, RayShardingMode.BATCH):
        two = train(params, RayDMatrix(X, yb, weight=w, sharding=mode), num_boost_round=4,
                    ray_params=RayParams(num_actors=2))
        assert two.save_raw() == one.save_raw()
    obst, _ = oracle.train(params, twin(X), yb, 4, weight=w)
    assert_same_model(one, obst)
