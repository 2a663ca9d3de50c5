"""The CSR bin layout on the GPU: one bin per stored entry instead of the two dense n x F copies.

Histograms are exact integer sums, so the layout must not change a bit of anything: the histogram kernel's int64 cells
against the dense kernel's, and every model, evaluation log, train margin and prediction of a CSR matrix trained under
bin_layout="csr" against the same matrix under "dense" (which tests/test_gpu_sparse.py pins to the dense twin)."""
import json

import numpy as np
import pytest
import scipy.sparse as sp

from tests.test_gpu_qbits_depth import window_edge_cases
from tests.test_gpu_sparse import rand_csr, target, twin, u32

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


# ---------------------------------------------------------------------------------------------- histogram kernel
def csr_of_bins(B, rng, keep_missing=0.5):
    """A CSR whose absent cells are the 255s of B: every other cell is stored, and a share keep_missing of the 255s too
    (a stored NaN / `missing`, or a real bin 255)."""
    stored = (B != 255) | (rng.uniform(size=B.shape) < keep_missing)
    rows, cols = np.nonzero(stored)
    indptr = np.zeros(B.shape[0] + 1, np.int64)
    np.cumsum(np.bincount(rows, minlength=B.shape[0]), out=indptr[1:])
    return indptr, cols.astype(np.int32), B[rows, cols]


def check_hist(eng, B, qg, qh, ridx=None, chunk_rows=2048, window_rows=8192, seed=0):
    ref, _ = eng.hist_build_raw(B, qg, qh, ridx=ridx, window_rows=window_rows, chunk_rows=min(chunk_rows, window_rows))
    indptr, indices, bins = csr_of_bins(B, np.random.RandomState(seed))
    got, _ = eng.hist_build_raw_csr(indptr, indices, bins, B.shape[1], qg, qh, ridx=ridx, chunk_rows=chunk_rows)
    assert np.array_equal(ref, got)


def structured_bins(n, f, seed):
    """Random bins with the row and column edges: empty rows, a row storing every column, all-absent columns, a column
    stored in every row whose bin 255 is real, and sparse columns."""
    rng = np.random.RandomState(seed)
    B = rng.randint(0, 256, size=(n, f)).astype(np.uint8)
    B[rng.uniform(size=(n, f)) < 0.9] = 255            # mostly absent
    B[:, f // 2] = rng.choice([0, 9, 254, 255], size=n)  # stored in every row (csr_of_bins keeps some 255s)
    B[:, f - 1] = 255                                     # never stored
    B[5:40] = 255                                         # empty rows
    B[50] = rng.randint(0, 255, size=f)                   # every column stored
    return B


@pytest.mark.parametrize("f", [31, 32, 33, 512, 513, 4300])
def test_hist_root_and_gathered(eng, f):
    n = 6000 if f < 4300 else 1500
    B = structured_bins(n, f, f)
    rng = np.random.RandomState(f + 1)
    qg = rng.randint(-(1 << 18), 1 << 18, size=n).astype(np.int32)
    qh = rng.randint(0, 1 << 18, size=n).astype(np.int32)
    check_hist(eng, B, qg, qh, seed=1)
    check_hist(eng, B, qg, qh, ridx=np.sort(rng.choice(n, n // 3, replace=False)).astype(np.int32), seed=2)
    check_hist(eng, B, qg, qh, ridx=rng.permutation(n).astype(np.int32), chunk_rows=512, seed=3)


@pytest.mark.parametrize("f", [37, 530])
def test_hist_qbits_window_edges(eng, f):
    """The cells of tests/test_gpu_qbits_depth.py, pushed to 2^30 at the int32 window of the dense kernel."""
    for label, B, qg, qh, ridx, window, chunk in window_edge_cases(f):
        check_hist(eng, B, qg, qh, ridx=ridx, chunk_rows=chunk, window_rows=window, seed=label[0])


def test_hist_qbits8_four_million_rows(eng):
    window = 1 << 22
    n, f = window + (1 << 18), 4
    rng = np.random.RandomState(8)
    B = rng.randint(0, 256, size=(n, f)).astype(np.uint8)
    B[:, 0] = 3
    qg = np.full(n, 256, np.int32)
    qg[window:] = np.where(rng.uniform(size=n - window) < 0.8, 256, -256)
    qh = np.full(n, 256, np.int32)
    check_hist(eng, B, qg, qh, chunk_rows=8192, window_rows=window)


# ---------------------------------------------------------------------------------------------- models
def check_layouts(eng, params, X, rounds=4, info=None, eval_info=None, eval_X=None, **dm_kw):
    """Train on X under both layouts; model bytes, evaluation logs, train margins and predictions must be identical."""
    info, eval_info = info or {}, eval_info or {}
    eval_X = X[: min(X.shape[0], 1500)] if eval_X is None else eval_X
    runs = []
    for layout in ("csr", "dense"):
        dtrain = eng.DMatrix(X, bin_layout=layout, **dm_kw)
        dtrain.set_info(**info)
        deval = eng.DMatrix(eval_X, bin_layout=layout, **dm_kw)
        deval.set_info(**eval_info)
        res = {}
        bst = eng.train(params, dtrain, rounds, evals=[(dtrain, "train"), (deval, "eval")], evals_result=res,
                        verbose_eval=False)
        margin = bst.predict(dtrain, output_margin=True, training=True)
        runs.append((dtrain, deval, bst, res, margin))
    (ds, es, bs, rs, ms), (dd, ed, bd, rd, md) = runs
    assert ds.device_bytes() != dd.device_bytes() or ds.num_row() * ds.num_col() == 0
    assert json.dumps(rs) == json.dumps(rd), "evals_result"
    assert bs.save_raw() == bd.save_raw(), "model"
    assert np.array_equal(u32(ms), u32(md)), "train margin"
    assert np.array_equal(ds.get_bins(), dd.get_bins())
    for a, b in ((es, ed), (ds, dd)):
        assert np.array_equal(u32(bs.predict(a, output_margin=True)), u32(bd.predict(b, output_margin=True)))
        assert np.array_equal(u32(bs.predict(a, pred_leaf=True)), u32(bd.predict(b, pred_leaf=True)))
    return bs, bd


REG = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5, "eval_metric": ["rmse"]}
BIN = {"objective": "binary:logistic", "max_depth": 6, "eta": 0.3, "eval_metric": ["logloss", "auc"]}


def test_binary_logistic(eng):
    X = rand_csr(5000, 40, 0.1, 1)
    y = target(X, 2, "bin")
    check_layouts(eng, BIN, X, info={"label": y}, eval_info={"label": y[:1500]})


def test_weights_and_base_margin(eng):
    X = rand_csr(5000, 20, 0.1, 3)
    rng = np.random.RandomState(4)
    y = target(X, 5)
    w = rng.uniform(0.2, 3.0, size=5000).astype(np.float32)
    bm = rng.normal(size=5000).astype(np.float32)
    check_layouts(eng, REG, X, info={"label": y, "weight": w, "base_margin": bm},
                  eval_info={"label": y[:1500], "weight": w[:1500], "base_margin": bm[:1500]})


def test_softprob(eng):
    X = rand_csr(5000, 30, 0.1, 6)
    y = np.random.RandomState(7).randint(0, 5, size=5000).astype(np.float32)
    check_layouts(eng, {"objective": "multi:softprob", "num_class": 5, "max_depth": 5, "eval_metric": ["mlogloss"]}, X,
                  info={"label": y}, eval_info={"label": y[:1500]})


def test_rank_ndcg(eng):
    X = rand_csr(4000, 25, 0.1, 8)
    rng = np.random.RandomState(9)
    qid = np.sort(rng.randint(0, 200, size=4000))
    y = rng.randint(0, 4, size=4000).astype(np.float32)
    check_layouts(eng, {"objective": "rank:ndcg", "max_depth": 5, "eval_metric": ["ndcg@5"]}, X,
                  info={"label": y, "qid": qid}, eval_info={"label": y[:1500], "qid": qid[:1500]})


def test_survival_aft(eng):
    X = rand_csr(4000, 15, 0.2, 10)
    rng = np.random.RandomState(11)
    lo = rng.uniform(1, 10, size=4000).astype(np.float32)
    hi = np.where(rng.uniform(size=4000) < 0.3, np.inf, lo * 1.5).astype(np.float32)
    check_layouts(eng, {"objective": "survival:aft", "max_depth": 4, "eval_metric": ["aft-nloglik"]}, X,
                  info={"label_lower_bound": lo, "label_upper_bound": hi},
                  eval_info={"label_lower_bound": lo[:1500], "label_upper_bound": hi[:1500]})


def test_quantile_two_alphas(eng):
    X = rand_csr(4000, 20, 0.15, 12)
    y = target(X, 13)
    check_layouts(eng, {"objective": "reg:quantileerror", "quantile_alpha": [0.2, 0.8], "max_depth": 5,
                        "eval_metric": ["quantile"]}, X, info={"label": y}, eval_info={"label": y[:1500]})


@pytest.mark.parametrize("depth", [3, 8, 14])
def test_depths(eng, depth):
    X = rand_csr(30000 if depth == 14 else 8000, 50, 0.08, 14 + depth)
    y = target(X, 15)
    check_layouts(eng, dict(REG, max_depth=depth), X, rounds=3, info={"label": y}, eval_info={"label": y[:1500]})


def test_colsample_bynode_feature_weights(eng):
    X = rand_csr(6000, 60, 0.1, 20)
    y = target(X, 21)
    fw = np.random.RandomState(22).uniform(0.1, 2.0, size=60).astype(np.float32)
    check_layouts(eng, dict(REG, max_depth=7, colsample_bynode=0.5, seed=4), X,
                  info={"label": y, "feature_weights": fw}, eval_info={"label": y[:1500]})


def test_interaction_constraints(eng):
    X = rand_csr(6000, 20, 0.2, 23)
    y = target(X, 24)
    check_layouts(eng, dict(REG, interaction_constraints="[[0, 1, 2, 3], [4, 5, 6, 7, 8], [9, 10, 11]]"), X,
                  info={"label": y}, eval_info={"label": y[:1500]})


def test_dart(eng):
    X = rand_csr(4000, 20, 0.15, 25)
    y = target(X, 26)
    check_layouts(eng, {"booster": "dart", "rate_drop": 0.3, "objective": "reg:squarederror", "max_depth": 5, "seed": 3}, X,
                  rounds=6, info={"label": y}, eval_info={"label": y[:1500]})


@pytest.mark.parametrize("strategy", ["one_output_per_tree", "multi_output_tree"])
def test_three_targets(eng, strategy):
    X = rand_csr(4000, 20, 0.15, 27)
    Y = np.stack([target(X, 28 + t) for t in range(3)], axis=1)
    check_layouts(eng, {"objective": "reg:squarederror", "multi_strategy": strategy, "max_depth": 5, "eval_metric": ["rmse"]},
                  X, info={"label": Y}, eval_info={"label": Y[:1500]}, multi_target=True)


def test_num_parallel_tree(eng):
    X = rand_csr(5000, 30, 0.1, 31)
    y = target(X, 32, "bin")
    check_layouts(eng, dict(BIN, num_parallel_tree=2, subsample=0.8, colsample_bytree=0.7, seed=5), X,
                  info={"label": y}, eval_info={"label": y[:1500]})


def test_categorical_and_value_edges(eng):
    """Categorical columns with absent codes, stored NaN and stored values equal to a non-NaN missing."""
    n, f = 5000, 10
    rng = np.random.RandomState(33)
    X = rand_csr(n, f, 0.4, 34).tolil()
    for j in (1, 4):
        col = rng.randint(0, 12, size=n).astype(np.float32)
        col[rng.uniform(size=n) < 0.4] = 0
        X[:, j] = col[:, None]
    X = X.tocsr()
    X.eliminate_zeros()
    pick = rng.uniform(size=X.nnz) < 0.1
    X.data[pick] = np.where(rng.uniform(size=int(pick.sum())) < 0.5, np.nan, -999.0).astype(np.float32)
    X.data[np.isin(X.indices, (1, 4)) & ~np.isfinite(X.data)] = 3.0   # codes stay valid
    X.data[np.isin(X.indices, (1, 4)) & (X.data == -999.0)] = 3.0
    y = target(X, 35, "bin")
    types = ["c" if j in (1, 4) else "q" for j in range(f)]
    check_layouts(eng, dict(BIN, max_cat_to_onehot=4), X, info={"label": y}, eval_info={"label": y[:1500]},
                  feature_types=types, enable_categorical=True, missing=-999.0)


def test_refresh_and_continuation(eng):
    X = rand_csr(5000, 20, 0.2, 36)
    y, y2 = target(X, 37), target(X, 38)
    out = []
    for layout in ("csr", "dense"):
        base = eng.train(REG, eng.DMatrix(X, label=y, bin_layout=layout), 3, verbose_eval=False)
        cont = eng.train(REG, eng.DMatrix(X, label=y2, bin_layout=layout), 2, xgb_model=base, verbose_eval=False)
        upd = eng.train(dict(REG, process_type="update", updater="refresh"), eng.DMatrix(X, label=y2, bin_layout=layout),
                        3, xgb_model=base, verbose_eval=False)
        out.append((cont.save_raw(), upd.save_raw(), u32(upd.predict(eng.DMatrix(X)))))
    assert out[0][0] == out[1][0] and out[0][1] == out[1][1] and np.array_equal(out[0][2], out[1][2])


@pytest.mark.timeout(900)
def test_ray_one_and_two_gpus(eng):
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    X = rand_csr(20000, 40, 0.05, 39)
    y = target(X, 40, "bin")
    p = {"objective": "binary:logistic", "max_depth": 5, "eta": 0.3}
    ref = train(p, RayDMatrix(X, y, bin_layout="dense"), num_boost_round=4, ray_params=RayParams(num_actors=1)).save_raw()
    for actors in ((1, 2) if eng.device_count() >= 2 else (1,)):
        bst = train(p, RayDMatrix(X, y, bin_layout="csr"), num_boost_round=4, ray_params=RayParams(num_actors=actors))
        assert bst.save_raw() == ref, actors
    if eng.device_count() < 2:
        pytest.skip("two actors need 2 GPUs")


# ---------------------------------------------------------------------------------------------- accessors
def dense_bin_bytes(n, f):
    groups = (f + 31) // 32
    return max(n, 1) * groups * 32 + ((max(n, 1) + 127) // 128 * 128) * f


def test_device_bytes_of_the_csr_layout(eng):
    n, f = 20000, 300
    X = rand_csr(n, f, 0.01, 41)
    y = target(X, 42)
    ds, dd = eng.DMatrix(X, label=y, bin_layout="csr"), eng.DMatrix(X, label=y, bin_layout="dense")
    raw = ds.device_bytes()
    assert raw == dd.device_bytes()
    ds._ensure_quantized(256)
    dd._ensure_quantized(256)
    # both hold the same cuts and info; the CSR layout keeps indptr and indices and one bin byte per entry, the dense
    # layout its two bin copies
    assert ds.device_bytes() - dd.device_bytes() == 8 * (n + 1) + 4 * X.nnz + X.nnz - dense_bin_bytes(n, f)
    quantised = ds.device_bytes()
    ds._ensure_raw()   # the values come back, nothing else
    assert ds.device_bytes() == quantised + 4 * X.nnz
    assert np.array_equal(ds.get_bins(), dd.get_bins())


def test_slice_and_cv_keep_the_layout(eng):
    X = rand_csr(6000, 30, 0.1, 43)
    y = target(X, 44)
    rows = np.random.RandomState(45).choice(6000, 2500, replace=False)
    outs = []
    for layout in ("csr", "dense"):
        d = eng.DMatrix(X, label=y, bin_layout=layout)
        eng.train(REG, d, 1, verbose_eval=False)   # the parent is quantised: the slice re-uploads its values
        s = d.slice(rows)
        assert s.bin_layout == layout
        bst = eng.train(REG, s, 3, verbose_eval=False)
        res = eng.cv(REG, eng.DMatrix(X, label=y, bin_layout=layout), 3, nfold=3, seed=1, as_pandas=False)
        outs.append((bst.save_raw(), s.get_bins(), s.device_bytes(), json.dumps(res)))
    assert outs[0][0] == outs[1][0] and np.array_equal(outs[0][1], outs[1][1]) and outs[0][3] == outs[1][3]
    assert outs[0][2] < outs[1][2]


# ---------------------------------------------------------------------------------------------- auto
def test_auto_keeps_small_matrices_dense(eng):
    X = rand_csr(20000, 300, 0.01, 46)
    y = target(X, 47)
    da, dd = eng.DMatrix(X, label=y), eng.DMatrix(twin(X), label=y)
    da._ensure_quantized(256)
    dd._ensure_quantized(256)
    assert da.device_bytes() == dd.device_bytes()


@pytest.mark.timeout(900)
def test_auto_takes_csr_past_half_the_card(eng):
    """3M rows x 16,000 columns, 64 of them populated: the dense bins would take 96 GB.  The model must equal the one
    trained on the dense matrix of the populated columns, with feature indices mapped back: columns without a stored
    entry never split and the order of the others is kept, so the trees are the same."""
    n, f, used = 3_000_000, 16_000, 64
    rng = np.random.RandomState(48)
    cols = np.sort(rng.choice(f, used, replace=False)).astype(np.int32)
    per_row = 4   # one column out of each quarter of the populated ones: distinct and increasing within a row
    ci = (np.arange(per_row) * (used // per_row) + rng.randint(0, used // per_row, size=(n, per_row))).astype(np.int32)
    vals = np.round(rng.uniform(-5, 5, size=(n, per_row)), 2).astype(np.float32)
    indptr = np.arange(0, n * per_row + 1, per_row, dtype=np.int64)
    Xc = sp.csr_matrix((vals.reshape(-1), ci.reshape(-1).astype(np.int32), indptr), shape=(n, used))
    X = sp.csr_matrix((vals.reshape(-1), cols[ci.reshape(-1)], indptr), shape=(n, f))
    y = (vals[:, 0] * (ci[:, 0] < 8) + vals[:, 1] + rng.normal(scale=0.3, size=n)).astype(np.float32)
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5}
    d = eng.DMatrix(X, label=y)
    bst = eng.train(params, d, 3, verbose_eval=False)
    assert d.device_bytes() < 2 ** 30
    dc = eng.DMatrix(Xc, label=y, bin_layout="dense")
    ref = eng.train(params, dc, 3, verbose_eval=False)
    for a, b in zip(bst.get_trees(), ref.get_trees()):
        leaf = b["split_feature"] < 0
        assert np.array_equal(a["split_feature"][~leaf], cols[b["split_feature"][~leaf]])
        for k in ("left", "right", "split_bin", "default_left"):
            assert np.array_equal(a[k], b[k]), k
        assert np.array_equal(u32(a["value"]), u32(b["value"]))
    assert np.array_equal(u32(bst.predict(d, output_margin=True, training=True)),
                          u32(ref.predict(dc, output_margin=True, training=True)))


# ---------------------------------------------------------------------------------------------- refusals
def test_refusals(eng):
    X = np.zeros((10, 3), np.float32)
    with pytest.raises(eng.XGBoostError, match="scipy.sparse"):
        eng.DMatrix(X, bin_layout="csr")
    with pytest.raises(eng.XGBoostError, match="bin_layout"):
        eng.DMatrix(sp.csr_matrix(X), bin_layout="columnar")
