"""DMatrix.slice and cv() on the GPU (DESIGN.md 2 item 24).

A slice is gathered on the device from its parent's device data and sketched with its own cuts, so it must equal the
matrix built from the same rows on the host, DMatrix(X[idx], label=y[idx], ...), bit for bit: cuts, bins, the model
file, predictions and eval logs.  The parent must not change.  cv() must compute exactly what a sequential loop of
train() over the same slices computes: every mean and std compared with ==."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def E():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


BASE = {"max_depth": 4, "eta": 0.3, "seed": 7, "max_bin": 64}
IDX = np.r_[np.arange(1999, 1500, -3), [5, 5, 5, 0, 1999], np.arange(10, 900, 2)]   # unsorted, duplicated rows


def data(n=2000, f=6, seed=0, nan=0.05):
    rng = np.random.RandomState(seed)
    X = rng.normal(size=(n, f)).astype(np.float32)
    y = (X[:, 0] + 0.5 * X[:, 1] * X[:, 2] + 0.1 * rng.normal(size=n)).astype(np.float32)
    X[rng.rand(n, f) < nan] = np.nan
    return X, y


def train_and_compare(E, sl, built, params, rounds=3):
    """sl and built are the same rows: equal info and device bytes before training, then equal cuts, bins, model file,
    eval log and predictions."""
    assert sl.num_row() == built.num_row() and sl.num_col() == built.num_col()
    for get in ("get_label", "get_weight", "get_base_margin"):
        assert np.array_equal(getattr(sl, get)(), getattr(built, get)()), get
    assert sl.device_bytes() == built.device_bytes()
    logs = []
    boosters = []
    for d in (sl, built):
        log = {}
        boosters.append(E.train(params, d, rounds, evals=[(d, "train")], evals_result=log, verbose_eval=False))
        logs.append(log)
    for a, b in zip(sl.get_cuts(), built.get_cuts()):
        assert np.array_equal(a, b)
    assert np.array_equal(sl.get_bins(), built.get_bins())
    assert boosters[0].save_raw() == boosters[1].save_raw()
    assert logs[0] == logs[1]
    for d in (sl, built):   # each model on both matrices: the slice's rows reach the predictor through its host rows
        p0, p1 = boosters[0].predict(d), boosters[1].predict(d)
        assert np.array_equal(p0, p1)
    assert np.array_equal(boosters[0].predict(sl, output_margin=True), boosters[1].predict(built, output_margin=True))
    return boosters[0]


@pytest.mark.parametrize("missing", [None, -999.0])
def test_dense_slice_equals_built_rows(E, missing):
    X, y = data()
    if missing is not None:
        X[np.isnan(X)] = missing
    parent = E.DMatrix(X, label=y, missing=missing)
    bins_before = parent.device_bytes()
    train_and_compare(E, parent.slice(IDX), E.DMatrix(X[IDX], label=y[IDX], missing=missing), BASE)
    assert parent.device_bytes() == bins_before


@pytest.mark.parametrize("f", [5, 6, 8])   # row widths that take the float, float2 and float4 gathers
def test_slice_widths(E, f):
    X, y = data(f=f)
    sl = E.DMatrix(X, label=y).slice(IDX)
    train_and_compare(E, sl, E.DMatrix(X[IDX], label=y[IDX]), BASE, rounds=2)


def test_csr_slice_equals_built_rows_and_its_dense_twin(E):
    sp = pytest.importorskip("scipy.sparse")
    X, y = data(nan=0.0)
    X[np.abs(X) < 0.6] = 0
    csr = sp.csr_matrix(X)
    parent = E.DMatrix(csr, label=y)
    before = parent.device_bytes()
    sl = parent.slice(IDX)
    bst = train_and_compare(E, sl, E.DMatrix(csr[IDX], label=y[IDX]), BASE)
    assert parent.device_bytes() == before
    dense = np.where(X == 0, np.nan, X).astype(np.float32)
    twin = E.DMatrix(dense, label=y).slice(IDX)
    twin_bst = E.train(BASE, twin, 3, verbose_eval=False)
    assert twin_bst.save_raw() == bst.save_raw()
    assert np.array_equal(bst.predict(sl), twin_bst.predict(twin))


def test_row_block_parent_and_parent_without_raw(E):
    X, y = data()

    class Iter:
        def __init__(self):
            self.i = 0

        def reset(self):
            self.i = 0

        def next(self, input_data):
            if self.i == 3:
                return 0
            s = slice(self.i * 700, min((self.i + 1) * 700, len(X)))
            input_data(data=X[s], label=y[s])
            self.i += 1
            return 1

    it_parent = E.DMatrix(Iter())
    sl = it_parent.slice(IDX)
    # the rows stayed on the device: neither matrix holds host rows yet
    assert isinstance(it_parent._host, E._BlockList) and isinstance(sl._host, E._SliceRows)
    train_and_compare(E, sl, E.DMatrix(X[IDX], label=y[IDX]), BASE)
    assert isinstance(it_parent._host, E._BlockList)

    parent = E.DMatrix(X, label=y)
    model = E.train(BASE, parent, 3, verbose_eval=False)   # quantised without raw values on the device
    assert not parent._has_raw
    bins, cuts = parent.get_bins(), parent.get_cuts()
    sl = parent.slice(IDX)
    train_and_compare(E, sl, E.DMatrix(X[IDX], label=y[IDX]), BASE)
    assert np.array_equal(parent.get_bins(), bins)
    assert all(np.array_equal(a, b) for a, b in zip(parent.get_cuts(), cuts))
    assert np.array_equal(model.predict(parent), model.predict(E.DMatrix(X)))
    assert E.train(BASE, parent, 3, verbose_eval=False).save_raw() == model.save_raw()


def test_quantised_parent_keeps_bins_and_device_bytes(E):
    X, y = data()
    parent = E.DMatrix(X, label=y)
    parent._ensure_quantized(64, keep_raw=True)
    model = E.train(BASE, parent, 3, verbose_eval=False)
    bins, nbytes = parent.get_bins(), parent.device_bytes()
    for _ in range(2):
        parent.slice(IDX)
    assert np.array_equal(parent.get_bins(), bins) and parent.device_bytes() == nbytes
    assert E.train(BASE, parent, 3, verbose_eval=False).save_raw() == model.save_raw()


def test_categorical_weights_and_base_margin(E):
    X, y = data()
    rng = np.random.RandomState(1)
    X[:, 1] = rng.randint(0, 7, size=len(X))
    X[rng.rand(len(X)) < 0.05, 1] = np.nan
    w = rng.uniform(0.2, 2, size=len(X)).astype(np.float32)
    m = rng.normal(size=len(X)).astype(np.float32)
    ft = ["q", "c", "q", "q", "q", "q"]
    names = ["f%d" % i for i in range(6)]
    kw = dict(feature_types=ft, enable_categorical=True, feature_names=names)
    parent = E.DMatrix(X, label=y, weight=w, base_margin=m, **kw)
    parent.set_info(feature_weights=np.arange(1, 7, dtype=np.float32))
    built = E.DMatrix(X[IDX], label=y[IDX], weight=w[IDX], base_margin=m[IDX], **kw)
    built.set_info(feature_weights=np.arange(1, 7, dtype=np.float32))
    sl = parent.slice(IDX)
    assert sl.feature_names == names and sl.feature_types == ft
    train_and_compare(E, sl, built, dict(BASE, max_cat_to_onehot=1, colsample_bynode=0.5))

    K = 3
    yc = (np.nan_to_num(X[:, 0]) > 0).astype(np.float32) + (np.nan_to_num(X[:, 2]) > 0.5)
    mk = rng.normal(size=(len(X), K)).astype(np.float32)
    parent = E.DMatrix(X, label=yc, base_margin=mk, **kw)
    built = E.DMatrix(X[IDX], label=yc[IDX], base_margin=mk[IDX], **kw)
    train_and_compare(E, parent.slice(IDX), built, dict(BASE, objective="multi:softprob", num_class=K))


def test_multi_target_label_and_aft_bounds(E):
    X, y = data()
    Y = np.stack([y, -y, 2 * y], axis=1)
    parent = E.DMatrix(X, label=Y, multi_target=True)
    train_and_compare(E, parent.slice(IDX), E.DMatrix(X[IDX], label=Y[IDX], multi_target=True), BASE)

    lo = np.exp(y / 4).astype(np.float32)
    hi = np.where(np.arange(len(y)) % 3 == 0, np.inf, lo * 1.5).astype(np.float32)
    params = dict(BASE, objective="survival:aft", eval_metric="aft-nloglik")
    parent = E.DMatrix(X, label_lower_bound=lo, label_upper_bound=hi)
    built = E.DMatrix(X[IDX], label_lower_bound=lo[IDX], label_upper_bound=hi[IDX])
    train_and_compare(E, parent.slice(IDX), built, params)


def test_query_groups(E):
    X, y = data()
    y = np.floor(np.clip(y + 2, 0, 4)).astype(np.float32)
    sizes = np.full(100, 20)
    qid = np.repeat(np.arange(100), 20)
    parent = E.DMatrix(X, label=y, qid=qid)
    with pytest.raises(E.XGBoostError, match="query groups; pass allow_groups=True"):
        parent.slice(np.arange(40))
    groups = [7, 3, 50, 3]
    rows = np.concatenate([np.arange(g * 20, g * 20 + 20) for g in groups])
    sl = parent.slice(rows, allow_groups=True)
    assert sl.get_group().size == 0
    sl.set_group(sizes[groups])
    built = E.DMatrix(X[rows], label=y[rows], group=sizes[groups])
    train_and_compare(E, sl, built, dict(BASE, objective="rank:ndcg", eval_metric="ndcg@5"))


def test_slice_refusals(E):
    X, y = data()
    dm = E.DMatrix(X, label=y)
    with pytest.raises(E.XGBoostError, match=r"rindex\[1\] = 2000 is outside \[0, 2000\)"):
        dm.slice([0, 2000])
    with pytest.raises(E.XGBoostError, match="rindex is empty"):
        dm.slice([])
    with pytest.raises(E.XGBoostError, match="QuantileDMatrix"):
        E.QuantileDMatrix(X, label=y).slice([0, 1])
    # the C ABI checks the rows itself
    import ctypes as C
    rows = np.array([0, -3], np.int64)
    h = E._H(0)
    assert E.lib().B2_MatrixSlice(dm.handle, rows.ctypes.data_as(E._LP), 2, C.byref(h)) == -1
    assert b"row index -3 (position 1) is outside [0, 2000)" in E.lib().B2_GetLastError()


# ----------------------------------------------------------------------------- cv()
def loop_cv(E, params, dtrain, rounds, nfold=3, seed=0, stratified=False, obj=None, custom_metric=None,
            callbacks=None):
    """cv() restated as a sequential loop of train() over the same slices: the mean and std of each round's values."""
    spec = E.cv_folds(dtrain.num_row(), nfold, label=dtrain.get_label(), group_sizes=dtrain._group_sizes,
                      stratified=stratified, seed=seed)
    logs = []
    for tr, te, gtr, gte in spec:
        d_in, d_out = dtrain.slice(tr, allow_groups=gtr is not None), dtrain.slice(te, allow_groups=gtr is not None)
        if gtr is not None:
            d_in.set_group(gtr)
            d_out.set_group(gte)
        log = {}
        E.train(params, d_in, rounds, evals=[(d_in, "train"), (d_out, "test")], evals_result=log, obj=obj,
                custom_metric=custom_metric, verbose_eval=False, callbacks=callbacks() if callbacks else None)
        logs.append(log)
    out = {}
    for data in ("train", "test"):
        for metric in logs[0][data]:
            vals = np.array([lg[data][metric] for lg in logs])   # [fold][round]
            out["%s-%s-mean" % (data, metric)] = [float(np.mean(vals[:, r])) for r in range(vals.shape[1])]
            out["%s-%s-std" % (data, metric)] = [float(np.std(vals[:, r])) for r in range(vals.shape[1])]
    return out


def sq_obj(pred, dtrain):
    return pred - dtrain.get_label(), np.ones_like(pred)


def mae_metric(pred, dtrain):
    return "mymae", float(np.mean(np.abs(pred - dtrain.get_label())))


def cv_cases():
    X, y = data(n=1500)
    yb = (y > 0).astype(np.float32)
    yk = np.digitize(y, [-0.5, 0.5]).astype(np.float32)
    lo = np.exp(y / 4).astype(np.float32)
    hi = np.where(np.arange(len(y)) % 3 == 0, np.inf, lo * 1.5).astype(np.float32)
    Y = np.stack([y, -y], axis=1)
    yr = np.floor(np.clip(y + 2, 0, 4)).astype(np.float32)
    return {
        "squarederror": (dict(BASE), dict(data=X, label=y), {}),
        "logistic_stratified": (dict(BASE, objective="binary:logistic", eval_metric=["logloss", "auc"]),
                                dict(data=X, label=yb), dict(stratified=True)),
        "softprob": (dict(BASE, objective="multi:softprob", num_class=3), dict(data=X, label=yk), {}),
        "ndcg_groups": (dict(BASE, objective="rank:ndcg", eval_metric="ndcg@5"),
                        dict(data=X, label=yr, qid=np.repeat(np.arange(75), 20)), {}),
        "aft": (dict(BASE, objective="survival:aft"), dict(data=X, label_lower_bound=lo, label_upper_bound=hi), {}),
        "dart": (dict(BASE, booster="dart", rate_drop=0.3), dict(data=X, label=y), {}),
        "multi_target": (dict(BASE), dict(data=X, label=Y, multi_target=True), {}),
        "custom_obj_metric": (dict(BASE, base_score=0.0), dict(data=X, label=y),
                              dict(obj=sq_obj, custom_metric=mae_metric)),
    }


@pytest.mark.parametrize("case", list(cv_cases()))
def test_cv_equals_sequential_train_loop(E, case):
    params, kw, extra = cv_cases()[case]
    dtrain = E.DMatrix(**kw)
    got = E.cv(params, dtrain, num_boost_round=4, nfold=3, seed=11, as_pandas=False, **extra)
    want = loop_cv(E, params, dtrain, 4, nfold=3, seed=11, **extra)
    assert got == want
    again = E.cv(params, dtrain, num_boost_round=4, nfold=3, seed=11, as_pandas=False, **extra)
    assert again == got


def test_cv_early_stopping_and_learning_rate_schedule(E):
    X, y = data(n=1500)
    params = dict(BASE, eta=0.9, max_depth=6)
    dtrain = E.DMatrix(X, label=y)
    full = loop_cv(E, params, dtrain, 40, nfold=4)
    res = E.cv(params, dtrain, num_boost_round=40, nfold=4, early_stopping_rounds=3, as_pandas=False)
    means = full["test-rmse-mean"]
    best, stop = 0, None
    for r in range(1, len(means)):
        if means[r] < means[best]:
            best = r
        elif r - best >= 3:
            stop = r
            break
    assert stop is not None, "the case must stop early"
    assert res == {k: v[: best + 1] for k, v in full.items()}

    rates = [0.3, 0.2, 0.1, 0.05, 0.02]   # rate i is set after round i
    got = E.cv(BASE, dtrain, num_boost_round=5, nfold=3, callbacks=[E.LearningRateScheduler(rates)], as_pandas=False)
    want = loop_cv(E, BASE, dtrain, 5, nfold=3, callbacks=lambda: [E.LearningRateScheduler(rates)])
    assert got == want


def test_cv_dataframe_and_verbose_lines(E, capsys):
    pd = pytest.importorskip("pandas")
    X, y = data(n=1000)
    dtrain = E.DMatrix(X, label=y)
    df = E.cv(BASE, dtrain, num_boost_round=3, nfold=3, metrics=["mae", "rmse"], verbose_eval=True)
    assert isinstance(df, pd.DataFrame)
    assert list(df.columns) == ["train-mae-mean", "train-mae-std", "train-rmse-mean", "train-rmse-std",
                                "test-mae-mean", "test-mae-std", "test-rmse-mean", "test-rmse-std"]
    lines = capsys.readouterr().out.strip().split("\n")
    assert len(lines) == 3
    for r, ln in enumerate(lines):
        want = "[%d]" % r + "".join("\t%s-%s:%.5f+%.5f" % (d, m, df["%s-%s-mean" % (d, m)][r], df["%s-%s-std" % (d, m)][r])
                                    for d in ("train", "test") for m in ("mae", "rmse"))
        assert ln == want
