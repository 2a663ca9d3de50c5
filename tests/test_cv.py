"""cv() and DMatrix.slice without a device: the folds against an independent restatement of xgboost's mknfold /
mkgroupfold, the aggregation of the folds' eval strings, the callback loop of cv() driven by stand-in fold boosters,
the row checks of slice() and the lazy host rows of a slice.  tests/test_gpu_cv.py runs the same on the device."""
import re

import numpy as np
import pytest

from xgboost_ray_b200 import engine as E


# ----------------------------------------------------------------------------- folds
def restated_nfold(n, nfold, seed, shuffle):
    np.random.seed(seed)
    idx = np.random.permutation(n) if shuffle else np.arange(n)
    tests = np.array_split(idx, nfold)
    out = []
    for k in range(nfold):
        train = []
        for i in range(nfold):
            if i != k:
                train.extend(tests[i].tolist())
        out.append((np.array(train, np.int64), tests[k]))
    return out


def restated_groupfold(sizes, nfold, seed, shuffle):
    np.random.seed(seed)
    ptr = [0]
    for s in sizes:
        ptr.append(ptr[-1] + s)
    idx = np.random.permutation(len(sizes)) if shuffle else np.arange(len(sizes))
    test_groups = np.array_split(idx, nfold)
    out = []
    for k in range(nfold):
        train_groups = [g for i in range(nfold) if i != k for g in test_groups[i]]
        rows = lambda gs: np.array([r for g in gs for r in range(ptr[g], ptr[g + 1])], np.int64)  # noqa: E731
        out.append((rows(train_groups), rows(test_groups[k]), np.array([sizes[g] for g in train_groups]),
                    np.array([sizes[g] for g in test_groups[k]])))
    return out


@pytest.mark.parametrize("n,nfold", [(100, 5), (103, 5), (10, 3), (7, 7)])
@pytest.mark.parametrize("shuffle", [True, False])
def test_row_folds_match_mknfold(n, nfold, shuffle):
    got = E.cv_folds(n, nfold, seed=3, shuffle=shuffle)
    want = restated_nfold(n, nfold, 3, shuffle)
    assert len(got) == nfold
    for (tr, te, gtr, gte), (wtr, wte) in zip(got, want):
        assert np.array_equal(tr, wtr) and np.array_equal(te, wte)
        assert gtr is None and gte is None
        assert sorted(np.r_[tr, te].tolist()) == list(range(n))


def test_seed_picks_the_permutation():
    a = E.cv_folds(50, 3, seed=0)
    b = E.cv_folds(50, 3, seed=0)
    c = E.cv_folds(50, 3, seed=1)
    assert all(np.array_equal(x[1], y[1]) for x, y in zip(a, b))
    assert not all(np.array_equal(x[1], y[1]) for x, y in zip(a, c))


def test_stratified_folds_are_sklearns():
    sk = pytest.importorskip("sklearn.model_selection")
    y = np.random.RandomState(0).randint(0, 3, size=91).astype(np.float32)
    got = E.cv_folds(y.size, 4, label=y, stratified=True, seed=7)
    want = list(sk.StratifiedKFold(n_splits=4, shuffle=True, random_state=7).split(X=y, y=y))
    assert len(got) == 4
    for (tr, te, _, _), (wtr, wte) in zip(got, want):
        assert np.array_equal(tr, wtr) and np.array_equal(te, wte)


def test_folds_as_pairs_and_as_a_splitter():
    sk = pytest.importorskip("sklearn.model_selection")
    pairs = [(np.array([0, 1, 2]), np.array([3, 4])), ([4, 3], [0]), ((1,), (2, 2))]
    got = E.cv_folds(5, 99, folds=pairs)
    assert len(got) == 3
    for (tr, te, g1, g2), (a, b) in zip(got, pairs):
        assert np.array_equal(tr, np.asarray(a)) and np.array_equal(te, np.asarray(b)) and g1 is None and g2 is None
    y = np.arange(20, dtype=np.float32)
    kf = sk.KFold(n_splits=4, shuffle=True, random_state=2)
    got = E.cv_folds(20, 3, label=y, folds=kf)
    want = list(kf.split(X=y, y=y))
    assert len(got) == 4
    for (tr, te, _, _), (wtr, wte) in zip(got, want):
        assert np.array_equal(tr, wtr) and np.array_equal(te, wte)


@pytest.mark.parametrize("shuffle", [True, False])
@pytest.mark.parametrize("nfold", [2, 3, 4])
def test_group_folds_match_mkgroupfold(shuffle, nfold):
    sizes = np.random.RandomState(nfold).randint(1, 9, size=11)
    got = E.cv_folds(int(sizes.sum()), nfold, group_sizes=sizes, seed=5, shuffle=shuffle)
    want = restated_groupfold(sizes.tolist(), nfold, 5, shuffle)
    for g, w in zip(got, want):
        for a, b in zip(g, w):
            assert np.array_equal(a, b)
        assert g[2].sum() == g[0].size and g[3].sum() == g[1].size


def test_fold_refusals():
    for bad in (1, 0, -2, 2.5, True):
        with pytest.raises(E.XGBoostError, match="nfold must be an integer >= 2"):
            E.cv_folds(10, bad)
    with pytest.raises(E.XGBoostError, match="list of \\(train_idx, test_idx\\) pairs or an object with split"):
        E.cv_folds(10, 3, folds=[1, 2])
    with pytest.raises(E.XGBoostError, match="list of \\(train_idx, test_idx\\) pairs or an object with split"):
        E.cv_folds(10, 3, folds=5)
    with pytest.raises(E.XGBoostError, match="must be a \\(train_idx, test_idx\\) pair"):
        E.cv_folds(10, 3, folds=[([0, 1],)])
    with pytest.raises(E.XGBoostError, match="holds no fold"):
        E.cv_folds(10, 3, folds=[])


# ----------------------------------------------------------------------------- aggregation
def test_aggcv_is_mean_and_population_std_of_the_printed_values():
    msgs = ["[4]\ttrain-rmse:0.125000\ttrain-mae:0.100000\ttest-rmse:0.250001\ttest-mae:0.200000",
            "[4]\ttrain-rmse:0.135000\ttrain-mae:0.110000\ttest-rmse:0.270003\ttest-mae:0.190000",
            "[4]\ttrain-rmse:0.115000\ttrain-mae:0.090000\ttest-rmse:0.230000\ttest-mae:0.210007"]
    got = E.aggcv(msgs)
    assert [k for k, _, _ in got] == ["train-rmse", "train-mae", "test-rmse", "test-mae"]
    for j, (k, mean, std) in enumerate(got):
        vals = np.array([float(m.split("\t")[j + 1].split(":")[1]) for m in msgs])
        assert mean == np.mean(vals) and std == np.std(vals)
    assert E.aggcv(["[0]\ttest-ndcg@5-:0.500000"]) == [("test-ndcg@5-", 0.5, 0.0)]
    with pytest.raises(E.XGBoostError, match="different rounds"):
        E.aggcv(["[1]\ttest-rmse:0.1", "[2]\ttest-rmse:0.1"])


# ----------------------------------------------------------------------------- the cv() loop
class FakeMatrix:
    """Rows and query groups; slice() keeps the rows it was given."""

    def __init__(self, rows, label=None, groups=None):
        self.rows = np.asarray(rows)
        self.label = np.zeros(self.rows.size, np.float32) if label is None else label
        self._group_sizes = groups
        self.allow = []

    def num_row(self):
        return self.rows.size

    def get_label(self):
        return self.label

    def slice(self, idx, allow_groups=False):
        self.allow.append(allow_groups)
        return FakeMatrix(self.rows[np.asarray(idx)], self.label[np.asarray(idx)])

    def set_group(self, g):
        self._group_sizes = np.asarray(g)


class FakeBooster:
    """Metric value of round r on a side = a fixed curve plus the mean row id of that side (so folds differ)."""
    made = []

    def __init__(self, params):
        self.params = dict(params)
        self.rounds, self.eta_log, self.best_iteration, self.best_score, self._attrs = 0, [], None, None, {}
        FakeBooster.made.append(self)

    def _attach(self, d):
        self.train = d

    def update(self, d, it, fobj=None):
        assert d is self.train and it == self.rounds
        self.rounds += 1

    def num_boosted_rounds(self):
        return self.rounds

    def set_param(self, k, v=None):
        self.eta_log.append((k, v))

    def set_attr(self, **kw):
        self._attrs.update(kw)

    def attr(self, k):
        return self._attrs.get(k)

    def eval_set(self, evals, it, feval=None, output_margin=True):
        parts = ["[%d]" % it]
        for d, name in evals:
            for m in (self.params.get("eval_metric") or ["rmse"]):
                v = CURVE[min(it, len(CURVE) - 1)] + (0.5 if name == "test" else 0) + d.rows.mean() * 1e-3
                parts.append("%s-%s:%.6f" % (name, m, v))
        return "\t".join(parts)


CURVE = [1.0, 0.8, 0.7, 0.65, 0.66, 0.67, 0.68, 0.69, 0.70, 0.71]


@pytest.fixture
def fake(monkeypatch):
    FakeBooster.made = []
    monkeypatch.setattr(E, "Booster", FakeBooster)
    return FakeMatrix(np.arange(60))


def test_cv_keys_values_and_forms(fake):
    pd = pytest.importorskip("pandas")
    res = E.cv({"eval_metric": "mae"}, fake, num_boost_round=4, nfold=3, metrics=["rmse", "mae"], as_pandas=False)
    assert list(res) == ["train-rmse-mean", "train-rmse-std", "train-mae-mean", "train-mae-std",
                         "test-rmse-mean", "test-rmse-std", "test-mae-mean", "test-mae-std"]
    assert all(len(v) == 4 for v in res.values())
    assert [b.params["eval_metric"] for b in FakeBooster.made] == [["rmse", "mae"]] * 3
    for r in range(4):
        msgs = [b.eval_set([(b.train, "train"), (b.train, "test")], r) for b in FakeBooster.made]
        tr = np.array([float(m.split("\t")[1].split(":")[1]) for m in msgs])
        assert res["train-rmse-mean"][r] == np.mean(tr) and res["train-rmse-std"][r] == np.std(tr)
    df = E.cv({"eval_metric": "mae"}, fake, num_boost_round=4, nfold=3)
    assert isinstance(df, pd.DataFrame) and list(df.columns) == ["train-mae-mean", "train-mae-std", "test-mae-mean",
                                                                  "test-mae-std"]
    assert df.shape == (4, 4)


def test_cv_early_stopping_truncates_to_the_best_round(fake):
    res = E.cv({}, fake, num_boost_round=10, nfold=3, early_stopping_rounds=2, as_pandas=False)
    # test mean falls until round 3 and rises after: rounds 4 and 5 do not improve, so training stops after round 5
    assert len(res["test-rmse-mean"]) == 4
    assert all(b.rounds == 6 and b.best_iteration == 3 for b in FakeBooster.made)
    assert FakeBooster.made[0].best_score == res["test-rmse-mean"][3]
    res = E.cv({}, fake, num_boost_round=10, nfold=3, early_stopping_rounds=2, maximize=True, as_pandas=False)
    assert len(res["test-rmse-mean"]) == 1


def test_cv_callbacks_see_one_model_and_mean_std_history(fake):
    seen = []

    class Probe(E.TrainingCallback):
        def after_iteration(self, model, epoch, evals_log):
            seen.append((epoch, {d: {m: list(v) for m, v in log.items()} for d, log in evals_log.items()}))
            return epoch == 2

    res = E.cv({}, fake, num_boost_round=6, nfold=3, callbacks=[Probe(), E.LearningRateScheduler([0.3, 0.2, 0.1])],
               as_pandas=False)
    assert len(res["test-rmse-mean"]) == 3   # stopped by a callback without best_iteration: nothing is cut
    last = seen[-1][1]
    assert last["test"]["rmse"] == list(zip(res["test-rmse-mean"], res["test-rmse-std"]))
    for b in FakeBooster.made:
        assert b.eta_log == [("learning_rate", 0.3), ("learning_rate", 0.2), ("learning_rate", 0.1)]


def test_cv_verbose_lines(fake, capsys):
    res = E.cv({}, fake, num_boost_round=5, nfold=3, verbose_eval=2, as_pandas=False)
    lines = capsys.readouterr().out.strip().split("\n")
    assert [ln.split("\t")[0] for ln in lines] == ["[0]", "[2]", "[4]"]
    for ln in lines:
        r = int(ln[1:ln.index("]")])
        assert ln == "[%d]\ttrain-rmse:%.5f+%.5f\ttest-rmse:%.5f+%.5f" % (
            r, res["train-rmse-mean"][r], res["train-rmse-std"][r], res["test-rmse-mean"][r], res["test-rmse-std"][r])
        assert re.fullmatch(r"\[\d+\](\t(train|test)-rmse:\d+\.\d{5}\+\d+\.\d{5}){2}", ln)
    E.cv({}, fake, num_boost_round=4, nfold=3, verbose_eval=3, show_stdv=False, as_pandas=False)
    lines = capsys.readouterr().out.strip().split("\n")
    assert [ln.split("\t")[0] for ln in lines] == ["[0]", "[3]"] and "+" not in lines[0]


def test_cv_slices_whole_groups(fake):
    fake._group_sizes = np.array([10, 20, 30])
    E.cv({}, fake, num_boost_round=1, nfold=3, as_pandas=False)
    assert fake.allow == [True] * 6
    for b in FakeBooster.made:
        assert b.train._group_sizes.sum() == b.train.rows.size


def test_cv_refusals(fake):
    with pytest.raises(E.XGBoostError, match="save_best=True"):
        E.cv({}, fake, callbacks=[E.EarlyStopping(2, save_best=True)])
    with pytest.raises(E.XGBoostError, match="nfold must be an integer >= 2"):
        E.cv({}, fake, nfold=1)
    with pytest.raises(E.XGBoostError, match="pairs or an object with split"):
        E.cv({}, fake, folds=[3, 4])


# ----------------------------------------------------------------------------- slice rows
def test_slice_row_checks():
    assert E.slice_rows([3, 0, 3], 4).tolist() == [3, 0, 3]
    assert E.slice_rows(np.array([1], np.uint8), 2).dtype == np.int64
    with pytest.raises(E.XGBoostError, match=r"rindex\[2\] = 4 is outside \[0, 4\)"):
        E.slice_rows([0, 1, 4], 4)
    with pytest.raises(E.XGBoostError, match=r"rindex\[1\] = -1 is outside \[0, 4\)"):
        E.slice_rows([0, -1], 4)
    with pytest.raises(E.XGBoostError, match=r"rindex\[1\] = 1.5 is not an integer"):
        E.slice_rows([0, 1.5], 4)
    with pytest.raises(E.XGBoostError, match=r"rindex\[0\] = True is not an integer"):
        E.slice_rows([True, False], 4)
    with pytest.raises(E.XGBoostError, match="rindex is empty"):
        E.slice_rows([], 4)


def test_slice_host_rows_are_the_parents_rows():
    sp = pytest.importorskip("scipy.sparse")
    rng = np.random.RandomState(0)
    X = rng.rand(30, 5).astype(np.float32)
    X[X < 0.4] = 0
    idx = np.array([7, 3, 3, 29, 0, 12])
    assert np.array_equal(E._SliceRows(X, idx).rows(), X[idx])
    blocks = E._BlockList([X[:10], X[10:]])
    assert np.array_equal(E._SliceRows(blocks, idx).rows(), X[idx])
    c = E.canonical_csr(sp.csr_matrix(X))
    got = E._SliceRows(c, idx).rows()
    want = E.canonical_csr(sp.csr_matrix(X[idx]))
    for a in ("indptr", "indices", "values"):
        assert np.array_equal(getattr(got, a), getattr(want, a))
    assert got.shape == (6, 5)
    two = E._SliceRows(E._SliceRows(X, idx), np.array([5, 0]))   # a slice of a slice indexes the first parent
    assert two.host is X and np.array_equal(two.rows(), X[[12, 7]])
