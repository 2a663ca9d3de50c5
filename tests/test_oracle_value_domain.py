"""The CPU oracle's cuts and bins at the edges of the float domain and with a non-NaN `missing`, against known
answers derived by hand from A.2 (DESIGN.md §2 items 1-2), and the model file's treatment of non-finite split
conditions.  The GPU side is tests/test_gpu_value_domain.py.

A.2 for a numeric feature: the distinct non-missing values v_0 < ... < v_{m-1} (-0.0 counted as +0.0); without
pruning (m <= cap + 1, cap = max_bin, or 255 when the feature has missing values and max_bin > 255) the cuts are
v_1 .. v_{r-1} with r = min(m, cap), then v_{m-1} + (|v_{m-1}| + 1e-5); min = v_0 - |v_0| - 1e-5, all in binary32.
A value's bin is upper_bound(cuts, x) clamped to the last bin; a missing value's bin is 255."""
import json
import pickle

import numpy as np
import pytest

F = np.float32
FLT_MAX = np.finfo(F).max
TINY = np.array([1], np.uint32).view(F)[0]          # 1e-45, the smallest subnormal
MISSING_BIN = 255


def is_missing(x, missing):
    return np.isnan(x) | (False if np.isnan(missing) else x == F(missing))


def hand_cuts(col, max_bin, missing=np.nan):
    """A.2 without pruning, restated in NumPy binary32: (cuts, min, has_missing)"""
    col = np.asarray(col, F)
    miss = is_missing(col, missing)
    v = np.unique(col[~miss] + F(0.0))                  # -0.0 + 0.0 == +0.0
    cap = 255 if miss.any() and max_bin > 255 else max_bin
    m = len(v)
    assert m <= min(m, cap) + 1, "pruned: no hand answer"
    with np.errstate(over="ignore"):
        if m == 0:
            mn = F(F(0.0) - F(0.0)) - F(1e-5)
            return np.array([mn + (abs(mn) + F(1e-5))], F), mn, bool(miss.any())
        r = min(m, cap)
        last = v[-1] + F(abs(v[-1]) + F(1e-5))
        mn = F(v[0] - abs(v[0])) - F(1e-5)
    return np.append(v[1:r], last).astype(F), F(mn), bool(miss.any())


def hand_bins(col, cuts, missing=np.nan):
    col = np.asarray(col, F)
    b = np.minimum(np.searchsorted(cuts, col, side="right"), len(cuts) - 1)
    return np.where(is_missing(col, missing), MISSING_BIN, b).astype(np.uint8)


def oracle_cuts(oracle, col, max_bin=256, missing=np.nan, weight=None):
    X = np.asarray(col, F).reshape(-1, 1)
    c = oracle.Cuts.from_data(X, max_bin, missing, weight=weight)
    return c, c.vals[c.ptrs[0]:c.ptrs[1]], c.mins[0], bool(c.has_missing[0]), c.bin(X, missing)[:, 0]


def bits(a):
    return np.asarray(a, F).view(np.uint32)


def assert_known_answer(oracle, col, want_cuts, want_min, want_missing, missing=np.nan, max_bin=256):
    c, cuts, mn, hm, b = oracle_cuts(oracle, col, max_bin, missing)
    assert np.array_equal(bits(cuts), bits(want_cuts)), (cuts, want_cuts)
    assert bits(mn) == bits(want_min), (mn, want_min)
    assert hm == want_missing
    assert np.array_equal(b, hand_bins(col, want_cuts, missing))
    hc, hmn, hhm = hand_cuts(col, max_bin, missing)     # the restatement agrees with the hand-written answer
    assert np.array_equal(bits(hc), bits(want_cuts)) and bits(hmn) == bits(want_min) and hhm == want_missing
    return b


# ------------------------------------------------------------------ hand-derived cuts
def test_flt_max_column(oracle):
    # min = -FLT_MAX - FLT_MAX overflows to -inf, the last cut FLT_MAX + FLT_MAX to +inf
    col = [FLT_MAX, 1, -FLT_MAX, 0]
    b = assert_known_answer(oracle, col, [0, 1, FLT_MAX, np.inf], -np.inf, False)
    assert list(b) == [3, 2, 0, 1]                      # FLT_MAX lands in the +inf cut's bin, below it: bin 3


def test_subnormals_and_signed_zeros(oracle):
    # 1e-45 + (1e-45 + 1e-5) rounds to 1e-5; -0.0 is +0.0
    col = [TINY, -TINY, 0.0, -0.0]
    b = assert_known_answer(oracle, col, [0, TINY, F(1e-5)], F(F(-TINY - TINY) - F(1e-5)), False)
    assert list(b) == [2, 0, 1, 1]                      # -0.0 in the bin of +0.0


def test_plus_inf_with_nan(oracle):
    # distinct {1, 2, inf}: the cuts 2, inf and inf + inf = inf; the repeated +inf cut is kept
    col = [np.inf, np.nan, 1, 2]
    b = assert_known_answer(oracle, col, [2, np.inf, np.inf], F(F(1 - 1) - F(1e-5)), True)
    assert list(b) == [2, MISSING_BIN, 0, 1]


def test_minus_inf_column(oracle):
    col = [-np.inf, 3, 5, -np.inf]
    b = assert_known_answer(oracle, col, [3, 5, F(5 + F(5 + F(1e-5)))], -np.inf, False)
    assert list(b) == [0, 1, 2, 0]


def test_missing_zero_takes_negative_zero(oracle):
    col = [0.0, -0.0, 1, 2, np.nan, 3]
    b = assert_known_answer(oracle, col, [2, 3, F(3 + F(3 + F(1e-5)))], F(F(1 - 1) - F(1e-5)), True, missing=0.0)
    assert list(b) == [MISSING_BIN, MISSING_BIN, 0, 1, MISSING_BIN, 2]


@pytest.mark.parametrize("missing,want_cuts,want_bins", [
    (-999.0, [1, np.inf, np.inf], [MISSING_BIN, 0, 1, 2, MISSING_BIN, 2]),
    (np.inf, [1, F(1 + F(1 + F(1e-5)))], [0, 0, 1, MISSING_BIN, MISSING_BIN, MISSING_BIN])])
def test_sentinels(oracle, missing, want_cuts, want_bins):
    # -999 and +inf as the sentinel: NaN stays missing too, the other infinity is a value
    col = [-999.0, 0.0, 1.0, np.inf, np.nan, np.inf]
    if missing == np.inf:
        col = [0.0, -0.0, 1.0, np.inf, np.nan, np.inf]
    b = assert_known_answer(oracle, col, want_cuts, F(-1e-5), True, missing=missing)
    assert list(b) == want_bins


def test_all_missing_and_sentinel_only_columns(oracle):
    one = hand_cuts([np.nan], 256)
    assert_known_answer(oracle, [np.nan] * 5, one[0], one[1], True)
    assert_known_answer(oracle, [-999.0, np.nan, -999.0], one[0], one[1], True, missing=-999.0)
    c, cuts, mn, hm, b = oracle_cuts(oracle, [7.0, 7.0], 256, -999.0)   # sentinel absent: no missing
    assert not hm and list(b) == [0, 0]


@pytest.mark.parametrize("max_bin,m", [(256, 254), (256, 255), (256, 256), (256, 257), (16, 15), (16, 16), (16, 17)])
@pytest.mark.parametrize("with_missing", [False, True])
def test_prune_boundary_distinct_counts(oracle, max_bin, m, with_missing):
    rng = np.random.RandomState(m)
    vals = (np.arange(m, dtype=np.float64) * 0.75 - 40).astype(F)
    col = np.concatenate([vals, rng.choice(vals, 300)]).astype(F)
    if with_missing:
        col[rng.uniform(size=col.size) < 0.1] = np.nan
        col[:m] = vals                                  # keep every distinct value present
    c, cuts, mn, hm, b = oracle_cuts(oracle, col, max_bin)
    cap = 255 if with_missing and max_bin > 255 else max_bin
    assert hm == with_missing
    assert cuts[-1] == F(vals[-1] + F(abs(vals[-1]) + F(1e-5)))
    if m <= cap + 1:                                    # no pruning: every distinct value but the first is a cut
        assert len(cuts) == min(m, cap)
        hc, hmn, _ = hand_cuts(col, max_bin)
        assert np.array_equal(bits(cuts), bits(hc)) and bits(mn) == bits(hmn)
    else:                                               # pruned (unequal ranks merge picks): increasing data values
        assert 2 <= len(cuts) <= cap
        assert np.all(np.diff(cuts) > 0) and np.all(np.isin(cuts[:-1], vals)) and cuts[0] > vals[0]
    assert np.array_equal(b, hand_bins(col, cuts))
    if m <= cap:                                        # one bin per distinct value
        assert len(np.unique(b[~np.isnan(col)])) == m


# ------------------------------------------------------------------ non-finite split conditions in the model file
def _strict_loads(raw):
    def bad(c):
        raise ValueError("non-JSON constant %r in the model file" % c)
    return json.loads(raw, parse_constant=bad)


def _engine_tree(t):
    return {k: np.array(getattr(t, k)) for k in ("left", "right", "parent", "split_feature", "split_bin", "split_cond",
                                                 "default_left", "value", "base_weight", "loss_chg", "sum_hess",
                                                 "split_type", "cat_bits")}


def _hand_tree(conds):
    """a root on feature 0 and one numeric node per further condition down the left spine, plus a categorical node"""
    k = len(conds)
    n = 2 * k + 3
    left, right, parent = np.full(n, -1, np.int32), np.full(n, -1, np.int32), np.full(n, -1, np.int32)
    feat = np.full(n, -1, np.int32)
    for i in range(k + 1):                              # inner nodes 0..k, node k is categorical
        left[i], right[i] = (i + 1 if i < k else 2 * k + 1), k + 1 + i if i < k else 2 * k + 2
        parent[left[i]] = parent[right[i]] = i
        feat[i] = i % 2
    st = np.zeros(n, np.uint8)
    st[k] = 1
    bits = np.zeros((n, 8), np.uint32)
    bits[k, 0] = 0b1010
    cond = np.zeros(n, F)
    cond[:k] = conds
    cond[k] = np.nan
    leaf = feat < 0
    value = np.where(leaf, np.arange(n, dtype=F) * F(0.125) - F(1), 0).astype(F)
    cond[leaf] = value[leaf]
    return dict(left=left, right=right, parent=parent, split_feature=feat,
                split_bin=np.where(leaf, -1, np.arange(n) % 7).astype(np.int32), split_cond=cond,
                default_left=(np.arange(n) % 2).astype(np.uint8), value=value, base_weight=value.copy(),
                loss_chg=np.where(leaf, 0, 1.5).astype(F), sum_hess=np.full(n, 4.0), split_type=st, cat_bits=bits)


def _booster(trees, n_features=2, dart=False):
    from xgboost_ray_b200 import engine as E
    params = {"objective": "reg:squarederror", "base_score": 0.5}
    if dart:
        params.update(booster="dart", rate_drop=0.1)
    b = E.Booster(params)
    b.n_features = n_features
    b._trees = [dict(t) for t in trees]
    if dart:
        b._weights = np.linspace(0.5, 1.0, len(trees)).astype(F)
    return b


def _assert_same_trees(a, b):
    assert len(a) == len(b)
    for t, u in zip(a, b):
        for k in ("left", "right", "parent", "split_feature", "split_bin", "default_left", "split_type", "cat_bits"):
            assert np.array_equal(t[k], u[k]), k
        leaf = t["split_feature"] < 0
        num = ~leaf & (t["split_type"] == 0)
        assert np.array_equal(bits(t["value"][leaf]), bits(u["value"][leaf]))
        assert np.array_equal(bits(t["split_cond"][num]), bits(u["split_cond"][num])), (t["split_cond"], u["split_cond"])


@pytest.mark.parametrize("dart", [False, True])
def test_infinite_conditions_survive_the_model_file_and_pickle(tmp_path, dart):
    from xgboost_ray_b200 import engine as E
    conds = [np.inf, -np.inf, FLT_MAX, F(2.5), -FLT_MAX, F(-0.0)]
    trees = [_hand_tree(conds), _hand_tree([F(1.0), np.inf])]
    b = _booster(trees, dart=dart)
    raw = bytes(b.save_raw())
    d = _strict_loads(raw.decode())                     # strict JSON: no Infinity literal
    gb = d["learner"]["gradient_booster"]
    t0 = (gb["gbtree"] if dart else gb)["model"]["trees"][0]
    # a stock reader sees the nearest finite float32
    assert t0["split_conditions"][:6] == [float(FLT_MAX), float(-FLT_MAX), float(FLT_MAX), 2.5, float(-FLT_MAX), 0.0]
    assert json.loads(d["learner"]["attributes"]["b2.split_conds"]) == [[0, 0, "inf"], [0, 1, "-inf"], [1, 1, "inf"]]
    f = str(tmp_path / "m.json")
    b.save_model(f)
    for b2 in (E.Booster(model_file=f), pickle.loads(pickle.dumps(b)), b.copy()):
        _assert_same_trees(b._trees, b2._trees)
        assert bytes(b2.save_raw()) == raw
        assert "b2.split_conds" not in b2.attributes()  # engine-private, not a user attribute
    assert np.isposinf(pickle.loads(pickle.dumps(b))._trees[0]["split_cond"][0])


def test_finite_conditions_leave_the_file_unchanged():
    b = _booster([_hand_tree([F(1.0), F(-3.0)])])
    d = _strict_loads(bytes(b.save_raw()).decode())
    assert "b2.split_conds" not in d["learner"]["attributes"]


def test_saved_file_with_infinite_condition_validates_against_the_schema():
    import jsonschema
    from tests.model_schema import MODEL
    b = _booster([_hand_tree([np.inf, -np.inf])])
    jsonschema.validate(_strict_loads(bytes(b.save_raw()).decode()), MODEL)


def _inf_split_case(rng, n, replace):
    """a column 0..19 with 19 replaced by FLT_MAX (or a tenth of it by +inf), a tenth NaN, label 5 * isnan(x): the best
    root split sends every real bin left and the missing rows right, so its condition is the last cut, +inf"""
    x = rng.randint(0, 20, size=n).astype(F)
    if replace == "flt_max":
        x[x == 19] = FLT_MAX
    else:
        x[rng.uniform(size=n) < 0.1] = np.inf
    x[rng.uniform(size=n) < 0.1] = np.nan
    X = np.stack([x, rng.uniform(0, 1, size=n).astype(F)], axis=1)
    return X, (5.0 * np.isnan(x)).astype(F)


@pytest.mark.parametrize("replace", ["flt_max", "inf"])
def test_oracle_grows_an_infinite_condition_and_the_model_file_keeps_it(oracle, tmp_path, replace):
    from xgboost_ray_b200 import engine as E
    X, y = _inf_split_case(np.random.RandomState(3), 4000, replace)
    params = {"objective": "reg:squarederror", "max_depth": 3, "base_score": 0.5}
    obst, _ = oracle.train(params, X, y, 2)
    root = obst.tree(0)
    last_bin = obst.cuts.ptrs[1] - 1                    # 19 with FLT_MAX, 20 with +inf (cuts ..., 19, inf, inf)
    assert root.split_feature[0] == 0 and root.split_bin[0] == last_bin and np.isposinf(root.split_cond[0])
    assert root.default_left[0] == 0
    b = _booster([_engine_tree(t) for t in obst.trees()])
    f = str(tmp_path / "m.json")
    b.save_model(f)
    for b2 in (E.Booster(model_file=f), pickle.loads(pickle.dumps(b))):
        _assert_same_trees(b._trees, b2._trees)


# ------------------------------------------------------------------ borrowed categorical cuts and missing values
def _cat_columns(rng, n, codes, missing_frac=0.0):
    X = np.stack([rng.uniform(0, 10, size=n), rng.choice(np.asarray(codes, F), size=n)], axis=1).astype(F)
    X[:len(codes), 1] = codes
    if missing_frac:
        X[rng.uniform(size=n) < missing_frac, 1] = np.nan
    return X


def test_borrowed_categorical_cuts_mark_missing_values(oracle):
    """cuts of codes 0..9 without missing values, borrowed by even codes with NaN: bin 255 of the categorical feature
    must be routed by the default direction, as prediction routes NaN; with the borrowed has_missing = 0 the scan
    takes it for an unknown category and the training margin disagrees with predict_margin"""
    rng = np.random.RandomState(5)
    X1 = _cat_columns(rng, 5000, range(10))
    X2 = _cat_columns(rng, 20011, range(0, 10, 2), missing_frac=0.05)
    y = (np.isin(X2[:, 1], [2, 6]) * 3 + X2[:, 0] * 0.2 + rng.normal(scale=0.1, size=len(X2))).astype(F)
    params = {"objective": "reg:squarederror", "max_depth": 4, "base_score": 0.5}
    borrowed = oracle.Cuts.from_data(X1, 256, is_cat=[0, 1])
    assert list(borrowed.has_missing) == [0, 0]
    assert list(borrowed.borrowed_by(X1).has_missing) == [0, 0]           # nothing missing: the same cuts
    assert list(borrowed.borrowed_by(X2).has_missing) == [0, 1]
    X2num = X2.copy()
    X2num[:100, 0] = np.nan                                             # a numeric feature keeps its flag
    assert list(borrowed.borrowed_by(X2num).has_missing) == [0, 1]
    bst, _ = oracle.train(params, X2, y, 3, cuts=borrowed)
    assert any(t.split_type.any() for t in bst.trees())
    assert np.array_equal(bst.margin[:, 0], bst.predict_margin(X2)[:, 0])
    raw = oracle.Booster(params, borrowed)                              # without the rule
    raw.init_margin(len(X2))
    for _ in range(3):
        raw.boost(borrowed.bin(X2), y)
    assert not np.array_equal(raw.margin[:, 0], raw.predict_margin(X2)[:, 0])
