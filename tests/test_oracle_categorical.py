"""Known-answer tests for the categorical part of the oracle (SURVEY.md A.2 / A.6 / A.8; C5 uses 50 categorical
features).  Hand-checkable cases: bin = category code, one-hot below max_cat_to_onehot, sorted-by-weight partition
otherwise, categories in the stored set go RIGHT, missing follows default_left."""
import numpy as np
import pytest

from tests import categorical_reference as CR

P1 = {"objective": "reg:squarederror", "max_depth": 1, "eta": 1.0, "base_score": 0.0, "lambda": 0.0}


def test_categorical_cuts_and_bins(oracle):
    X = np.array([[0.5, 3], [1.5, 0], [2.5, np.nan], [3.5, 5]], np.float32)
    c = oracle.Cuts.from_data(X, 256, is_cat=[0, 1])
    assert list(c.is_cat) == [0, 1]
    # categorical cuts are the codes 0..max (HistogramCuts::AddCategories); the feature has a missing value
    assert list(c.vals[c.ptrs[1]:c.ptrs[2]]) == [0, 1, 2, 3, 4, 5] and c.has_missing[1] == 1
    bins = c.bin(X)
    assert list(bins[:, 1]) == [3, 0, 255, 5]
    # a code the cuts have not seen clamps to the last category
    assert c.bin(np.array([[0.0, 9.0]], np.float32))[0, 1] == 5


@pytest.mark.parametrize("bad", [-1.0, 2.5, 256.0])
def test_invalid_category_is_rejected(oracle, bad):
    X = np.array([[0.0, 1.0], [1.0, bad]], np.float32)
    with pytest.raises(ValueError):
        oracle.Cuts.from_data(X, 256, is_cat=[0, 1])


def test_missing_leaves_254_codes(oracle):
    X = np.array([[255.0], [np.nan]], np.float32)
    with pytest.raises(ValueError):
        oracle.Cuts.from_data(X, 256, is_cat=[1])
    oracle.Cuts.from_data(np.array([[255.0], [3.0]], np.float32), 256, is_cat=[1])   # without missing: 256 codes


def test_onehot_split_known_answer(oracle):
    rng = np.random.RandomState(0)
    n = 300
    c = rng.randint(0, 3, size=n).astype(np.float32)           # 3 categories < max_cat_to_onehot (4)
    X = np.stack([rng.uniform(0, 1, size=n).astype(np.float32), c], 1)
    y = (c == 1).astype(np.float32) * 2.0
    b, _ = oracle.train(P1, X, y, 1, is_cat=[0, 1])
    t = b.tree(0)
    assert t.split_feature[0] == 1 and t.split_type[0] == 1
    assert t.categories(0) == [1]                              # the chosen category goes right
    assert t.split_cond[0] == 1.0 and t.default_left[0] == 1   # no missing: the missing-left variant is enumerated first
    assert t.value[t.left[0]] == 0.0 and t.value[t.right[0]] == 2.0
    assert np.array_equal(b.predict(X), y)


def test_partition_split_known_answer(oracle):
    rng = np.random.RandomState(1)
    n = 400
    c = rng.randint(0, 8, size=n).astype(np.float32)           # 8 categories >= 4: sorted-partition split
    X = np.stack([rng.uniform(0, 1, size=n).astype(np.float32), c], 1)
    y = np.isin(c, [1, 4, 6]).astype(np.float32) * 3.0
    b, _ = oracle.train(P1, X, y, 1, is_cat=[0, 1])
    t = b.tree(0)
    assert t.split_feature[0] == 1 and t.split_type[0] == 1 and np.isnan(t.split_cond[0]) and t.split_bin[0] == -1
    # weights -G/H = mean(y): the light categories {0,2,3,5,7} are the sorted prefix, forward scan sends them right
    assert t.categories(0) == [0, 2, 3, 5, 7] and t.default_left[0] == 1
    assert t.value[t.left[0]] == 3.0 and t.value[t.right[0]] == 0.0
    assert np.array_equal(b.predict(X), y)


def test_partition_respects_max_cat_threshold(oracle):
    rng = np.random.RandomState(2)
    n = 2000
    c = rng.randint(0, 16, size=n).astype(np.float32)
    X = c.reshape(-1, 1)
    y = (c >= 8).astype(np.float32) + 0.01 * c                 # 8 light + 8 heavy categories, all distinct weights
    full, _ = oracle.train(P1, X, y, 1, is_cat=[1])
    assert full.tree(0).categories(0) == list(range(8))
    # with max_cat_threshold=4 a direction may move at most 3 categories: the heavy {13,14,15} go left (backward
    # scan, missing right) or the light {0,1,2} go right (forward); the better one is chosen
    lim, _ = oracle.train(dict(P1, max_cat_threshold=4), X, y, 1, is_cat=[1])
    cats = lim.tree(0).categories(0)
    assert cats in ([0, 1, 2], list(range(13))), cats


def test_missing_category_follows_default(oracle):
    rng = np.random.RandomState(3)
    n = 600
    c = rng.randint(0, 6, size=n).astype(np.float32)
    y = np.isin(c, [0, 5]).astype(np.float32)
    miss = rng.uniform(size=n) < 0.2
    y[miss] = 1.0                                              # missing rows look like the heavy categories
    c[miss] = np.nan
    X = c.reshape(-1, 1)
    b, bins = oracle.train(P1, X, y, 1, is_cat=[1])
    t = b.tree(0)
    assert t.categories(0) == [1, 2, 3, 4]                     # light categories right ...
    assert t.default_left[0] == 1                              # ... missing with the heavy ones on the left
    assert np.array_equal(b.predict(X), y)
    # unseen / invalid codes at prediction time go left (common/categorical.h Decision)
    out = b.predict(np.array([[77.0], [-3.0], [2.0]], np.float32))
    assert out[0] == t.value[t.left[0]] and out[1] == t.value[t.left[0]] and out[2] == t.value[t.right[0]]


def test_mixed_numeric_and_categorical_multiclass(oracle):
    rng = np.random.RandomState(4)
    n = 3000
    Xn = rng.uniform(0, 10, size=(n, 3)).astype(np.float32)
    c1 = rng.randint(0, 3, size=n); c2 = rng.randint(0, 20, size=n)
    X = np.column_stack([Xn, c1, c2]).astype(np.float32)
    y = ((Xn[:, 0] > 5).astype(int) + (c2 % 3 == 0).astype(int) + (c1 == 2).astype(int)).astype(np.float32)
    params = {"objective": "multi:softprob", "num_class": 4, "max_depth": 4, "eta": 0.5}
    b, _ = oracle.train(params, X, y, 4, is_cat=[0, 0, 0, 1, 1])
    pred = b.predict(X).argmax(1)
    assert (pred == y).mean() > 0.97
    used = set()
    for t in b.trees():
        used |= {(int(f), int(st)) for f, st in zip(t.split_feature, t.split_type) if f >= 0}
    assert (3, 1) in used and (4, 1) in used and (0, 0) in used      # one-hot, partition and numeric splits all occur


# ------------------------------------------------------------------ the oracle against tests/categorical_reference.py
ROOT = {"objective": "reg:squarederror", "max_depth": 1, "eta": 1.0, "base_score": 0.0}
F32 = np.float32
CARDS = [1, 2, 3, 4, 5, 31, 32, 33, 64, 65, 128, 224, 225, 255, 256]


def _root_against_reference(oracle, params, X, y, w=None):
    params = dict(ROOT, **params)
    b, _ = oracle.train(params, X, y, 1, weight=w, is_cat=[1] * X.shape[1])
    g = (F32(0.0) - y).astype(F32) * (F32(1.0) if w is None else w)
    h = np.ones_like(g) if w is None else w.astype(F32)
    split, hist = CR.root_split(X, g.astype(F32), h, int(params.get("hist_qbits", 18)), params)
    CR.root_matches(vars(b.tree(0)), split, hist)
    return split, hist


@pytest.mark.parametrize("seed,params,nan_frac,weighted", [
    (0, {}, 0.0, False),
    (1, {"max_cat_to_onehot": 257}, 0.1, False),               # every feature one-hot, candidate keys up to 2 * 255 + 1
    (2, {"max_cat_threshold": 1}, 0.1, True),                  # no partition candidate: only the one-hot features split
    (3, {"max_cat_threshold": 2, "hist_qbits": 8}, 0.1, False),
    (4, {"max_cat_threshold": 300, "hist_qbits": 24, "lambda": 0.0}, 0.0, True),
    (5, {"max_cat_to_onehot": 33, "alpha": 2.0, "min_child_weight": 40.0}, 0.1, False),
    (6, {"max_cat_to_onehot": 1, "max_delta_step": 0.4, "lambda": 3.0}, 0.1, True),
])
def test_reference_root_scan_matches_oracle_random(oracle, seed, params, nan_frac, weighted):
    X, y, w = CR.random_case(seed, CARDS, 6000, nan_frac, weighted)
    split, _ = _root_against_reference(oracle, params, X, y, w)
    if params.get("max_cat_threshold") == 1:
        assert split["kind"] == "onehot"


@pytest.mark.parametrize("values,thr,kind", [
    ((0.5, 1.0, 2.0, 4.0), 2, "backward"), ((0.5, 1.0, 2.0, 4.0), 6, "backward"),
    ((3.0, 3.5, 4.0), 4, "forward"), ((3.0, 3.5, 4.0), 6, "forward"),
])
def test_reference_root_scan_matches_oracle_ties(oracle, values, thr, kind):
    X, y = CR.tie_case(0, values=values)
    params = {"lambda": 0.5, "min_child_weight": 3.0, "max_cat_threshold": thr}
    split, hist = _root_against_reference(oracle, params, X, y)
    assert split["feature"] == 0 and split["kind"] == kind
    # the chosen set cuts through categories of equal weight (-0.0, +0.0 of empty and light categories included):
    # only the stable order decides which of them go right
    cat_g, cat_h, nf, _, _, sg, sh = hist
    assert CR.tied_across(split, cat_g, cat_h, nf, sg, sh, params)
