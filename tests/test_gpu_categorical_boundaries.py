"""Categorical splits on the H100 at the boundaries of eval_cat_splits_kernel (split_kernel.cu; DESIGN.md §2 item 6):
cardinalities 1-256 (thread 255 of the CTA, word 7 of the category set, bin 255 as a category), the enumeration limits
max_cat_threshold / max_cat_to_onehot at their edges, tied leaf weights built on purpose, deep trees at hist_qbits 8 and
24 with weights, and every path that reads a high-code category set back.  Trees are compared bit for bit with the CPU
oracle; root splits also with tests/categorical_reference.py, a NumPy restatement of the scan.  Every case asserts
that the boundary it names was reached."""
import pickle

import numpy as np
import pytest

from tests import categorical_reference as CR
from tests import shap_reference as R
from tests.test_gpu_parity import assert_same_model

pytestmark = pytest.mark.gpu

F = np.float32
# categorical features in this order: kCatCtas = 4 CTAs take them round-robin, so each CTA scans low and high
# cardinalities (CTA 0: 1, 5, 64, 225; CTA 1: 2, 31, 65, 255; CTA 2: 3, 32, 128, 256; CTA 3: 4, 33, 224, all missing)
CARDS = [1, 2, 3, 4, 5, 31, 32, 33, 64, 65, 128, 224, 225, 255, 256, 0]   # 255: codes 0-254 and NaN; 0: every row NaN
N_NUM = 3
IS_CAT = [0] * N_NUM + [1] * len(CARDS)
TYPES = ["q"] * N_NUM + ["c"] * len(CARDS)
COL = {k: N_NUM + i for i, k in enumerate(CARDS)}         # cardinality -> column
SQ = {"objective": "reg:squarederror", "eta": 0.3, "base_score": 0.0}


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def card_matrix(n=60000, seed=0, nan_frac=0.0):
    """3 numeric columns, then one categorical column per entry of CARDS; every code of a column is present.  Labels
    add a random effect per (column, code), with strong ones at the top codes of the widest columns and on the
    narrowest columns, so that splits on both are chosen."""
    rng = np.random.RandomState(seed)
    cols = [rng.uniform(0, 10, size=n) for _ in range(N_NUM)]
    y = 0.3 * cols[0] + rng.normal(scale=0.2, size=n)
    for k in CARDS:
        if k == 0:
            cols.append(np.full(n, np.nan))
            continue
        c = rng.randint(0, k, size=n).astype(np.float64)
        c[:k] = np.arange(k)
        effect = rng.normal(size=k) * (2.0 if k <= 5 else 1.0)
        if k >= 224:                                # strong effects at the top codes, the last one lightest
            effect[k - 1], effect[k - 30] = -3.0, 3.0
        y += effect[c.astype(int)]
        frac = 0.05 if k == 255 else (nan_frac if k < 255 else 0.0)
        if frac > 0:
            miss = rng.uniform(size=n) < frac
            miss[:k] = False
            c[miss] = np.nan
            y[miss] += 0.7
        cols.append(c)
    return np.column_stack(cols).astype(F), y.astype(F)


def train_both(eng, oracle, params, X, y, rounds, is_cat, w=None):
    obst, _ = oracle.train(params, X, y, rounds, weight=w, is_cat=is_cat)
    types = ["c" if c else "q" for c in is_cat]
    dm = eng.DMatrix(X, label=y, weight=w, feature_types=types, enable_categorical=True)
    ebst = eng.train(params, dm, num_boost_round=rounds, verbose_eval=False)
    assert_same_model(ebst, obst)
    return ebst, obst, dm


def cat_splits(trees):
    """(feature, bin, default_left, category set) of every categorical split; bin -1 = partition, else one-hot."""
    out = []
    for t in trees:
        for nid in np.nonzero((t["split_feature"] >= 0) & (t["split_type"] != 0))[0]:
            w = t["cat_bits"][nid]
            cats = {b for b in range(256) if (int(w[b >> 5]) >> (b & 31)) & 1}
            out.append((int(t["split_feature"][nid]), int(t["split_bin"][nid]), int(t["default_left"][nid]), cats))
    return out


# ------------------------------------------------------------------ cardinality
@pytest.mark.parametrize("extra", [{}, {"max_cat_to_onehot": 257}], ids=["partition", "onehot257"])
def test_cardinalities_1_to_256(eng, oracle, extra):
    X, y = card_matrix(nan_frac=0.1)
    ebst, _, _ = train_both(eng, oracle, dict(SQ, max_depth=6, **extra), X, y, 4, IS_CAT)
    splits = cat_splits(ebst.get_trees())
    used = {f for f, _, _, _ in splits}
    assert COL[255] in used and used & {COL[k] for k in (2, 3, 4, 5)}
    assert any(max(s) >= 224 for _, _, _, s in splits)                       # word 7 of the set
    if extra:                                       # one-hot over up to 256 categories: candidate orders up to 511
        assert all(b >= 0 and len(s) == 1 for _, b, _, s in splits)       # (test_onehot_switch_... takes code 255)
    else:
        assert COL[256] in used
        assert any(255 in s for f, _, _, s in splits if f == COL[256])      # bin 255 as a category, bit 31 of word 7
        assert any(b >= 0 for _, b, _, _ in splits) and any(b < 0 for _, b, _, _ in splits)
        dirs = {dl for _, b, dl, _ in splits if b < 0}
        assert dirs == {0, 1}                       # forward (missing left) and backward (missing right) partitions


@pytest.mark.parametrize("thr", [1, 2, 32, 33, 38, 300])   # 32, 33, 38: nf - 1, nf, nf + 5 of the 33-category column
def test_max_cat_threshold(eng, oracle, thr):
    X, y = card_matrix(n=40000, seed=thr, nan_frac=0.1)
    ebst, _, _ = train_both(eng, oracle, dict(SQ, max_depth=5, max_cat_threshold=thr), X, y, 3, IS_CAT)
    splits = cat_splits(ebst.get_trees())
    assert splits
    if thr == 1:                                    # n_iter = 0: no partition candidate at all
        assert all(b >= 0 for _, b, _, _ in splits)
    else:
        assert any(b < 0 for _, b, _, _ in splits)


# ------------------------------------------------------------------ one feature, one heavy category: root splits
def heavy_case(nf, heavy, n=20000, seed=1, nan_frac=0.05):
    """One categorical column of nf codes, all present; the `heavy` code has label 5, the others small labels and the
    missing rows labels like the light codes.  The best split isolates the heavy code."""
    rng = np.random.RandomState(seed)
    c = rng.randint(0, nf, size=n).astype(F)
    c[:nf] = np.arange(nf)
    y = rng.uniform(0, 0.5, size=n)
    y[c == heavy] = 5.0
    miss = rng.uniform(size=n) < nan_frac
    miss[:nf] = False
    c[miss] = np.nan
    return c.reshape(-1, 1), y.astype(F)


def root_both(eng, oracle, params, X, y, w=None):
    """Root split of one tree against the oracle and the NumPy reference; returns the reference's split."""
    params = dict(SQ, max_depth=1, **params)
    ebst, _, _ = train_both(eng, oracle, params, X, y, 1, [1] * X.shape[1], w)
    g = ((F(0.0) - y) * (F(1.0) if w is None else w)).astype(F)
    h = np.ones_like(g) if w is None else w.astype(F)
    split, hist = CR.root_split(X, g, h, int(params.get("hist_qbits", 18)), params)
    CR.root_matches(ebst.get_trees()[0], split, hist)
    return split, hist


@pytest.mark.parametrize("nf,heavy", [(33, 7), (255, 200), (256, 255)])
def test_threshold_edges_choose_direction(eng, oracle, nf, heavy):
    X, y = heavy_case(nf, heavy, nan_frac=0.0 if nf == 256 else 0.05)
    # one category alone on the left: backward t = 0 always; forward needs nf - 1 steps.  Without missing rows both
    # candidates have the same loss_chg and the forward one (earlier in enumeration) wins
    s, _ = root_both(eng, oracle, {"max_cat_threshold": 2}, X, y)
    assert s["kind"] == "backward" and s["right"] == set(range(nf)) - {heavy}
    s, _ = root_both(eng, oracle, {"max_cat_threshold": nf - 1}, X, y)
    assert s["kind"] == "backward"
    s, _ = root_both(eng, oracle, {"max_cat_threshold": nf}, X, y)
    assert s["kind"] == ("forward" if nf == 256 else "backward")


@pytest.mark.parametrize("nf,heavy", [(5, 3), (64, 40), (256, 255)])
def test_onehot_switch_at_max_cat_to_onehot(eng, oracle, nf, heavy):
    X, y = heavy_case(nf, heavy, nan_frac=0.0 if nf == 256 else 0.1)
    s, _ = root_both(eng, oracle, {"max_cat_to_onehot": nf}, X, y)          # nf == max_cat_to_onehot: partition
    assert s["kind"] != "onehot"
    s, _ = root_both(eng, oracle, {"max_cat_to_onehot": nf + 1}, X, y)      # nf < max_cat_to_onehot: one-hot
    assert s["kind"] == "onehot" and s["right"] == {heavy}
    if nf < 256:                                    # missing rows look light: they stay left with the light codes
        assert s["default_left"] == 1


def test_single_category_and_all_missing(eng, oracle):
    rng = np.random.RandomState(5)
    n = 5000
    X = np.column_stack([np.zeros(n), np.full(n, np.nan), rng.randint(0, 6, size=n)]).astype(F)
    X[rng.uniform(size=n) < 0.2, 0] = np.nan
    y = (X[:, 2] == 4).astype(F) * 2 + rng.uniform(0, 0.1, size=n).astype(F)
    for onehot in (1, 4):
        s, hist = root_both(eng, oracle, {"max_cat_to_onehot": onehot, "min_child_weight": 0.0}, X, y)
        assert s["feature"] == 2 and list(hist[2][:2]) == [1, 1]


# ------------------------------------------------------------------ ties
@pytest.mark.parametrize("values,thr,kind", [
    ((0.5, 1.0, 2.0, 4.0), 2, "backward"), ((0.5, 1.0, 2.0, 4.0), 6, "backward"),
    ((3.0, 3.5, 4.0), 4, "forward"), ((3.0, 3.5, 4.0), 6, "forward"),
])
def test_tied_weights_at_root(eng, oracle, values, thr, kind):
    X, y = CR.tie_case(0, values=values)
    params = {"lambda": 0.5, "min_child_weight": 3.0, "max_cat_threshold": thr}
    s, hist = root_both(eng, oracle, params, X, y)
    assert s["feature"] == 0 and s["kind"] == kind
    cat_g, cat_h, nf, _, _, sg, sh = hist
    assert CR.tied_across(s, cat_g, cat_h, nf, sg, sh, params)


@pytest.mark.parametrize("extra", [{}, {"alpha": 1.5, "lambda": 0.0}, {"max_cat_threshold": 5, "min_child_weight": 8.0}])
def test_tied_weights_deep(eng, oracle, extra):
    X, y = CR.tie_case(3, nf=120, m=60, n_missing=900)
    params = dict(SQ, max_depth=7, **dict({"lambda": 0.5, "min_child_weight": 3.0}, **extra))
    ebst, _, _ = train_both(eng, oracle, params, X, y, 3, [1] * X.shape[1])
    assert any(f == 0 and b < 0 for f, b, _, _ in cat_splits(ebst.get_trees()))


# ------------------------------------------------------------------ depth x hist_qbits x weights
@pytest.mark.parametrize("qbits", [8, 24])
@pytest.mark.parametrize("nan_frac", [0.0, 0.1])
def test_deep_trees_qbits_and_weights(eng, oracle, qbits, nan_frac):
    X, y = card_matrix(n=50000, seed=7 + qbits, nan_frac=nan_frac)
    w = np.random.RandomState(qbits).uniform(0.2, 3.0, size=len(y)).astype(F)
    params = dict(SQ, max_depth=10 + (qbits == 24) * 2, hist_qbits=qbits, max_bin=16, min_child_weight=0.5)
    ebst, _, dm = train_both(eng, oracle, params, X, y, 2, IS_CAT, w)
    ptrs = dm.get_cuts()[0]
    assert ptrs[COL[256] + 1] - ptrs[COL[256]] == 256           # categorical cuts ignore max_bin
    splits = cat_splits(ebst.get_trees())
    assert any(f == COL[256] and 255 in s for f, _, _, s in splits)
    depth_of = lambda t: max(len(bin(i + 1)) - 2 for i in range(len(t["left"])))   # noqa: E731
    assert max(depth_of(t) for t in ebst.get_trees()) >= 10


# ------------------------------------------------------------------ read paths of a high-code model
CAT_PROBES = [-1.0, -0.0, 2.5, 223.0, 224.0, 254.0, 254.9, 255.0, 256.0, 1e9, np.inf, -np.inf, np.nan]


def probe_rows(trees, X, seed=0, max_trees=3):
    rng = np.random.RandomState(seed)
    rows = []
    for t, nid in ((t, nid) for t in trees[:max_trees] for nid in np.nonzero(t["split_type"] != 0)[0]):
        f = int(t["split_feature"][nid])
        w = t["cat_bits"][nid]
        cats = [b for b in range(256) if (int(w[b >> 5]) >> (b & 31)) & 1]
        out = [b for b in range(256) if b not in cats]
        for v in cats[:2] + cats[-2:] + out[:2] + out[-2:] + CAT_PROBES:
            r = X[rng.randint(len(X))].copy()
            r[f] = F(v)
            rows.append(r)
    return np.asarray(rows, F)


def test_read_paths_on_high_code_model(eng, oracle, tmp_path):
    X, y = card_matrix(nan_frac=0.1, seed=11)
    params = dict(SQ, max_depth=6)
    ebst, obst, dm = train_both(eng, oracle, params, X, y, 4, IS_CAT)
    trees = ebst.get_trees()
    assert any(255 in s for f, _, _, s in cat_splits(trees[:3]) if f == COL[256])
    P = np.concatenate([X[:2000], probe_rows(trees, X)])
    d = eng.DMatrix(P, feature_types=TYPES, enable_categorical=True)
    leaf = ebst.predict(d, pred_leaf=True)
    assert np.array_equal(leaf, R.leaf_index(trees, P))
    margin = ebst.predict(d, output_margin=True)
    assert np.max(np.abs(margin - obst.predict_margin(P)[:, 0])) <= 1e-5
    sub = P[-400:]
    ds = eng.DMatrix(sub, feature_types=TYPES, enable_categorical=True)
    phi = ebst.predict(ds, pred_contribs=True)
    ref = R.shap_contribs(trees, sub, base_value=0.0)[:, 0]
    tol = 1e-5 * np.maximum(1.0, np.abs(margin[-400:]))[:, None]
    assert np.all(np.abs(phi - ref) <= tol), float(np.max(np.abs(phi - ref)))
    f = str(tmp_path / "m.json")
    ebst.save_model(f)
    for other in (eng.Booster(model_file=f), pickle.loads(pickle.dumps(ebst))):
        assert other.predict(d, pred_leaf=True).tobytes() == leaf.tobytes()
        assert other.predict(d, output_margin=True).tobytes() == margin.tobytes()
        assert other.predict(ds, pred_contribs=True).tobytes() == phi.tobytes()
    # refreshing the model on its own training data changes no leaf value and no prediction
    upd = eng.train(dict(params, process_type="update", updater="refresh"),
                    eng.DMatrix(X, label=y, feature_types=TYPES, enable_categorical=True), 4, xgb_model=ebst)
    for tn, to in zip(upd.get_trees(), trees):
        leafs = to["split_feature"] < 0
        assert np.array_equal(tn["value"][leafs].view(np.uint32), to["value"][leafs].view(np.uint32))
        assert np.array_equal(tn["cat_bits"], to["cat_bits"])
    assert upd.predict(d, output_margin=True).tobytes() == margin.tobytes()


# ------------------------------------------------------------------ two GPUs: the feature slots are sharded
@pytest.mark.timeout(600)
def test_two_actors_identical_to_one(eng):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    X, y = card_matrix(nan_frac=0.1, seed=13)
    params = dict(SQ, max_depth=6)
    b = [train(params, RayDMatrix(X, y, feature_types=TYPES, enable_categorical=True), num_boost_round=3,
               ray_params=RayParams(num_actors=k)) for k in (1, 2)]
    assert any(255 in s for f, _, _, s in cat_splits(b[0].get_trees()) if f == COL[256])
    assert b[0].get_dump(dump_format="json", with_stats=True) == b[1].get_dump(dump_format="json", with_stats=True)
