"""Trees of max_depth 15 and 16, and TreeSHAP paths of up to 32 elements (the bias plus 31 features), on the GPU.

Depth 16 is the deepest tree whose leaf indices fit the uint16_t row -> leaf map (2^16 leaves, indices 0-65,535).
Every parity case asserts the shape it exercises: the deepest level is reached and, at depth 16, one tree has more
than 32,768 leaves, so rows carry leaf indices of 2^15 and above.  Trees are compared with the oracle exactly
(topology, splits, default directions, loss_chg) and leaf values within 1e-5.

Device memory: depth 16 keeps 2 x 2^15 x 128 KiB = 8 GiB of level histograms per feature group, so every deep case
uses at most 32 features (one group).  The 2M-row cases take a few seconds of oracle time per tree."""
import json

import numpy as np
import pytest

from tests import dart_reference as DR
from tests import quantile_reference as QR
from tests import shap_reference as SR
from tests.refresh_reference import refresh_model
from tests.test_gpu_parity import LEAF_TOL, assert_same_model, make_data

pytestmark = pytest.mark.gpu

F32 = np.float32
BIG = 2_000_000
N_CAT = 24                       # categories of the categorical column (partition splits)


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def node_depths(t):
    d = np.zeros(len(t["left"]), np.int32)
    for nid in range(1, len(d)):       # a child's id is larger than its parent's
        d[nid] = d[t["parent"][nid]] + 1
    return d


def deep_data(n, f, seed, nan_frac=0.05, cat=True):
    """f - 1 numeric columns with NaNs (plus a categorical last column when cat) and a centred noisy label: with
    min_child_weight 0 nearly every node splits down to max_depth"""
    X = make_data(n, f, seed, "uniform", nan_frac=nan_frac)
    rng = np.random.RandomState(seed + 1)
    Z = np.nan_to_num(X, nan=5.0)
    y = Z[:, :8].sum(axis=1) + np.sin(Z[:, 0] * 2) * 3 + rng.normal(scale=2.0, size=n)
    if cat:
        c = rng.randint(0, N_CAT, size=n)
        X[:, f - 1] = c
        y += (c % 3 == 0) * 2.0 + (c % 5 < 2) * 1.5
    return X, (y - y.mean()).astype(F32)


def types_of(f, cat):
    return ["q"] * (f - 1) + ["c"] if cat else None


def assert_deep_shape(bst, depth, min_leaves=None):
    """the deepest level is reached and one tree has more than min_leaves (default 2^(depth-1)) leaves, so leaf
    indices past it occur"""
    trees = bst.get_trees()
    assert max(int(node_depths(t).max()) for t in trees) == depth
    most = max(int((t["split_feature"] < 0).sum()) for t in trees)
    assert most > (min_leaves or 1 << (depth - 1)), most


def assert_margins(eng, bst, dm, K):
    """train margin == predict == base + the sum of the leaf values each row reaches (pred_leaf)"""
    train_m = np.asarray(bst.predict(dm, output_margin=True, training=True)).reshape(-1, K)
    pred_m = np.asarray(bst.predict(dm, output_margin=True)).reshape(-1, K)
    assert np.max(np.abs(train_m - pred_m)) <= LEAF_TOL
    leaf = np.asarray(bst.predict(dm, pred_leaf=True)).reshape(pred_m.shape[0], -1).astype(np.int64)
    trees = bst.get_trees()
    s = np.zeros(pred_m.shape, np.float64)
    for i, t in enumerate(trees):
        s[:, i % K] += t["value"][leaf[:, i]]
    base = pred_m - s
    assert np.max(np.abs(base - base[0])) <= LEAF_TOL      # one base margin for every row
    return pred_m


# ------------------------------------------------------------------ gbtree at depth 15 and 16 against the oracle
DEEP_CASES = [
    (15, "reg:squarederror", {}),
    (16, "reg:squarederror", {}),
    (16, "binary:logistic", {}),
    (16, "multi:softprob", {"num_class": 3}),
    (16, "reg:squarederror", {"colsample_bynode": 0.6, "seed": 5, "feature_weights": True}),
]


@pytest.mark.timeout(900)
@pytest.mark.parametrize("depth,objective,extra", DEEP_CASES)
def test_deep_trees_identical(eng, oracle, depth, objective, extra):
    f = 20
    X, y = deep_data(BIG, f, 3 + depth)
    if objective == "binary:logistic":
        y = (y > np.median(y)).astype(F32)
    elif objective == "multi:softprob":
        y = np.digitize(y, np.quantile(y, [1 / 3, 2 / 3])).astype(F32)
    w = np.random.RandomState(depth).uniform(0.5, 2.0, BIG).astype(F32)
    extra = dict(extra)
    fw = None
    if extra.pop("feature_weights", False):
        fw = np.linspace(0.2, 2.0, f).astype(F32)
    params = dict({"objective": objective, "max_depth": depth, "eta": 0.3, "base_score": 0.5, "min_child_weight": 0.0},
                  **extra)
    K = int(params.get("num_class", 1))
    is_cat = [0] * (f - 1) + [1]
    obst, _ = oracle.train(params, X, y, 2, weight=w, is_cat=is_cat, feature_weights=fw)
    dm = eng.DMatrix(X, label=y, weight=w, feature_types=types_of(f, True), enable_categorical=True)
    if fw is not None:
        dm.set_info(feature_weights=fw)
    bst = eng.train(params, dm, num_boost_round=2, verbose_eval=False)
    assert bst.num_trees() == 2 * K
    assert_same_model(bst, obst)
    assert_deep_shape(bst, depth)
    assert any(t["split_type"].any() for t in bst.get_trees())        # categorical splits in the deep trees
    m = assert_margins(eng, bst, dm, K)
    assert np.max(np.abs(m - obst.margin.reshape(-1, K))) <= LEAF_TOL


# ------------------------------------------------------------------ the other tree kinds at depth 16
def test_dart_depth16(eng, oracle):
    X, y = deep_data(400_000, 16, 31, cat=False)
    params = {"booster": "dart", "objective": "reg:squarederror", "max_depth": 16, "rate_drop": 0.3, "seed": 3,
              "base_score": 0.5, "min_child_weight": 0}
    bst = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=4, verbose_eval=False)
    ref = DR.train(oracle, params, X, y, 4)
    assert_same_model(bst, ref)
    assert bst.get_tree_weights().tobytes() == ref.weights.tobytes()
    assert_deep_shape(bst, 16)


def quantile_depth16(eng, oracle, weighted):
    X, y = deep_data(400_000, 16, 37, cat=False)
    params = {"objective": "reg:quantileerror", "quantile_alpha": [0.3, 0.7], "max_depth": 16, "min_child_weight": 0}
    w = np.random.RandomState(38).randint(0, 4, size=len(y)).astype(F32) if weighted else None
    bst = eng.train(params, eng.DMatrix(X, label=y, weight=w), num_boost_round=2, verbose_eval=False)
    ref = QR.train(oracle, params, X, y, 2, weight=w)
    assert_same_model(bst, ref)
    for i, t in enumerate(bst.get_trees()):
        leaf = t["split_feature"] < 0
        assert t["value"][leaf].tobytes() == ref.tree(i).value[leaf].tobytes(), "tree %d leaf values" % i
    assert_deep_shape(bst, 16, min_leaves=1 << 14)     # pinball gradients stop more nodes early


def test_quantile_depth16(eng, oracle):
    quantile_depth16(eng, oracle, False)


@pytest.mark.timeout(900)
def test_quantile_depth16_weighted(eng, oracle):
    """integer weights 0-3: rows of hessian 0 are skipped, the others count by fixed-point mass in the global-memory
    histograms of the weighted count pass"""
    quantile_depth16(eng, oracle, True)


def test_refresh_depth16_is_identity(eng):
    """self-refresh of a depth-16 model keeps every leaf value and prediction bit for bit"""
    X, y = deep_data(BIG, 16, 41, cat=False)
    params = {"objective": "reg:squarederror", "max_depth": 16, "eta": 0.3, "base_score": 0.5, "min_child_weight": 0}
    dm = eng.DMatrix(X, label=y)
    bst = eng.train(params, dm, 2, verbose_eval=False)
    assert_deep_shape(bst, 16)
    new = eng.train(dict(params, process_type="update", updater="refresh"), eng.DMatrix(X, label=y), 2, xgb_model=bst)
    for tn, to in zip(new.get_trees(), bst.get_trees()):
        assert np.array_equal(tn["left"], to["left"]) and np.array_equal(tn["split_feature"], to["split_feature"])
        leaf = to["split_feature"] < 0
        assert np.array_equal(tn["value"][leaf].view(np.uint32), to["value"][leaf].view(np.uint32))
    assert np.array_equal(new.predict(dm, output_margin=True).view(np.uint32),
                          bst.predict(dm, output_margin=True).view(np.uint32))


def full_tree_model(depth, n_features, seed):
    """an xgboost JSON model of one complete tree of the given depth (2^depth leaves)"""
    rng = np.random.RandomState(seed)
    n = (1 << (depth + 1)) - 1
    inner = np.arange(n) < (1 << depth) - 1
    left = np.where(inner, 2 * np.arange(n) + 1, -1).tolist()
    right = np.where(inner, 2 * np.arange(n) + 2, -1).tolist()
    parent = [2147483647] + [(i - 1) // 2 for i in range(1, n)]
    feat = np.where(inner, rng.randint(n_features, size=n), 0).tolist()
    cond = np.where(inner, rng.uniform(-1, 1, size=n), rng.normal(0, 0.1, size=n)).astype(F32).tolist()
    tree = {"base_weights": [0.0] * n, "categories": [], "categories_nodes": [], "categories_segments": [],
            "categories_sizes": [], "default_left": rng.randint(2, size=n).tolist(), "id": 0, "left_children": left,
            "loss_changes": [0.0] * n, "parents": parent, "right_children": right, "split_conditions": cond,
            "split_indices": feat, "split_type": [0] * n, "sum_hessian": [1.0] * n,
            "tree_param": {"num_deleted": "0", "num_feature": str(n_features), "num_nodes": str(n),
                           "size_leaf_vector": "1"}}
    return model_json([tree], n_features)


def model_json(trees, n_features, base_score="0.25"):
    for i, t in enumerate(trees):
        t["id"] = i
    return {"learner": {"attributes": {}, "feature_names": [], "feature_types": [],
                        "gradient_booster": {"model": {"gbtree_model_param": {"num_parallel_tree": "1",
                                                                              "num_trees": str(len(trees))},
                                                       "iteration_indptr": list(range(len(trees) + 1)),
                                                       "tree_info": [0] * len(trees), "trees": trees},
                                             "name": "gbtree"},
                        "learner_model_param": {"base_score": base_score, "boost_from_average": "1", "num_class": "0",
                                                "num_feature": str(n_features), "num_target": "1"},
                        "objective": {"name": "reg:squarederror", "reg_loss_param": {"scale_pos_weight": "1"}}},
            "version": [2, 0, 3]}


def test_refresh_full_depth16_tree_of_65536_leaves(eng, tmp_path):
    """2^16 leaves: the largest compact leaf index, 65,535, is a real leaf; the refreshed tree equals the reference"""
    path = tmp_path / "full16.json"
    path.write_text(json.dumps(full_tree_model(16, 8, 2)))
    src = eng.Booster(model_file=str(path))
    assert int((src.get_trees()[0]["split_feature"] < 0).sum()) == 65536
    rng = np.random.RandomState(3)
    n = 600_000
    X = rng.uniform(-1.2, 1.2, (n, 8)).astype(F32)
    X[rng.rand(n) < 0.05, 2] = np.nan
    y = rng.normal(0, 1, n).astype(F32)

    def grad(margin):
        return (margin.reshape(-1) - y).astype(F32).reshape(-1, 1), np.ones((n, 1), F32)

    new = eng.train({"process_type": "update", "updater": "refresh", "eta": 0.5}, eng.DMatrix(X, label=y), 1,
                    xgb_model=str(path))
    ref, _ = refresh_model(src.get_trees(), X, {"eta": 0.5}, 1, 1, np.full(n, 0.25, F32), grad)
    tn, tr = new.get_trees()[0], ref[0]
    assert np.array_equal(tn["left"], tr["left"])
    assert np.allclose(tn["value"], tr["value"], atol=1e-5, rtol=0)
    leaf = np.asarray(new.predict(eng.DMatrix(X), pred_leaf=True)).reshape(-1).astype(np.int64)
    assert leaf.max() == len(tn["left"]) - 1      # rows reach the last leaf: compact index 65,535


def test_interaction_constraints_depth16(eng, oracle):
    """disjoint sets: the root picks a feature of set A (y depends on A), so the tree is the oracle's on the matrix
    whose set-B columns are constant"""
    X, y = deep_data(1_000_000, 16, 43, cat=False)
    params = {"objective": "reg:squarederror", "max_depth": 16, "eta": 0.3, "base_score": 0.5, "min_child_weight": 0}
    bst = eng.train(dict(params, interaction_constraints=[list(range(8)), list(range(8, 16))]),
                    eng.DMatrix(X, label=y), 1, verbose_eval=False)
    Xa = X.copy()
    Xa[:, 8:] = 0.0
    obst, _ = oracle.train(params, Xa, y, 1)
    assert_same_model(bst, obst)
    assert bst.get_trees()[0]["split_feature"].max() < 8
    assert_deep_shape(bst, 16)


def test_vector_leaf_depth16_doubles_the_scalar_tree(eng, oracle):
    """T = 2 with Y = [y, y]: the scalar tree (itself the oracle's), loss_chg doubled, leaf vectors (v, v)"""
    X, y = deep_data(1_000_000, 16, 47, cat=False)
    params = {"objective": "reg:squarederror", "max_depth": 16, "eta": 0.3, "base_score": 0.5, "min_child_weight": 0,
              "gamma": 0}
    ref = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=2, verbose_eval=False)
    obst, _ = oracle.train(params, X, y, 2)
    assert_same_model(ref, obst)
    assert_deep_shape(ref, 16)
    d2 = eng.DMatrix(X, label=np.stack([y, y], 1), multi_target=True)
    vec = eng.train(dict(params, multi_strategy="multi_output_tree"), d2, num_boost_round=2, verbose_eval=False)
    for tv, tr in zip(vec.get_trees(), ref.get_trees()):
        for k in ("left", "right", "split_feature", "split_bin", "default_left"):
            assert np.array_equal(tv[k], tr[k]), k
        internal = tr["split_feature"] >= 0
        assert np.array_equal(tv["loss_chg"][internal], F32(2) * tr["loss_chg"][internal])
        for k in range(2):
            assert np.array_equal(tv["leaf_vector"][~internal, k], tr["value"][~internal])
    m = vec.predict(d2, output_margin=True)
    r = ref.predict(eng.DMatrix(X), output_margin=True)
    assert np.array_equal(m[:, 0], r) and np.array_equal(m[:, 1], r)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_two_gpus_depth16(eng, oracle, exchange, monkeypatch):
    if eng.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    monkeypatch.setenv("B2_EXCHANGE", exchange)
    X, y = deep_data(BIG, 20, 53)
    params = {"objective": "reg:squarederror", "max_depth": 16, "eta": 0.3, "base_score": 0.5, "min_child_weight": 0}
    types = types_of(20, True)
    b2 = train(params, RayDMatrix(X, y, feature_types=types, enable_categorical=True), num_boost_round=2,
               ray_params=RayParams(num_actors=2))
    obst, _ = oracle.train(params, X, y, 2, is_cat=[0] * 19 + [1])
    assert_same_model(b2, obst)
    assert_deep_shape(b2, 16)


# ------------------------------------------------------------------ TreeSHAP
def path_lengths(t):
    """distinct features on the root -> leaf path of every leaf"""
    out = []

    def walk(nid, feats):
        f = int(t["split_feature"][nid])
        if f < 0:
            out.append(len(feats))
            return
        walk(int(t["left"][nid]), feats | {f})
        walk(int(t["right"][nid]), feats | {f})
    walk(0, frozenset())
    return np.array(out)


def assert_contribs(eng, bst, X, base_value, K=1, kw=None):
    d = eng.DMatrix(X, **(kw or {}))
    phi = bst.predict(d, pred_contribs=True, strict_shape=True)
    ref = SR.shap_contribs(bst.get_trees(), X, num_class=K, base_value=base_value)
    margin = np.asarray(bst.predict(d, output_margin=True)).reshape(len(X), K)
    tol = 1e-5 * np.maximum(1.0, np.abs(margin))[:, :, None]
    assert np.all(np.abs(phi - ref) <= tol), float(np.max(np.abs(phi - ref)))
    assert np.all(np.abs(phi.astype(np.float64).sum(axis=2) - margin) <= tol[:, :, 0])
    again = bst.predict(d, pred_contribs=True, strict_shape=True)
    assert again.tobytes() == phi.tobytes()
    return phi


def shap_case(n, f, seed, binary):
    """every feature matters a little.  binary: 0/1 features (and NaN), which a path can split only once each, so
    a leaf at depth 16 lies below 16 distinct features"""
    rng = np.random.RandomState(seed)
    X = (rng.randint(0, 2, size=(n, f)) if binary else rng.uniform(0, 10, size=(n, f))).astype(F32)
    X[rng.uniform(size=X.shape) < 0.03] = np.nan
    Z = np.nan_to_num(X, nan=0.5 if binary else 5.0)
    y = (Z > (0.5 if binary else 5.0)).astype(np.float64) @ (1.0 + 0.05 * np.arange(f)) + rng.normal(scale=0.5, size=n)
    return X, (y - y.mean()).astype(F32)


def test_contribs_depth16_model(eng):
    X, y = shap_case(12000, 24, 61, binary=True)
    bst = eng.train({"objective": "reg:squarederror", "max_depth": 16, "eta": 0.3, "base_score": 0.5,
                     "min_child_weight": 0}, eng.DMatrix(X, label=y), num_boost_round=2, verbose_eval=False)
    trees = bst.get_trees()
    assert max(int(node_depths(t).max()) for t in trees) == 16
    lens = np.concatenate([path_lengths(t) for t in trees])
    assert lens.max() >= 16 and (lens <= 15).any()          # full-warp and half-warp paths in one model
    assert_contribs(eng, bst, X[:100], 0.5)


def test_interactions_depth16_small_f(eng):
    X, y = shap_case(6000, 6, 67, binary=False)
    bst = eng.train({"objective": "reg:squarederror", "max_depth": 16, "eta": 0.3, "base_score": 0.5,
                     "min_child_weight": 0}, eng.DMatrix(X, label=y), num_boost_round=1, verbose_eval=False)
    assert int(node_depths(bst.get_trees()[0]).max()) == 16
    xs = X[:20]
    d = eng.DMatrix(xs)
    inter = bst.predict(d, pred_interactions=True, strict_shape=True)
    ref = SR.shap_contribs(bst.get_trees(), xs, interactions=True, base_value=0.5)
    margin = np.asarray(bst.predict(d, output_margin=True)).reshape(len(xs), 1)
    tol = 1e-5 * np.maximum(1.0, np.abs(margin))[:, :, None, None]
    assert np.all(np.abs(inter - ref) <= tol), float(np.max(np.abs(inter - ref)))


def test_contribs_local_accuracy_big_depth16(eng):
    X, y = deep_data(BIG, 20, 71)
    dm = eng.DMatrix(X, label=y, feature_types=types_of(20, True), enable_categorical=True)
    bst = eng.train({"objective": "reg:squarederror", "max_depth": 16, "eta": 0.3, "base_score": 0.5,
                     "min_child_weight": 0}, dm, num_boost_round=2, verbose_eval=False)
    assert_deep_shape(bst, 16)
    xs = X[:20000]
    d = eng.DMatrix(xs, feature_types=types_of(20, True), enable_categorical=True)
    phi = bst.predict(d, pred_contribs=True)
    margin = bst.predict(d, output_margin=True)
    assert np.max(np.abs(phi.astype(np.float64).sum(axis=1) - margin)) <= 1e-5 * max(1.0, float(np.abs(margin).max()))
    assert bst.predict(d, pred_contribs=True).tobytes() == phi.tobytes()


def chain_tree(n_features, chain, seed, sides):
    """a chain of `chain` splits on distinct features 0, 1, ...; at chain node i the chain continues on side
    sides[i] (0 left) and the other child is a leaf; the last chain node has two leaves.  The deepest leaves lie
    below `chain` distinct features."""
    rng = np.random.RandomState(seed)
    left, right, parent, feat, cond, dl, hess = [], [], [], [], [], [], []

    def node(p):
        left.append(-1); right.append(-1); parent.append(p); feat.append(0); cond.append(float(rng.normal(0, 1)))
        dl.append(int(rng.randint(2))); hess.append(0.0)
        return len(left) - 1

    nid = node(2147483647)
    for i in range(chain):
        a, b = node(nid), node(nid)
        left[nid], right[nid] = a, b
        feat[nid] = i % n_features
        cond[nid] = float(rng.uniform(2, 8))
        nid = a if sides[i] == 0 else b
    n = len(left)
    for i in reversed(range(n)):                    # covers: leaves random, splits the sum of their children
        hess[i] = float(rng.uniform(1, 10)) if left[i] < 0 else hess[left[i]] + hess[right[i]]
    return {"base_weights": [0.0] * n, "categories": [], "categories_nodes": [], "categories_segments": [],
            "categories_sizes": [], "default_left": dl, "id": 0, "left_children": left, "loss_changes": [0.0] * n,
            "parents": parent, "right_children": right, "split_conditions": cond,
            "split_indices": [feat[i] if left[i] >= 0 else 0 for i in range(n)], "split_type": [0] * n,
            "sum_hessian": hess,
            "tree_param": {"num_deleted": "0", "num_feature": str(n_features), "num_nodes": str(n),
                           "size_leaf_vector": "1"}}


def test_contribs_long_paths_from_json(eng, tmp_path):
    """short trees, a chain whose deepest leaves are below 31 distinct features, and chains of 16 and 20: paths of 2
    to 32 elements in mixed order"""
    F = 40
    rng = np.random.RandomState(7)
    trees = [chain_tree(F, 3, 1, [0, 1, 0]), chain_tree(F, 31, 2, rng.randint(2, size=31)),
             chain_tree(F, 16, 3, [1] * 16), chain_tree(F, 20, 4, rng.randint(2, size=20)), chain_tree(F, 5, 5, [1] * 5)]
    path = tmp_path / "long.json"
    path.write_text(json.dumps(model_json(trees, F)))
    bst = eng.Booster(model_file=str(path))
    lens = np.concatenate([path_lengths(t) for t in bst.get_trees()])
    assert lens.max() == 31 and (lens <= 15).any()
    X = rng.uniform(0, 10, size=(500, F)).astype(F32)
    X[rng.uniform(size=X.shape) < 0.1] = np.nan
    X[:100, :31] = 5.0 + rng.uniform(-0.01, 0.01, size=(100, 31)).astype(F32)   # rows that walk deep into the chains
    phi = assert_contribs(eng, bst, X, 0.25)
    xs = X[:40]
    d = eng.DMatrix(xs)
    inter = bst.predict(d, pred_interactions=True, strict_shape=True)
    ref = SR.shap_contribs(bst.get_trees(), xs, interactions=True, base_value=0.25)
    margin = np.asarray(bst.predict(d, output_margin=True)).reshape(len(xs), 1)
    tol = 1e-5 * np.maximum(1.0, np.abs(margin))[:, :, None, None]
    assert np.all(np.abs(inter - ref) <= tol), float(np.max(np.abs(inter - ref)))
    assert bst.predict(d, pred_interactions=True, strict_shape=True).tobytes() == inter.tobytes()
    # a path's values do not depend on its neighbours: the chain alone gives the same bits as inside the model
    alone = tmp_path / "alone.json"
    alone.write_text(json.dumps(model_json([trees[1]], F, base_score="0")))
    b1 = eng.Booster(model_file=str(alone))
    full = bst.predict(eng.DMatrix(X), pred_contribs=True, iteration_range=(1, 2))
    assert b1.predict(eng.DMatrix(X), pred_contribs=True)[:, :F].tobytes() == full[:, :F].tobytes()
    assert np.abs(phi).max() > 0


def test_path_of_32_features_refused(eng, tmp_path):
    F = 40
    path = tmp_path / "too_long.json"
    path.write_text(json.dumps(model_json([chain_tree(F, 32, 9, [0] * 32)], F)))
    bst = eng.Booster(model_file=str(path))
    X = np.random.RandomState(1).uniform(0, 10, size=(10, F)).astype(F32)
    with pytest.raises(eng.XGBoostError, match="at most 31 distinct features"):
        bst.predict(eng.DMatrix(X), pred_contribs=True)
    assert bst.predict(eng.DMatrix(X)).shape == (10,)      # plain prediction still works


# ------------------------------------------------------------------ refusals
def test_max_depth_17_refused(eng):
    X, y = deep_data(1000, 8, 1, cat=False)
    with pytest.raises(eng.XGBoostError, match=r"max_depth must be in \[1, 16\], got 17"):
        eng.train({"max_depth": 17}, eng.DMatrix(X, label=y), 1)


def test_wide_depth16_refused_by_the_memory_check(eng):
    X = np.random.RandomState(2).uniform(0, 10, size=(2000, 4300)).astype(F32)
    y = X[:, 0].copy()
    dm = eng.DMatrix(X, label=y)
    with pytest.raises(eng.XGBoostError, match=r"max_depth 16 with 135 feature groups needs [0-9.]+ GiB of level "
                                               r"histograms, and [0-9.]+ GiB of device memory is free"):
        eng.train({"max_depth": 16}, dm, 1)
    bst = eng.train({"max_depth": 6}, dm, 1)      # the same matrix trains at a depth that fits
    assert bst.num_trees() == 1
