"""interaction_constraints on the GPU.

Parity: when a tree's root splits on a feature of set S and the sets are disjoint, every node below may only use the
features of S.  Such a tree is then exactly the oracle's tree on the same matrix with every feature outside S made
constant (a constant column has one bin and never splits; the other columns keep their cuts, bins and gradients).  The
data below makes the root pick a feature of S, the tests check that it did, and then compare the GPU model with that
oracle model: split feature, bin, condition, default direction and topology bit-identical, leaves within 1e-5.  Shapes
that do not reduce to one feature mask (overlapping sets, features in no set) are checked node by node against the
rule as stated and compared with tests/interaction_reference.py, the oracle's growth restated with the rule written
out literally (checked against the oracle itself without constraints in tests/test_interaction_constraints.py)."""
import json

import numpy as np
import pytest

from tests.test_gpu_parity import assert_same_model, make_data
from tests import interaction_reference as R
from tests.test_interaction_constraints import rule_violations

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def masked(X, keep):
    Xm = X.copy()
    drop = np.ones(X.shape[1], bool)
    drop[list(keep)] = False
    Xm[:, drop] = 0.0
    return Xm


def assert_obeys(bst, sets, n_features):
    for i, t in enumerate(bst.get_trees()):
        assert rule_violations(t, sets, n_features) == [], "tree %d" % i


def roots_in(bst, feats):
    roots = [int(t["split_feature"][0]) for t in bst.get_trees()]
    assert all(r in feats for r in roots if r >= 0), roots


def signal(X, feats, rng):
    """y driven by the features `feats` (products, so that a path wants several of them) plus a little noise."""
    Z = np.nan_to_num(X[:, feats], nan=5.0)
    y = Z.sum(axis=1) * 0.3 + np.prod(Z[:, :2] - 5.0, axis=1) * 0.2 + rng.normal(scale=0.3, size=X.shape[0])
    return y.astype(np.float32)


OBJECTIVES = ["reg:squarederror", "binary:logistic", "multi:softprob"]


def labels(objective, y):
    if objective == "binary:logistic":
        return (y > np.median(y)).astype(np.float32)
    if objective == "multi:softprob":
        return np.digitize(y, np.quantile(y, [1 / 3, 2 / 3])).astype(np.float32)
    return y


@pytest.mark.parametrize("objective", OBJECTIVES)
@pytest.mark.parametrize("depth", [3, 8])
@pytest.mark.parametrize("sets,signal_feats", [
    ([[0, 1, 2, 3, 4], [5, 6, 7, 8, 9, 10, 11]], [0, 1, 2, 3]),          # disjoint sets
    ([[2, 3, 4], [6, 7], [9, 10, 11, 12, 13]], [2, 3, 4]),               # features 0, 1, 5, 8, 14.. in no set
    ([[3], [7], [9], [0, 1, 2]], [0, 1, 2]),                             # singletons next to a real set
])
def test_parity_with_masked_oracle(eng, oracle, objective, depth, sets, signal_feats):
    n, f = 40000, 20
    rng = np.random.RandomState(depth * 7 + len(sets))
    X = make_data(n, f, 100 + depth, "uniform", nan_frac=0.05)
    y = labels(objective, signal(X, signal_feats, rng))
    w = rng.uniform(0.5, 2.0, size=n).astype(np.float32)
    params = {"objective": objective, "max_depth": depth, "eta": 0.3, "base_score": 0.5}
    if objective == "multi:softprob":
        params["num_class"] = 3
    keep = next(s for s in sets if set(signal_feats) <= set(s))
    ebst = eng.train(dict(params, interaction_constraints=sets), eng.DMatrix(X, label=y, weight=w), num_boost_round=6,
                     verbose_eval=False)
    roots_in(ebst, keep)
    assert_obeys(ebst, sets, f)
    obst, _ = oracle.train(params, masked(X, keep), y, 6, weight=w)
    assert_same_model(ebst, obst)


def test_num_parallel_tree_equals_masked_matrix(eng):
    """num_parallel_tree > 1 grows its trees with direct launches; the oracle grows one tree per round, so the
    reference here is the engine itself, unconstrained, on the masked matrix"""
    n, f = 30000, 16
    rng = np.random.RandomState(3)
    X = make_data(n, f, 31, "uniform", nan_frac=0.05)
    y = signal(X, [4, 5, 6], rng)
    sets = [[4, 5, 6, 7], [0, 1, 2, 3], [8, 9, 10, 11, 12, 13, 14, 15]]
    params = {"objective": "reg:squarederror", "max_depth": 6, "num_parallel_tree": 3, "subsample": 0.8,
              "colsample_bynode": 0.8, "base_score": 0.5}
    ebst = eng.train(dict(params, interaction_constraints=sets), eng.DMatrix(X, label=y), num_boost_round=3,
                     verbose_eval=False)
    roots_in(ebst, sets[0])
    assert_obeys(ebst, sets, f)
    ref = eng.train(params, eng.DMatrix(masked(X, sets[0]), label=y), num_boost_round=3, verbose_eval=False)
    for a, b in zip(ebst.get_trees(), ref.get_trees()):
        for k in ("left", "right", "split_feature", "split_bin", "default_left", "value"):
            assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("depth", [3, 8])
@pytest.mark.parametrize("sets", [[[0, 1], [1, 2]], [[0, 1, 2, 3], [2, 3, 4, 5], [5, 6, 7]], [[0, 5], [5, 9], [9, 0]],
                                  [[0, 1], [3, 4], [4, 7]], [[2], [5], [0, 1, 6]]])
def test_every_shape_against_the_reference(eng, sets, depth):
    """overlapping sets, features in no set, singletons: the model equals the CPU reference growth of
    tests/interaction_reference.py (the oracle's growth with the rule written out), whatever sets the roots pick"""
    n, f = 20000, 12
    rng = np.random.RandomState(4 + depth)
    X = make_data(n, f, 41, "uniform", nan_frac=0.05)
    y = signal(X, sorted({v for s in sets for v in s}), rng) + np.nan_to_num(X[:, 11], nan=5.0) * 0.05   # 11: no set
    w = rng.uniform(0.5, 2.0, size=n).astype(np.float32)
    params = {"objective": "reg:squarederror", "max_depth": depth, "base_score": 0.5}
    bst = eng.train(dict(params, interaction_constraints=sets), eng.DMatrix(X, label=y, weight=w), num_boost_round=6,
                    verbose_eval=False)
    assert_obeys(bst, sets, f)
    assert max(len(t["left"]) for t in bst.get_trees()) > 7     # real paths, not stumps
    assert_same_model(bst, R.train(params, X, y, 6, sets=sets, weight=w))


def test_overlapping_sets_allow_the_union(eng):
    """root on 1 with [[0, 1], [1, 2]]: below it 0 on one path and 2 on the other (the union of both sets), and the
    model equals the reference"""
    n, f = 20000, 4
    rng = np.random.RandomState(5)
    X = rng.uniform(0, 10, size=(n, f)).astype(np.float32)
    y = (10 * (X[:, 1] > 5) + np.where(X[:, 1] > 5, X[:, 0], X[:, 2]) + rng.normal(scale=0.1, size=n)).astype(np.float32)
    sets = [[0, 1], [1, 2]]
    params = {"objective": "reg:squarederror", "max_depth": 3, "base_score": 0.5}
    bst = eng.train(dict(params, interaction_constraints=sets), eng.DMatrix(X, label=y), num_boost_round=3,
                    verbose_eval=False)
    t = bst.get_trees()[0]
    assert t["split_feature"][0] == 1
    assert {int(t["split_feature"][t["left"][0]]), int(t["split_feature"][t["right"][0]])} == {0, 2}
    assert_same_model(bst, R.train(params, X, y, 3, sets=sets))


def test_root_on_a_feature_in_no_set_gives_a_stump(eng, oracle):
    n, f = 20000, 8
    rng = np.random.RandomState(5)
    X = make_data(n, f, 51, "uniform")
    y = ((X[:, 7] > 5) * 10.0 + X[:, 0] * X[:, 1] * 0.05 + rng.normal(scale=0.1, size=n)).astype(np.float32)
    params = {"objective": "reg:squarederror", "max_depth": 6, "base_score": 0.5}
    ebst = eng.train(dict(params, interaction_constraints=[[0, 1], [2, 3]]), eng.DMatrix(X, label=y),
                     num_boost_round=1, verbose_eval=False)
    t = ebst.get_trees()[0]
    assert int(t["split_feature"][0]) == 7 and len(t["left"]) == 3
    obst, _ = oracle.train(dict(params, max_depth=1), X, y, 1)
    assert_same_model(ebst, obst)


def test_liveness_constraint_changes_the_tree(eng):
    """y = x0 x1 + x2 x3: unconstrained trees mix the two pairs on one path, [[0, 1], [2, 3]] never does, and the
    constrained model equals the reference"""
    n, f = 40000, 4
    X = make_data(n, f, 61, "uniform")
    y = (X[:, 0] * X[:, 1] + X[:, 2] * X[:, 3]).astype(np.float32)
    params = {"objective": "reg:squarederror", "max_depth": 4, "base_score": 0.5}
    sets = [[0, 1], [2, 3]]
    free = eng.train(params, eng.DMatrix(X, label=y), num_boost_round=4, verbose_eval=False)
    assert any(rule_violations(t, sets, f) for t in free.get_trees())
    bst = eng.train(dict(params, interaction_constraints=sets), eng.DMatrix(X, label=y), num_boost_round=4,
                    verbose_eval=False)
    assert_obeys(bst, sets, f)
    assert_same_model(bst, R.train(params, X, y, 4, sets=sets))


def test_categorical_inside_and_outside_the_sets(eng, oracle):
    """one-hot (3 categories) and partition (20, 200 categories) splits, categorical features in and out of the set;
    feature 3 dominates, so that every root stays in its set"""
    rng = np.random.RandomState(7)
    n = 40000
    Xn = rng.uniform(0, 10, size=(n, 3))
    X = np.column_stack([Xn, rng.randint(0, 3, size=n), rng.randint(0, 20, size=n), rng.randint(0, 200, size=n)]).astype(np.float32)
    X[rng.uniform(size=X.shape) < 0.03] = np.nan
    y = ((X[:, 3] == 2) * 8.0 + (X[:, 4] % 3 == 0) * 1.5 + (Xn[:, 0] > 5) * 0.5 + (X[:, 5] % 7 < 2) * 0.5 +
         rng.normal(scale=0.1, size=n)).astype(np.float32)
    types, is_cat = ["q", "q", "q", "c", "c", "c"], [0, 0, 0, 1, 1, 1]
    sets = [[0, 3, 4], [1, 2, 5]]
    params = {"objective": "reg:squarederror", "max_depth": 5, "base_score": 0.5, "max_cat_to_onehot": 4}
    dm = eng.DMatrix(X, label=y, feature_types=types, enable_categorical=True)
    ebst = eng.train(dict(params, interaction_constraints=sets), dm, num_boost_round=4, verbose_eval=False)
    roots_in(ebst, sets[0])
    assert_obeys(ebst, sets, 6)
    kinds = {(int(t["split_feature"][i]), int(t["split_type"][i])) for t in ebst.get_trees() for i in range(len(t["left"]))}
    assert (3, 1) in kinds and (4, 1) in kinds          # categorical splits on both kinds of feature of the set
    obst, _ = oracle.train(params, masked(X, sets[0]), y, 4, is_cat=is_cat)
    assert_same_model(ebst, obst)


@pytest.mark.parametrize("extra", [{"colsample_bytree": 0.7}, {"colsample_bylevel": 0.6}, {"colsample_bynode": 0.5},
                                   {"colsample_bytree": 0.8, "colsample_bylevel": 0.8, "colsample_bynode": 0.7}])
def test_column_sampling_with_feature_weights(eng, oracle, extra):
    n, f = 30000, 24
    rng = np.random.RandomState(8)
    X = make_data(n, f, 81, "uniform", nan_frac=0.03)
    y = signal(X, [0, 1, 2, 3, 4, 5], rng)
    fw = rng.uniform(0.2, 3.0, size=f).astype(np.float32)
    sets = [list(range(0, 10)), list(range(10, 24))]
    params = dict({"objective": "reg:squarederror", "max_depth": 6, "base_score": 0.5, "seed": 3}, **extra)
    dm = eng.DMatrix(X, label=y)
    dm.set_info(feature_weights=fw)
    ebst = eng.train(dict(params, interaction_constraints=sets), dm, num_boost_round=6, verbose_eval=False)
    roots_in(ebst, sets[0])
    assert_obeys(ebst, sets, f)
    obst, _ = oracle.train(params, masked(X, sets[0]), y, 6, feature_weights=fw)
    assert_same_model(ebst, obst)


def test_wide_150_sets(eng, oracle):
    """F = 1000, 150 disjoint sets of 6 features (3 mask words), 100 features in no set; the signal lives in set 140"""
    n, f = 20000, 1000
    rng = np.random.RandomState(9)
    X = rng.uniform(0, 10, size=(n, f)).astype(np.float32)
    sets = [list(range(6 * k, 6 * k + 6)) for k in range(150)]
    y = signal(X, sets[140][:4], rng)
    params = {"objective": "reg:squarederror", "max_depth": 6, "base_score": 0.5}
    ebst = eng.train(dict(params, interaction_constraints=sets), eng.DMatrix(X, label=y), num_boost_round=4,
                     verbose_eval=False)
    roots_in(ebst, sets[140])
    obst, _ = oracle.train(params, masked(X, sets[140]), y, 4)
    assert_same_model(ebst, obst)


def test_depth_14(eng, oracle):
    n, f = 200000, 12
    rng = np.random.RandomState(10)
    X = make_data(n, f, 91, "uniform", nan_frac=0.02)
    y = signal(X, [6, 7, 8], rng)
    sets = [[6, 7, 8, 9, 10, 11], [0, 1, 2, 3, 4, 5]]
    params = {"objective": "reg:squarederror", "max_depth": 14, "base_score": 0.5}
    ebst = eng.train(dict(params, interaction_constraints=sets), eng.DMatrix(X, label=y), num_boost_round=2,
                     verbose_eval=False)
    roots_in(ebst, sets[0])
    def depth(t, nid=0):
        return 0 if t["left"][nid] < 0 else 1 + max(depth(t, t["left"][nid]), depth(t, t["right"][nid]))
    assert max(depth(t) for t in ebst.get_trees()) == 14
    obst, _ = oracle.train(params, masked(X, sets[0]), y, 2)
    assert_same_model(ebst, obst)


def test_one_set_of_every_feature_is_bit_identical_to_none(eng):
    import bench
    X, y = bench.synth_block(0, 1_000_000, 100)
    params = dict(bench.PARAMS)
    dumps = []
    for ic in (None, [list(range(100))], [], "[]"):
        p = dict(params) if ic is None else dict(params, interaction_constraints=ic)
        bst = eng.train(p, eng.DMatrix(X, label=y), num_boost_round=5, verbose_eval=False)
        dumps.append(bst.get_dump(dump_format="json", with_stats=True))
    assert all(d == dumps[0] for d in dumps[1:])


def test_engine_rejects_index_past_the_features(eng):
    X = make_data(100, 5, 1)
    with pytest.raises(eng.XGBoostError, match="outside"):
        eng.train({"interaction_constraints": [[0, 5]]}, eng.DMatrix(X, label=X[:, 0]), num_boost_round=1)


@pytest.mark.parametrize("form", ["string", "list"])
def test_reference_constraint_parameters(form):
    """xgboost_ray's test_sklearn.py test_constraint_parameters: the value comes back from save_config()"""
    from xgboost_ray_b200.sklearn import RayXGBRegressor
    rng = np.random.RandomState(0)
    X, y = rng.randn(10, 10).astype(np.float32), rng.randn(10).astype(np.float32)
    ic = "[[0, 1], [2, 3, 4]]" if form == "string" else [[0, 1], [2, 3, 4]]
    reg = RayXGBRegressor(n_estimators=4, interaction_constraints=ic)
    reg.fit(X, y)
    config = json.loads(reg.get_booster().save_config())
    assert config["learner"]["gradient_booster"]["tree_train_param"]["interaction_constraints"] == "[[0, 1], [2, 3, 4]]"


def test_feature_names_through_a_dataframe_and_actors():
    pd = pytest.importorskip("pandas")
    from xgboost_ray_b200 import RayDMatrix, RayParams, predict, train
    rng = np.random.RandomState(11)
    n = 20000
    df = pd.DataFrame(rng.uniform(0, 10, size=(n, 6)).astype(np.float32), columns=list("abcdef"))
    y = (df["a"] * df["b"] + df["d"] * df["e"]).to_numpy(np.float32)
    ic = [["a", "b", "c"], ["d", "e", "f"]]
    bst = train({"objective": "reg:squarederror", "max_depth": 5, "interaction_constraints": ic}, RayDMatrix(df, y),
                num_boost_round=4, ray_params=RayParams(num_actors=1))
    assert_obeys(bst, [[0, 1, 2], [3, 4, 5]], 6)
    assert json.loads(bst.save_config())["learner"]["gradient_booster"]["tree_train_param"][
        "interaction_constraints"] == "[[0, 1, 2], [3, 4, 5]]"
    p = predict(bst, RayDMatrix(df), ray_params=RayParams(num_actors=1))
    assert p.shape == (n,) and np.all(np.isfinite(p))


def test_shap_interactions_vanish_between_sets(eng):
    n, f = 20000, 8
    rng = np.random.RandomState(12)
    X = make_data(n, f, 121, "uniform", nan_frac=0.02)
    y = signal(X, list(range(f)), rng)
    sets = [[0, 1, 2], [3, 4], [5, 6, 7]]
    bst = eng.train({"objective": "reg:squarederror", "max_depth": 8, "interaction_constraints": sets},
                    eng.DMatrix(X, label=y), num_boost_round=6, verbose_eval=False)
    assert_obeys(bst, sets, f)
    dm = eng.DMatrix(X[:2000])
    inter = bst.predict(dm, pred_interactions=True)
    share = np.zeros((f, f), bool)
    for s in sets:
        share[np.ix_(s, s)] = True
    off = ~share & ~np.eye(f, dtype=bool)
    assert np.all(inter[:, :f, :f][:, off] == 0.0)
    margin = bst.predict(dm, output_margin=True)
    assert np.max(np.abs(inter.sum(axis=(1, 2)) - margin)) <= 1e-3 * max(1.0, np.max(np.abs(margin)))


def test_count_poisson_against_objective_reference():
    """count:poisson, constrained with overlapping sets: the engine's own objective against the reference growth fed
    with the gradients of tests/objective_reference.py (its custom-gradient path, max_delta_step 0.7)"""
    from tests import objective_reference as OR
    from xgboost_ray_b200 import engine as E
    n, f = 20000, 10
    rng = np.random.RandomState(13)
    X = make_data(n, f, 131, "uniform", nan_frac=0.03)
    Z = np.nan_to_num(X, nan=5.0)
    y = rng.poisson(np.exp(0.15 * Z[:, 0] + 0.1 * Z[:, 1] - 0.05 * Z[:, 2] * Z[:, 3] / 10 - 1.0)).astype(np.float32)
    sets = [[0, 1, 2], [2, 3, 4], [5, 6]]
    params = {"objective": "count:poisson", "max_depth": 5, "base_score": 0.5}
    bst = E.train(dict(params, interaction_constraints=sets), E.DMatrix(X, label=y), num_boost_round=4, verbose_eval=False)
    assert_obeys(bst, sets, f)
    tree_params = {"objective": "reg:squarederror", "max_depth": 5, "base_score": OR.base_margin("count:poisson", 0.5),
                   "max_delta_step": OR.max_delta_step(params)}

    def grads(margin):
        g, h, bad = OR.gradients(params, margin, y)
        assert bad == 0
        return g, h

    assert_same_model(bst, R.train(tree_params, X, y, 4, sets=sets, gradients=grads))


def _ngpu():
    from xgboost_ray_b200 import engine
    return engine.device_count()


@pytest.mark.timeout(300)
@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_two_gpus_identical_to_one_and_to_oracle(oracle, exchange, monkeypatch):
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    import xgboost_ray_b200.main as M
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    M.shutdown_actors()
    if exchange == "nccl":
        monkeypatch.setenv("B2_EXCHANGE", "nccl")
    else:
        monkeypatch.delenv("B2_EXCHANGE", raising=False)
    n, f = 60013, 20
    rng = np.random.RandomState(14)
    X = make_data(n, f, 141, "uniform", nan_frac=0.03)
    y = signal(X, [0, 1, 2], rng)
    sets = [[0, 1, 2, 3, 4], [5, 6, 7, 8, 9, 10]]
    params = {"objective": "reg:squarederror", "max_depth": 8, "base_score": 0.5}
    pc = dict(params, interaction_constraints=sets)
    b1 = train(pc, RayDMatrix(X, y), num_boost_round=6, ray_params=RayParams(num_actors=1))
    b2 = train(pc, RayDMatrix(X, y), num_boost_round=6, ray_params=RayParams(num_actors=2))
    d1, d2 = (b.get_dump(dump_format="json", with_stats=True) for b in (b1, b2))
    assert d1 == d2
    roots_in(b2, sets[0])
    obst, _ = oracle.train(params, masked(X, sets[0]), y, 6)
    assert_same_model(b2, obst)
    M.shutdown_actors()
