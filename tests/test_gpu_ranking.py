"""GPU checks of learning to rank: rank:pairwise / rank:ndcg gradients bit-equal to tests/ranking_reference.py (read
back with B2_BoosterGetGradients), trees identical to the oracle grown from them, the ndcg / map / pre metrics, input
errors, save / load / continuation, SHAP, the golden fixtures and the public train / predict with qid on one and two
GPUs."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from tests import ranking_reference as R
from tests.golden.make_golden_ranking import CASES as RANKING_CASES, case_data
from tests.test_gpu_parity import assert_same_model, make_data

pytestmark = pytest.mark.gpu

SIZES = (1, 2, 3, 100, 5000, 40000)


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def get_gradients(eng, bst, n):
    g = np.zeros(n, np.float32)
    h = np.zeros(n, np.float32)
    eng._check(eng.lib().B2_BoosterGetGradients(bst.handle, g.ctypes.data_as(C.POINTER(C.c_float)),
                                                  h.ctypes.data_as(C.POINTER(C.c_float)), n))
    return g, h


def groups(sizes, seed, levels=5):
    """qid of consecutive groups of the given sizes and integer labels 0..levels-1."""
    rng = np.random.RandomState(seed)
    qid = np.repeat(np.arange(len(sizes)), sizes)
    y = rng.randint(0, levels, len(qid)).astype(np.float32)
    return qid, y


def same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize("objective", R.OBJECTIVES)
@pytest.mark.parametrize("k", [1, 5, 32, 10000])
@pytest.mark.parametrize("exp_gain", [True, False])
@pytest.mark.parametrize("margins", ["round0", "base_margin"])
def test_gradients_bit_equal_to_reference(eng, objective, k, exp_gain, margins):
    """Group sizes 1 .. 40000 (the largest is read from global memory, not shared memory), all-tied margins at round 0
    and a base_margin with +-0.0 and repeated values: the gradient pairs equal the reference bit for bit.  With
    k = 10^4 the 40000-row group is left out (4 * 10^8 pairs of one group)."""
    sizes = SIZES if k < 10000 else SIZES[:-1]
    qid, y = groups(sizes, 1)
    n = len(qid)
    X = make_data(n, 3, 2, "uniform")
    rng = np.random.RandomState(k)
    params = {"objective": objective, "lambdarank_num_pair_per_sample": k, "ndcg_exp_gain": exp_gain, "max_depth": 2}
    kw = {}
    if margins == "base_margin":
        m = np.round(rng.normal(size=n), 1).astype(np.float32)        # many repeated values
        m[::7] = 0.0
        m[3::7] = -0.0
        kw["base_margin"] = m
    else:
        m = np.full(n, 0.5, np.float32)                                 # base_score, identity transform
    dm = eng.DMatrix(X, label=y, qid=qid, **kw)
    bst = eng.Booster(params, cache=[dm])
    bst.update(dm, 0)
    g, h = get_gradients(eng, bst, n)
    rg, rh, bad = R.gradients(params, m, y, R.group_ptr(qid))
    assert not bad
    assert same_bits(g, rg), np.nonzero(g != rg)[0][:10]
    assert same_bits(h, rh), np.nonzero(h != rh)[0][:10]


def test_delta_ndcg_on_the_gpu_equals_swap(eng):
    """One 6-row group, k = 6, distinct margins: before normalisation the engine's per-row sums are the reference's;
    the reference's Delta itself is checked against a brute-force swap on the CPU (test_ranking_reference.py)."""
    qid, y = groups((6,), 3)
    X = make_data(6, 2, 4, "uniform")
    m = np.array([0.3, -1.2, 2.0, 0.7, 0.1, -0.4], np.float32)
    params = {"objective": "rank:ndcg", "lambdarank_num_pair_per_sample": 6, "max_depth": 1}
    dm = eng.DMatrix(X, label=y, qid=qid, base_margin=m)
    bst = eng.Booster(params, cache=[dm])
    bst.update(dm, 0)
    g, h = get_gradients(eng, bst, 6)
    rg, rh = R.group_gradients("rank:ndcg", m, y, 6, True)
    assert same_bits(g, rg) and same_bits(h, rh)


@pytest.mark.parametrize("objective", R.OBJECTIVES)
@pytest.mark.parametrize("depth", [3, 6])
def test_trees_identical_to_oracle(eng, oracle, objective, depth):
    sizes = [1, 2, 3, 37, 100] * 12 + [3000]
    qid, y = groups(sizes, 5 + depth)
    n, f = len(qid), 8
    X = make_data(n, f, 31, "uniform", nan_frac=0.1)
    y = np.where(X[:, 0] > 0.3, np.minimum(y + 1, 4), y).astype(np.float32)
    params = {"objective": objective, "max_depth": depth, "eta": 0.3, "lambdarank_num_pair_per_sample": 8}
    obst = R.train(oracle, params, X, y, qid, 4)
    ebst = eng.train(params, eng.DMatrix(X, label=y, qid=qid), num_boost_round=4, verbose_eval=False)
    assert_same_model(ebst, obst)
    Xt = make_data(2000, f, 99, "uniform")
    pe, po = ebst.predict(eng.DMatrix(Xt)), obst.predict(Xt)
    assert np.max(np.abs(pe - po) / np.maximum(1.0, np.abs(po))) <= 1e-5


METRICS = ["ndcg", "ndcg@3", "ndcg-", "ndcg@5-", "ndcg@200", "map", "map@2", "map-", "map@4-", "pre@1", "pre@5",
           "pre@200"]


@pytest.mark.parametrize("exp_gain", [True, False])
def test_metrics_match_reference(eng, exp_gain):
    sizes = [1, 2, 3, 7, 37, 100, 2500] * 3
    qid, y = groups(sizes, 6, levels=3)
    y[:3] = 0.0                                      # groups without any relevant row
    n = len(qid)
    X = make_data(n, 5, 7, "uniform")
    qv, yv = groups([4, 9, 50, 1, 300], 8, levels=4)
    Xv = make_data(len(qv), 5, 8, "uniform")
    params = {"objective": "rank:pairwise", "max_depth": 3, "ndcg_exp_gain": exp_gain, "eval_metric": METRICS}
    dm, dv = eng.DMatrix(X, label=y, qid=qid), eng.DMatrix(Xv, label=yv, qid=qv)
    bst = eng.Booster(params, cache=[dm])
    for r in range(3):
        bst.update(dm, r)
        mt = bst.predict(dm, output_margin=True, training=True)
        mv = bst.predict(dv, output_margin=True)
        for name in METRICS:
            for d, m, yy, q in ((dm, mt, y, qid), (dv, mv, yv, qv)):
                out = C.c_double(0)
                eng._check(eng.lib().B2_BoosterEvalSet(bst.handle, d.handle, name.encode(), C.byref(out)))
                want = R.metric(name, m, yy, R.group_ptr(q), exp_gain)
                assert abs(out.value - want) <= 1e-12 * max(1.0, abs(want)), (r, name, out.value, want)
                again = C.c_double(0)
                eng._check(eng.lib().B2_BoosterEvalSet(bst.handle, d.handle, name.encode(), C.byref(again)))
                assert again.value == out.value                  # deterministic: no atomics on the value
    # the metrics work with any single-output objective, on the prediction order
    b2 = eng.train({"objective": "binary:logistic", "max_depth": 3}, eng.DMatrix(X, label=(y > 0).astype(np.float32),
                                                                                  qid=qid), 2, verbose_eval=False)
    out = C.c_double(0)
    eng._check(eng.lib().B2_BoosterEvalSet(b2.handle, dv.handle, b"ndcg@5", C.byref(out)))
    assert abs(out.value - R.metric("ndcg@5", b2.predict(dv), yv, R.group_ptr(qv))) <= 1e-12


def test_default_metric_base_score_and_early_stopping(eng):
    qid, y = groups([20] * 40, 9)
    X = make_data(len(qid), 6, 10, "uniform")
    y = np.where(X[:, 1] > 0, np.minimum(y + 2, 4), y).astype(np.float32)
    dm = eng.DMatrix(X, label=y, qid=qid)
    for obj, k, want in (("rank:pairwise", None, "ndcg@32"), ("rank:ndcg", 7, "ndcg@7")):
        res = {}
        p = {"objective": obj} if k is None else {"objective": obj, "lambdarank_num_pair_per_sample": k}
        bst = eng.train(p, dm, 2, evals=[(dm, "t")], evals_result=res, verbose_eval=False)
        assert list(res["t"]) == [want]
        assert bst.params["base_score"] == 0.5
        assert np.all(bst.predict(dm, output_margin=True) == bst.predict(dm))      # identity transform
    for metric in ("ndcg@5-", "map", "pre@3"):
        res = {}
        bst = eng.train({"objective": "rank:ndcg", "eval_metric": metric, "max_depth": 3}, dm, 8, evals=[(dm, "t")],
                        evals_result=res, early_stopping_rounds=2, verbose_eval=False)
        vals = res["t"][metric]
        assert bst.best_score == max(vals[:bst.best_iteration + 1])      # maximised


def test_input_errors(eng):
    qid, y = groups([10] * 20, 11)
    X = make_data(len(qid), 3, 12, "uniform")
    E = eng.XGBoostError
    p = {"objective": "rank:ndcg"}
    with pytest.raises(E, match="qid"):
        eng.train(p, eng.DMatrix(X, label=y), 1, verbose_eval=False)
    with pytest.raises(E, match="non-decreasing"):
        eng.DMatrix(X, label=y, qid=qid[::-1])
    with pytest.raises(E, match="per-group weights"):
        eng.DMatrix(X, label=y, qid=qid, weight=np.ones(len(y), np.float32))
    dm = eng.DMatrix(X, label=y, qid=qid)
    with pytest.raises(E, match="per-group weights"):
        dm.set_info(weight=np.ones(len(y), np.float32))
    with pytest.raises(E, match="group sizes"):
        eng.DMatrix(X, label=y, group=[10] * 19)
    assert np.array_equal(eng.DMatrix(X, label=y, group=[10] * 20).get_group(), dm.get_group())
    for bad, msg in ((np.where(np.arange(len(y)) == 3, np.nan, y), "finite and >= 0"),
                     (np.where(np.arange(len(y)) == 3, -1.0, y), "finite and >= 0"),
                     (np.where(np.arange(len(y)) == 3, np.inf, y), "finite and >= 0"),
                     (np.where(np.arange(len(y)) == 3, 32.0, y), "<= 31")):
        with pytest.raises(E, match=msg):
            eng.train(p, eng.DMatrix(X, label=bad.astype(np.float32), qid=qid), 1, verbose_eval=False)
    eng.train(dict(p, ndcg_exp_gain=False), eng.DMatrix(X, label=(y * 20).astype(np.float32), qid=qid), 1,
              verbose_eval=False)                   # labels above 31 are fine with the linear gain
    with pytest.raises(E, match="not supported"):
        eng.train(dict(p, lambdarank_pair_method="mean"), dm, 1, verbose_eval=False)
    with pytest.raises(E, match="not supported"):
        eng.train(dict(p, lambdarank_unbiased=True), dm, 1, verbose_eval=False)
    for k in (0, -3, "x"):
        with pytest.raises(E, match="lambdarank_num_pair_per_sample"):
            eng.train(dict(p, lambdarank_num_pair_per_sample=k), dm, 1, verbose_eval=False)
    with pytest.raises(E, match="num_class"):
        eng.train(dict(p, num_class=3), dm, 1, verbose_eval=False)
    with pytest.raises(E, match="auc"):
        eng.train({"objective": "rank:pairwise", "eval_metric": "auc"}, dm, 1, evals=[(dm, "t")], verbose_eval=False)
    with pytest.raises(E, match="query groups"):
        eng.train({"objective": "reg:squarederror", "eval_metric": "ndcg"}, eng.DMatrix(X, label=y), 1,
                  evals=[(eng.DMatrix(X, label=y), "t")], verbose_eval=False)
    with pytest.raises(E, match="cut-off"):
        eng.train(dict(p, eval_metric="ndcg@x"), dm, 1, evals=[(dm, "t")], verbose_eval=False)
    # the pre-existing guards of the host layer
    from xgboost_ray_b200 import RayDMatrix, RayDeviceQuantileDMatrix
    with pytest.raises(NotImplementedError):
        RayDMatrix(X, y, qid=qid, weight=np.ones(len(y)))
    with pytest.raises(ValueError):
        RayDeviceQuantileDMatrix(X, y, qid=qid)


def test_save_load_and_continuation(eng, oracle, tmp_path):
    qid, y = groups([30] * 60, 13)
    X = make_data(len(qid), 6, 14, "uniform")
    params = {"objective": "rank:ndcg", "lambdarank_num_pair_per_sample": 10, "ndcg_exp_gain": False, "max_depth": 4}
    dm = eng.DMatrix(X, label=y, qid=qid)
    bst = eng.train(params, dm, 2, verbose_eval=False)
    path = str(tmp_path / "m.json")
    bst.save_model(path)
    d = json.load(open(path))
    assert d["learner"]["objective"] == {"name": "rank:ndcg", "lambdarank_param": {
        "lambdarank_pair_method": "topk", "lambdarank_num_pair_per_sample": "10", "lambdarank_unbiased": "0",
        "lambdarank_bias_norm": "2", "ndcg_exp_gain": "0"}}
    Xt = eng.DMatrix(make_data(1000, 6, 60, "uniform"))
    for raw in (open(path, "rb").read(), None):
        if raw is None:      # a stock xgboost file: only the objective block carries the parameters
            del d["learner"]["attributes"]["b2.params"]
            raw = json.dumps(d).encode()
        loaded = eng.Booster(model_file=bytearray(raw))
        assert int(loaded.params["lambdarank_num_pair_per_sample"]) == 10
        assert loaded.params["ndcg_exp_gain"] == "0"
        assert same_bits(bst.predict(Xt), loaded.predict(Xt))
    cont = eng.train(params, eng.DMatrix(X, label=y, qid=qid), 2, xgb_model=path, verbose_eval=False)
    assert_same_model(cont, R.train(oracle, params, X, y, qid, 4))


def test_pred_contribs_and_leaf(eng):
    qid, y = groups([25] * 80, 15)
    X = make_data(len(qid), 6, 16, "uniform", nan_frac=0.05)
    bst = eng.train({"objective": "rank:pairwise", "max_depth": 5}, eng.DMatrix(X, label=y, qid=qid), 5,
                    verbose_eval=False)
    d = eng.DMatrix(X[:500])
    c = bst.predict(d, pred_contribs=True)
    m = bst.predict(d, output_margin=True)
    assert c.shape == (500, 7)
    assert np.all(np.abs(c.sum(axis=1) - m) <= 1e-5 * np.maximum(1.0, np.abs(m)))
    assert bst.predict(d, pred_leaf=True).shape == (500, 5)


@pytest.mark.parametrize("name", RANKING_CASES)
def test_engine_reproduces_ranking_golden(eng, name):
    want = json.load(open(os.path.join(os.path.dirname(__file__), "golden", name + ".json")))
    x, y, qid, params, rounds = case_data(name)
    bst = eng.train(params, eng.DMatrix(x, label=y, qid=qid), num_boost_round=rounds, verbose_eval=False)
    trees = bst.get_trees()
    assert len(trees) == len(want["trees"])
    for t, g in zip(trees, want["trees"]):
        for k in ("left", "right", "split_feature", "split_bin", "default_left"):
            assert [int(v) for v in t[k]] == g[k], k
        leaf = np.asarray(g["split_feature"]) < 0
        assert np.max(np.abs(t["value"][leaf] - np.asarray(g["value"], np.float32)[leaf])) <= 1e-5
    pred = np.asarray(bst.predict(eng.DMatrix(x[:64])), np.float64)
    ref = np.asarray(want["pred_head"])
    assert np.max(np.abs(pred - ref) / np.maximum(1.0, np.abs(ref))) <= 1e-5


@pytest.mark.timeout(600)
@pytest.mark.parametrize("sharding", ["interleaved", "batch"])
def test_public_api_one_and_two_actors_byte_identical(eng, oracle, sharding):
    """train(RayDMatrix(X, y, qid=...)) with an unsorted qid: 1 and 2 actors give byte-identical models and
    predictions, equal to the oracle on the qid-sorted rows; predict returns the qid-sorted order."""
    from xgboost_ray_b200 import RayDMatrix, RayParams, RayShardingMode, predict, train
    mode = RayShardingMode.INTERLEAVED if sharding == "interleaved" else RayShardingMode.BATCH
    rng = np.random.RandomState(17)
    n = 6000
    X = make_data(n, 6, 18, "uniform")
    qid = rng.randint(0, 150, n)                     # unsorted ids
    y = rng.randint(0, 4, n).astype(np.float32)
    y = np.where(X[:, 2] > 0.2, np.minimum(y + 1, 4), y).astype(np.float32)
    order = np.argsort(qid, kind="mergesort")
    qv = np.repeat(np.arange(10), 30)
    Xv, yv = make_data(300, 6, 19, "uniform"), rng.randint(0, 4, 300).astype(np.float32)
    params = {"objective": "rank:ndcg", "max_depth": 5, "eta": 0.3, "lambdarank_num_pair_per_sample": 16}
    out = {}
    for actors in (1, 2):
        if actors > eng.device_count():
            continue
        dtrain = RayDMatrix(X, y, qid=qid, sharding=mode)
        res = {}
        bst = train(params, dtrain, num_boost_round=4, evals=[(RayDMatrix(Xv, yv, qid=qv, sharding=mode), "v")],
                    evals_result=res, ray_params=RayParams(num_actors=actors))
        assert list(res["v"]) == ["ndcg@16"]
        p = predict(bst, RayDMatrix(X, qid=qid, sharding=mode), ray_params=RayParams(num_actors=actors))
        out[actors] = (bytes(bst.save_raw()), p, bst)
    ob = R.train(oracle, params, X[order], y[order], qid[order], 4)
    assert_same_model(out[1][2], ob)
    assert np.max(np.abs(out[1][1] - ob.predict(X[order]))) <= 1e-5          # qid-sorted order
    if 2 in out:
        assert out[1][0] == out[2][0]
        assert same_bits(out[1][1], out[2][1])
    else:
        pytest.skip("the 2-actor half needs 2 GPUs")


def test_reference_ranking_scenarios(eng):
    """The reference's two ranking scenarios with ndcg in place of auc / aucpr: the 20-row, 4-group toy
    (test_end_to_end.py) and the 20 x 50 / 4 x 50 problem (test_sklearn.py) through train / predict."""
    from xgboost_ray_b200 import RayDMatrix, RayParams, predict, train
    actors = min(2, eng.device_count())
    rng = np.random.RandomState(20)
    X = rng.rand(20, 4).astype(np.float32)
    y = np.array([0, 1, 0, 1, 0, 1, 1, 0, 0, 1, 0, 0, 1, 1, 0, 1, 1, 0, 1, 0], np.float32)
    qid = np.array([0] * 5 + [1] * 5 + [2] * 5 + [3] * 5)
    res = {}
    train({"eta": 1, "objective": "rank:pairwise", "eval_metric": ["ndcg", "map"], "max_depth": 1},
          RayDMatrix(X, label=y, qid=qid), 10, evals=[(RayDMatrix(X, label=y, qid=qid), "train")], evals_result=res,
          ray_params=RayParams(num_actors=actors, max_actor_restarts=0))
    rec = res["train"]["ndcg"]
    assert len(rec) == 10 and rec[-1] >= rec[0]
    x_train, y_train = rng.rand(1000, 10), rng.randint(5, size=1000)
    train_qid = np.repeat(np.array([list(range(20))]), 50)
    x_valid, y_valid = rng.rand(200, 10), rng.randint(5, size=200)
    valid_qid = np.repeat(np.array([list(range(4))]), 50)
    params = {"objective": "rank:pairwise", "eta": 0.1, "gamma": 1.0, "min_child_weight": 0.1, "max_depth": 6,
              "random_state": 1}
    res = {}
    bst = train(params, RayDMatrix(x_train, y_train, qid=train_qid), num_boost_round=4,
                evals=[(RayDMatrix(x_valid, y_valid, qid=valid_qid), "validation")], evals_result=res,
                ray_params=RayParams(num_actors=actors, max_actor_restarts=0))
    assert len(res["validation"]["ndcg@32"]) == 4
    pred = predict(bst, RayDMatrix(rng.rand(100, 10)), ray_params=RayParams(num_actors=actors, max_actor_restarts=0))
    assert pred.shape == (100,) and np.all(np.isfinite(pred))
