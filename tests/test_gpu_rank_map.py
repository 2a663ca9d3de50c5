"""GPU checks of rank:map: gradients bit-equal to tests/rank_map_reference.py (read back with B2_BoosterGetGradients)
for staged and global-scratch groups, trees identical to the oracle grown from them, the default map@k metric and
early stopping, input errors, save / load / a stock model file / continuation, the golden fixture and the public
train / predict with qid on one and two GPUs."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from tests import rank_map_reference as M
from tests import ranking_reference as R
from tests.golden.make_golden_rank_map import CASES as MAP_CASES, case_data
from tests.test_gpu_parity import assert_same_model, make_data

pytestmark = pytest.mark.gpu

MAP = M.MAP_OBJECTIVE
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


def groups(sizes, seed, rate=0.3):
    """qid of consecutive groups of the given sizes and binary labels with P(1) = rate."""
    rng = np.random.RandomState(seed)
    qid = np.repeat(np.arange(len(sizes)), sizes)
    y = (rng.rand(len(qid)) < rate).astype(np.float32)
    return qid, y


def same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize("k", [1, 5, 32, 10000])
@pytest.mark.parametrize("rate", [0.0, 0.05, 0.5, 1.0])
@pytest.mark.parametrize("margins", ["round0", "base_margin"])
def test_gradients_bit_equal_to_reference(eng, k, rate, margins):
    """Group sizes 1 .. 40000 (5000 and 40000 are above the shared-memory stage: their A and R live in the global
    scratch), hit rates 0 / 5 % / 50 % / 100 %, all-tied margins at round 0 and a base_margin with +-0.0 and repeated
    values: the gradient pairs equal the reference bit for bit.  With k = 10^4 the 40000-row group is left out
    (4 * 10^8 pairs of one group)."""
    sizes = SIZES if k < 10000 else SIZES[:-1]
    qid, y = groups(sizes, 1, rate)
    n = len(qid)
    X = make_data(n, 3, 2, "uniform")
    rng = np.random.RandomState(k)
    params = {"objective": MAP, "lambdarank_num_pair_per_sample": k, "max_depth": 2}
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
    rg, rh, bad = M.gradients(params, m, y, R.group_ptr(qid))
    assert not bad
    assert same_bits(g, rg), np.nonzero(g != rg)[0][:10]
    assert same_bits(h, rh), np.nonzero(h != rh)[0][:10]
    if 0.0 < rate < 1.0:
        assert np.count_nonzero(g) > 0


@pytest.mark.parametrize("depth", [3, 6])
def test_trees_identical_to_oracle(eng, oracle, depth):
    sizes = [1, 2, 3, 37, 100] * 12 + [3000]
    qid, y = groups(sizes, 5 + depth, rate=0.15)
    n, f = len(qid), 8
    X = make_data(n, f, 31, "uniform", nan_frac=0.1)
    y = np.where(X[:, 0] > 0.5, 1.0, y).astype(np.float32)
    params = {"objective": MAP, "max_depth": depth, "eta": 0.3, "lambdarank_num_pair_per_sample": 8}
    obst = M.train(oracle, params, X, y, qid, 4)
    ebst = eng.train(params, eng.DMatrix(X, label=y, qid=qid), num_boost_round=4, verbose_eval=False)
    assert_same_model(ebst, obst)
    Xt = make_data(2000, f, 99, "uniform")
    pe, po = ebst.predict(eng.DMatrix(Xt)), obst.predict(Xt)
    assert np.max(np.abs(pe - po) / np.maximum(1.0, np.abs(po))) <= 1e-5


def test_default_metric_early_stopping_and_map_value(eng):
    qid, y = groups([20] * 40, 9)
    X = make_data(len(qid), 6, 10, "uniform")
    y = np.where(X[:, 1] > 0.4, 1.0, y).astype(np.float32)
    dm = eng.DMatrix(X, label=y, qid=qid)
    qv, yv = groups([15] * 10, 19)
    dv = eng.DMatrix(make_data(len(qv), 6, 20, "uniform"), label=yv, qid=qv)
    for k, want in ((None, "map@32"), (7, "map@7")):
        res = {}
        p = {"objective": MAP} if k is None else {"objective": MAP, "lambdarank_num_pair_per_sample": k}
        bst = eng.train(p, dm, 2, evals=[(dm, "t")], evals_result=res, verbose_eval=False)
        assert list(res["t"]) == [want]
        assert bst.params["base_score"] == 0.5
        assert np.all(bst.predict(dm, output_margin=True) == bst.predict(dm))      # identity transform
        for d, yy, q in ((dm, y, qid), (dv, yv, qv)):
            out = C.c_double(0)
            eng._check(eng.lib().B2_BoosterEvalSet(bst.handle, d.handle, want.encode(), C.byref(out)))
            ref = R.metric(want, bst.predict(d), yy, R.group_ptr(q))
            assert abs(out.value - ref) <= 1e-12 * max(1.0, abs(ref))
    res = {}
    bst = eng.train({"objective": MAP, "max_depth": 3, "eta": 0.5}, dm, 10, evals=[(dv, "v")], evals_result=res,
                    early_stopping_rounds=2, verbose_eval=False)
    vals = res["v"]["map@32"]
    assert bst.best_score == max(vals[:bst.best_iteration + 1])                      # maximised
    # training on rank:map raises the train map
    res = {}
    eng.train({"objective": MAP, "max_depth": 4}, dm, 8, evals=[(dm, "t")], evals_result=res, verbose_eval=False)
    assert res["t"]["map@32"][-1] > res["t"]["map@32"][0]


def test_input_errors(eng):
    qid, y = groups([10] * 20, 11)
    X = make_data(len(qid), 3, 12, "uniform")
    E = eng.XGBoostError
    p = {"objective": MAP}
    for bad in (0.5, 2.0, np.nan, -1.0, np.inf):
        yb = np.where(np.arange(len(y)) == 3, bad, y).astype(np.float32)
        with pytest.raises(E, match=r"rank:map.*0 or 1"):
            eng.train(p, eng.DMatrix(X, label=yb, qid=qid), 1, verbose_eval=False)
    # relevance grades 0..4, accepted by rank:ndcg, are refused
    with pytest.raises(E, match=r"rank:map.*0 or 1"):
        eng.train(p, eng.DMatrix(X, label=(y * 3).astype(np.float32), qid=qid), 1, verbose_eval=False)
    with pytest.raises(E, match="query groups"):
        eng.train(p, eng.DMatrix(X, label=y), 1, verbose_eval=False)
    with pytest.raises(E, match="per-group weights"):
        eng.DMatrix(X, label=y, qid=qid, weight=np.ones(len(y), np.float32))
    dm = eng.DMatrix(X, label=y, qid=qid)
    with pytest.raises(E, match="per-group weights"):
        dm.set_info(weight=np.ones(len(y), np.float32))
    with pytest.raises(E, match="num_class"):
        eng.train(dict(p, num_class=3), dm, 1, verbose_eval=False)
    with pytest.raises(E, match="not supported"):
        eng.train(dict(p, lambdarank_pair_method="mean"), dm, 1, verbose_eval=False)
    # ndcg_exp_gain is accepted and does not change rank:map
    a = eng.train(dict(p, ndcg_exp_gain=False), dm, 2, verbose_eval=False)
    b = eng.train(p, dm, 2, verbose_eval=False)
    assert same_bits(a.predict(dm), b.predict(dm))


def test_save_load_stock_file_and_continuation(eng, oracle, tmp_path):
    qid, y = groups([30] * 60, 13)
    X = make_data(len(qid), 6, 14, "uniform")
    y = np.where(X[:, 2] > 0.3, 1.0, y).astype(np.float32)
    params = {"objective": MAP, "lambdarank_num_pair_per_sample": 10, "max_depth": 4}
    dm = eng.DMatrix(X, label=y, qid=qid)
    bst = eng.train(params, dm, 2, verbose_eval=False)
    path = str(tmp_path / "m.json")
    bst.save_model(path)
    d = json.load(open(path))
    block = {"lambdarank_pair_method": "topk", "lambdarank_num_pair_per_sample": "10", "lambdarank_unbiased": "0",
             "lambdarank_bias_norm": "2", "ndcg_exp_gain": "1"}
    assert d["learner"]["objective"] == {"name": "rank:map", "lambdarank_param": block}
    cfg = json.loads(bst.save_config())
    assert cfg["learner"]["objective"] == {"name": "rank:map", "lambdarank_param": block}
    Xt = eng.DMatrix(make_data(1000, 6, 60, "uniform"))
    stock = str(tmp_path / "stock.json")
    del d["learner"]["attributes"]["b2.params"]      # a stock xgboost file: only the objective block carries them
    with open(stock, "w") as f:
        json.dump(d, f)
    for src in (path, stock):
        loaded = eng.Booster(model_file=bytearray(open(src, "rb").read()))
        assert loaded.params["objective"] == MAP
        assert int(loaded.params["lambdarank_num_pair_per_sample"]) == 10
        assert same_bits(bst.predict(Xt), loaded.predict(Xt))
        cont = eng.train(params, eng.DMatrix(X, label=y, qid=qid), 2, xgb_model=src, verbose_eval=False)
        assert_same_model(cont, M.train(oracle, params, X, y, qid, 4))


@pytest.mark.parametrize("name", MAP_CASES)
def test_engine_reproduces_rank_map_golden(eng, name):
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
    y = ((X[:, 2] > 0.2) & (rng.rand(n) < 0.6)).astype(np.float32)
    order = np.argsort(qid, kind="mergesort")
    qv = np.repeat(np.arange(10), 30)
    Xv, yv = make_data(300, 6, 19, "uniform"), (rng.rand(300) < 0.3).astype(np.float32)
    params = {"objective": MAP, "max_depth": 5, "eta": 0.3, "lambdarank_num_pair_per_sample": 16}
    out = {}
    for actors in (1, 2):
        if actors > eng.device_count():
            continue
        dtrain = RayDMatrix(X, y, qid=qid, sharding=mode)
        res = {}
        bst = train(params, dtrain, num_boost_round=4, evals=[(RayDMatrix(Xv, yv, qid=qv, sharding=mode), "v")],
                    evals_result=res, ray_params=RayParams(num_actors=actors))
        assert list(res["v"]) == ["map@16"]
        p = predict(bst, RayDMatrix(X, qid=qid, sharding=mode), ray_params=RayParams(num_actors=actors))
        out[actors] = (bytes(bst.save_raw()), p, bst)
    ob = M.train(oracle, params, X[order], y[order], qid[order], 4)
    assert_same_model(out[1][2], ob)
    assert np.max(np.abs(out[1][1] - ob.predict(X[order]))) <= 1e-5          # qid-sorted order
    if 2 in out:
        assert out[1][0] == out[2][0]
        assert same_bits(out[1][1], out[2][1])
    else:
        pytest.skip("the 2-actor half needs 2 GPUs")
