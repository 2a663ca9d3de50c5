"""Pipelined boosting rounds: update() enqueues round r+1 and finishes round r while the device works, so the round it
returns from is still pending.  Every test compares against the same training with a draining call (num_trees) after
every update(), which leaves no round pending between two calls."""
import gc
import pickle

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _data(n=30011, f=13, seed=0, classes=0):
    rng = np.random.RandomState(seed)
    x = rng.uniform(0, 10, size=(n, f)).astype(np.float32)
    x[rng.uniform(size=x.shape) < 0.03] = np.nan
    s = np.nan_to_num(x[:, 0]) + 0.5 * np.nan_to_num(x[:, 3]) * np.sin(np.nan_to_num(x[:, 5])) + rng.normal(size=n)
    if classes:
        y = np.clip((s / 16 * classes).astype(np.int64), 0, classes - 1).astype(np.float32)
    else:
        y = s.astype(np.float32)
    return x, y


PARAMS = {"reg:squarederror": {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5},
          "binary:logistic": {"objective": "binary:logistic", "max_depth": 6, "eta": 0.3, "base_score": 0.5},
          "multi:softprob": {"objective": "multi:softprob", "num_class": 3, "max_depth": 5, "eta": 0.3}}


def _matrix(E, objective):
    x, y = _data(classes=3 if objective == "multi:softprob" else 0)
    if objective == "binary:logistic":
        y = (y > 6).astype(np.float32)
    return E.DMatrix(x, label=y)


def _grow(E, params, dm, rounds, drain_each):
    bst = E.Booster(params, cache=[dm])
    for r in range(rounds):
        bst.update(dm, r)
        if drain_each:
            bst.num_trees()
    return bst


def _dump(bst):
    return bst.get_dump(dump_format="json", with_stats=True)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("objective", ["reg:squarederror", "binary:logistic", "multi:softprob"])
def test_thirty_pipelined_rounds_equal_the_drained_rounds(objective):
    """30 rounds cross both graph parities many times; a tree read back from the wrong round's block would differ."""
    from xgboost_ray_b200 import engine as E
    dm = _matrix(E, objective)
    ref = _grow(E, PARAMS[objective], dm, 30, drain_each=True)
    bst = _grow(E, PARAMS[objective], dm, 30, drain_each=False)
    k = PARAMS[objective].get("num_class", 1)
    assert bst.num_trees() == ref.num_trees() == 30 * k
    assert _dump(bst) == _dump(ref)
    assert len(set(_dump(bst))) > 20 * k     # the rounds grew different trees
    assert np.array_equal(bst.predict(dm, output_margin=True, training=True), ref.predict(dm, output_margin=True, training=True))


def _num_trees(bst, ref, dm, tmp_path):
    assert bst.num_trees() == ref.num_trees() == 7


def _get_dump(bst, ref, dm, tmp_path):
    assert _dump(bst) == _dump(ref)


def _predict(bst, ref, dm, tmp_path):
    assert np.array_equal(bst.predict(dm), ref.predict(dm))


def _train_margin(bst, ref, dm, tmp_path):
    assert np.array_equal(bst.predict(dm, output_margin=True, training=True),
                          ref.predict(dm, output_margin=True, training=True))


def _eval_set(bst, ref, dm, tmp_path):
    assert bst.eval_set([(dm, "train")], 7) == ref.eval_set([(dm, "train")], 7)


def _json_round_trip(bst, ref, dm, tmp_path):
    from xgboost_ray_b200 import engine as E
    bst.save_model(str(tmp_path / "m.json"))
    loaded = E.Booster(model_file=str(tmp_path / "m.json"))
    assert _dump(loaded) == _dump(ref)
    assert np.array_equal(loaded.predict(dm), ref.predict(dm))


def _pickle(bst, ref, dm, tmp_path):
    assert _dump(pickle.loads(pickle.dumps(bst))) == _dump(ref)


def _continuation(bst, ref, dm, tmp_path):
    from xgboost_ray_b200 import engine as E
    params = PARAMS["reg:squarederror"]
    more = E.train(params, dm, num_boost_round=3, xgb_model=bst, verbose_eval=False)
    more_ref = E.train(params, dm, num_boost_round=3, xgb_model=ref, verbose_eval=False)
    assert more.num_trees() == 10
    assert _dump(more) == _dump(more_ref)


def _timers(bst, ref, dm, tmp_path):
    t, r = bst.get_timers(reset=True), ref.get_timers(reset=True)
    assert t["rounds"] == r["rounds"] == 7
    assert t["hist_launches"] == r["hist_launches"] == 7 * 6     # root + 5 built levels per depth-6 tree
    assert t["kernel_launches"] == r["kernel_launches"]
    assert bst.get_timers()["rounds"] == 0


READS = [_num_trees, _get_dump, _predict, _train_margin, _eval_set, _json_round_trip, _pickle, _continuation, _timers]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("read", READS, ids=[f.__name__.lstrip("_") for f in READS])
def test_every_read_sees_the_pending_round(read, tmp_path):
    from xgboost_ray_b200 import engine as E
    dm = _matrix(E, "reg:squarederror")
    ref = _grow(E, PARAMS["reg:squarederror"], dm, 7, drain_each=True)
    bst = _grow(E, PARAMS["reg:squarederror"], dm, 7, drain_each=False)   # round 6 is pending here
    read(bst, ref, dm, tmp_path)


@pytest.mark.timeout(600)
def test_sampled_multiclass_parallel_trees_equal_the_drained_rounds():
    """Row and column sampling are seeded by the tree's position in the model, which counts the pending round's
    trees: K = 3 classes x 2 parallel trees = 6 trees per round."""
    from xgboost_ray_b200 import engine as E
    params = dict(PARAMS["multi:softprob"], num_parallel_tree=2, subsample=0.7, colsample_bytree=0.6,
                  colsample_bylevel=0.6, colsample_bynode=0.6, seed=11)
    dm = _matrix(E, "multi:softprob")
    ref = _grow(E, params, dm, 8, drain_each=True)
    bst = _grow(E, params, dm, 8, drain_each=False)
    assert bst.num_trees() == ref.num_trees() == 8 * 6
    assert _dump(bst) == _dump(ref)
    assert np.array_equal(bst.predict(dm), ref.predict(dm))


@pytest.mark.timeout(300)
@pytest.mark.parametrize("drain_each", [False, True])
def test_non_finite_gradient_fails_its_own_round(drain_each):
    """reg:gamma with labels far below exp(margin) and no L2 term: round 0 grows leaves near 1 - 1/y = -999, which
    puts the margin where exp overflows, so round 1's gradients are infinite.  update() of round 1 raises, and its
    trees never exist."""
    from xgboost_ray_b200 import engine as E
    x, _ = _data(n=4000, f=6, seed=2)
    y = np.full(x.shape[0], 1e-3, np.float32)
    params = {"objective": "reg:gamma", "base_score": 1.0, "eta": 1.0, "lambda": 1e-6, "min_child_weight": 0,
              "max_depth": 2}
    dm = E.DMatrix(x, label=y)
    bst = E.Booster(params, cache=[dm])
    done = 0
    with pytest.raises(E.XGBoostError, match="not finite"):
        for r in range(10):
            bst.update(dm, r)
            done += 1
            if drain_each:
                bst.num_trees()
    assert done >= 1
    assert bst.num_trees() == done


@pytest.mark.timeout(300)
def test_free_and_cancel_with_a_round_pending():
    from xgboost_ray_b200 import engine as E
    params = PARAMS["reg:squarederror"]
    dm = _matrix(E, "reg:squarederror")
    ref = _grow(E, params, dm, 5, drain_each=True)
    for _ in range(3):
        b = _grow(E, params, dm, 4, drain_each=False)    # freed with its last round pending
        del b
        gc.collect()
    b = _grow(E, params, dm, 4, drain_each=False)
    b.cancel()
    with pytest.raises(E.XGBoostError, match="training cancelled"):
        b.update(dm, 4)
    assert b.num_trees() == 4                            # the pending round was drained, the cancelled one never ran
    assert _dump(b) == _dump(ref)[:4]
    del b
    gc.collect()
    again = _grow(E, params, dm, 5, drain_each=False)    # a second booster on the same matrix trains normally
    assert _dump(again) == _dump(ref)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_two_gpu_pipelined_rounds_equal_one_gpu(exchange, monkeypatch):
    """Each rank pipelines its own stream; the exchange collectives stay in stream order.  Both exchanges, 30 rounds
    without reads between them (two graph parities per rank), against one GPU."""
    from xgboost_ray_b200 import engine
    if engine.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import xgboost_ray_b200.main as M
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    M.shutdown_actors()                       # the exchange kind is read by the actor processes when they start
    if exchange == "nccl":
        monkeypatch.setenv("B2_EXCHANGE", "nccl")
    else:
        monkeypatch.delenv("B2_EXCHANGE", raising=False)
    x, y = _data(n=60013, f=37, seed=21)
    params = {"objective": "reg:squarederror", "max_depth": 8, "eta": 0.3, "base_score": 0.5}
    b1 = train(params, RayDMatrix(x, y), num_boost_round=30, ray_params=RayParams(num_actors=1))
    b2 = train(params, RayDMatrix(x, y), num_boost_round=30, ray_params=RayParams(num_actors=2))
    assert b2.num_trees() == 30
    assert _dump(b1) == _dump(b2)
    M.shutdown_actors()
