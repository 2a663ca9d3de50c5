"""Parameters changed between boosting rounds, without a GPU: the oracle's restatement of a schedule, and the semantics
of callback.LearningRateScheduler (the hook, the epoch, the accepted forms, pickling) driven by the CPU stand-in."""
import pickle

import numpy as np
import pytest

from tests import cpu_engine
from tests import schedule_reference as S
from xgboost_ray_b200 import engine


def _data(n=2000, f=8, seed=0):
    rng = np.random.RandomState(seed)
    X = rng.uniform(0, 10, size=(n, f)).astype(np.float32)
    y = (X[:, 0] + 0.5 * X[:, 1] * X[:, 2] / 10 + rng.normal(size=n)).astype(np.float32)
    return X, y


def _tree_fields(t):
    return {k: getattr(t, k) for k in ("left", "right", "split_feature", "split_bin", "default_left", "value",
                                       "base_weight", "loss_chg", "sum_hess")}


def test_oracle_set_params_equals_fresh_booster_from_the_margin(oracle):
    X, y = _data()
    params = {"objective": "reg:squarederror", "max_depth": 4, "eta": 0.3, "base_score": 0.5}
    cuts = oracle.Cuts.from_data(X, 256)
    bins = cuts.bin(X)
    a = oracle.Booster(params, cuts)
    a.init_margin(len(y))
    for _ in range(5):
        a.boost(bins, y)
    margin5 = a.margin.copy()
    S.set_params(a, {"eta": 0.05})
    for _ in range(5):
        a.boost(bins, y)
    b = oracle.Booster(dict(params, eta=0.05), cuts)
    b.init_margin(len(y), base_margin=margin5)
    for _ in range(5):
        b.boost(bins, y)
    assert a.num_trees == 10 and b.num_trees == 5
    for i in range(5):
        ta, tb = _tree_fields(a.tree(5 + i)), _tree_fields(b.tree(i))
        for k in ta:
            assert np.array_equal(ta[k], tb[k]), (i, k)
    assert np.array_equal(a.margin, b.margin)
    # the trees before the change were grown with eta 0.3: their leaves are 0.3 x their weights
    t0 = a.tree(0)
    leaf = t0.split_feature < 0
    assert np.allclose(t0.value[leaf], t0.base_weight[leaf] * np.float32(0.3), rtol=1e-6, atol=0)


def _rate(epoch):
    return 0.5 / (1 + epoch)


@pytest.fixture
def recording_booster(monkeypatch):
    calls = []

    def set_param(self, params, value=None):
        if isinstance(params, str):
            params = {params: value}
        calls.append((dict(params), self.ob.num_trees))   # trees grown when the callback ran
        self.params.update(params)

    monkeypatch.setattr(cpu_engine.Booster, "set_param", set_param, raising=False)
    return calls


@pytest.mark.parametrize("rates", [[0.3, 0.2, 0.1, 0.05], (0.3, 0.2, 0.1, 0.05), np.array([0.3, 0.2, 0.1, 0.05]),
                                   _rate])
def test_scheduler_sets_rate_i_after_round_i(recording_booster, rates):
    X, y = _data(n=300)
    sched = engine.callback.LearningRateScheduler(rates)
    cpu_engine.train({"max_depth": 2, "eta": 0.3}, cpu_engine.DMatrix(X, y), num_boost_round=4, callbacks=[sched])
    want = [_rate(i) for i in range(4)] if callable(rates) else [0.3, 0.2, 0.1, 0.05]
    assert [c[1] for c in recording_booster] == [1, 2, 3, 4]    # after_iteration: round i is done when rate i is set
    assert [list(c[0]) for c in recording_booster] == [["learning_rate"]] * 4
    assert [c[0]["learning_rate"] for c in recording_booster] == pytest.approx(want, rel=0, abs=0)


def test_scheduler_refuses_other_forms():
    for bad in (0.1, "0.1,0.2", None, {"0": 0.1}):
        with pytest.raises(TypeError, match="learning_rates"):
            engine.callback.LearningRateScheduler(bad)


def test_scheduler_pickles_and_is_the_xgb_callback():
    from xgboost_ray_b200 import xgb
    assert xgb.xgboost.callback.LearningRateScheduler is engine.LearningRateScheduler
    assert issubclass(engine.LearningRateScheduler, engine.TrainingCallback)
    for rates in ([0.3, 0.1], _rate):
        s = pickle.loads(pickle.dumps(engine.LearningRateScheduler(rates)))
        got = []

        class M:
            def set_param(self, k, v):
                got.append((k, v))

        assert s.after_iteration(M(), 1, {}) is False
        assert got == [("learning_rate", 0.1 if isinstance(rates, list) else _rate(1))]
