"""Booster slicing (`bst[a:b:s]`, `iter(bst)`) and callback.EarlyStopping without a GPU (DESIGN.md 2 item 23).

Slicing is host-side: the boosters here are loaded with load_model from XGBoost 2.x JSON files written by
tests/model_files.py, and every slice is compared with the same file edited to keep the selected rounds.  EarlyStopping
is driven by hand-made evals_log dicts, the way train() calls it."""
import json
import pickle

import jsonschema
import numpy as np
import pytest

from tests.model_files import keep_rounds, xgb_model_file
from tests.model_schema import GBTREE, MODEL
from xgboost_ray_b200 import engine as E


def _load(raw):
    return E.Booster(model_file=bytearray(raw))


def _tags(bst):
    """The tree ids tests/model_files.py wrote into each tree's loss_chg."""
    return [int(t["loss_chg"][0]) - 1 for t in bst.get_trees()]


@pytest.fixture(scope="module")
def ten():
    raw = xgb_model_file(10, attrs={"owner": "slicing"})
    return raw, _load(raw)


@pytest.mark.parametrize("index,rounds", [
    (3, [3]), (np.int64(9), [9]), (0, [0]),
    (slice(2, 5), [2, 3, 4]), (slice(None, 4), [0, 1, 2, 3]), (slice(6, None), [6, 7, 8, 9]),
    (slice(None, None), list(range(10))), (slice(3, 0), list(range(3, 10))), (slice(0, 0), list(range(10))),
    (slice(1, 9, 3), [1, 4, 7]), (slice(None, None, 4), [0, 4, 8]), (slice(2, 10, 20), [2]),
    (slice(9, 10), [9]),
])
def test_slice_selects_rounds(ten, index, rounds):
    raw, bst = ten
    s = bst[index]
    assert isinstance(s, E.Booster) and s is not bst
    assert _tags(s) == rounds and s.num_boosted_rounds() == len(rounds)
    assert bytes(s.save_raw()) == bytes(_load(keep_rounds(raw, rounds)).save_raw())


@pytest.mark.parametrize("index,error,match", [
    (slice(5, 3), ValueError, "ends before it starts"),
    (slice(None, None, 0), ValueError, "step must be >= 1"),
    (slice(None, None, -1), ValueError, "step must be >= 1"),
    (-1, ValueError, "negative"),
    (slice(-3, None), ValueError, "negative"),
    (slice(2, -1), ValueError, "negative"),
    ((1, 2), ValueError, "only 1 dimension"),
    ((slice(None), 0), ValueError, "only 1 dimension"),
    ("1", TypeError, "int or a slice"),
    (1.0, TypeError, "int or a slice"),
    (None, TypeError, "int or a slice"),
    (slice(1.5, 3), TypeError, "integer"),
    (10, IndexError, "out of range: the model has 10 rounds"),
    (slice(10, None), IndexError, "out of range"),
    (slice(0, 11), IndexError, "out of range"),
    (slice(12, 0), IndexError, "out of range"),
])
def test_slice_argument_errors(ten, index, error, match):
    _, bst = ten
    with pytest.raises(error, match=match):
        bst[index]


def test_iter_yields_each_round(ten):
    raw, bst = ten
    layers = list(bst)
    assert len(layers) == 10 and [_tags(b) for b in layers] == [[i] for i in range(10)]
    for i, b in enumerate(layers):
        assert bytes(b.save_raw()) == bytes(bst[i].save_raw())
    assert [_tags(b) for b in iter(bst[7:])] == [[7], [8], [9]]


CASES = {
    "softprob_k20": dict(objective="multi:softprob", num_class=20),
    "parallel_3": dict(npt=3),
    "softprob_k3_parallel_2": dict(objective="multi:softprob", num_class=3, npt=2),
    "quantile_3_alphas": dict(objective="reg:quantileerror", alphas=[0.1, 0.5, 0.9]),
    "dart": dict(dart=True),
    "dart_softmax_parallel_2": dict(dart=True, objective="multi:softmax", num_class=3, npt=2),
    "vector_leaf_4": dict(vector=4),
    "categorical_inf": dict(categorical=True),
}
PER_ROUND = {"softprob_k20": 20, "parallel_3": 3, "softprob_k3_parallel_2": 6, "quantile_3_alphas": 3, "dart": 1,
             "dart_softmax_parallel_2": 6, "vector_leaf_4": 1, "categorical_inf": 1}


@pytest.mark.parametrize("case", list(CASES))
def test_layers_and_model_file(case):
    raw = xgb_model_file(5, **CASES[case])
    bst = _load(raw)
    per = PER_ROUND[case]
    assert bst._trees_per_round == per and bst.num_boosted_rounds() == 5 and bst.num_trees() == 5 * per
    before = bytes(bst.save_raw())
    for rounds, s in (([1, 3], bst[1:5:2]), ([4], bst[4]), ([0, 1, 2], bst[:3]), (list(range(5)), bst[:])):
        keep = [r * per + j for r in rounds for j in range(per)]
        assert _tags(s) == keep
        d = json.loads(bytes(s.save_raw()).decode())
        gb = d["learner"]["gradient_booster"]
        m = (gb["gbtree"] if gb["name"] == "dart" else gb)["model"]
        src = json.loads(raw.decode())["learner"]["gradient_booster"]
        src_m = (src["gbtree"] if src["name"] == "dart" else src)["model"]
        assert m["iteration_indptr"] == list(range(0, len(keep) + 1, per))
        assert m["tree_info"] == [src_m["tree_info"][t] for t in keep]
        assert [t["id"] for t in m["trees"]] == list(range(len(keep)))
        assert m["gbtree_model_param"] == {"num_parallel_tree": str(CASES[case].get("npt", 1)),
                                           "num_trees": str(len(keep))}
        jsonschema.validate(gb["gbtree"] if gb["name"] == "dart" else gb, GBTREE)
        if gb["name"] == "gbtree" and d["learner"]["objective"]["name"] in ("reg:squarederror", "multi:softprob",
                                                                            "multi:softmax"):
            jsonschema.validate(d, MODEL)
        if gb["name"] == "dart":   # weight_drop: the selected trees' float32 weights, bit for bit
            w = np.asarray(src["weight_drop"], np.float32)[keep]
            assert np.asarray(gb["weight_drop"], np.float32).tobytes() == w.tobytes()
            assert s.get_tree_weights().tobytes() == w.tobytes()
        whole = json.loads(bytes(bst.save_raw()).decode())["learner"]
        for k in ("learner_model_param", "objective", "feature_names", "feature_types"):
            assert d["learner"][k] == whole[k], k
        assert bytes(s.save_raw()) == bytes(_load(keep_rounds(raw, rounds)).save_raw())
    assert bytes(bst.save_raw()) == before         # slicing leaves the source as it was


def test_slice_carries_every_tree_field_params_and_attributes():
    raw = xgb_model_file(6, categorical=True, attrs={"note": "kept"})
    bst = _load(raw)
    bst.set_param({"eval_metric": "mae", "max_depth": 3})
    bst.best_iteration, bst.best_score = 4, 0.125
    bst._cuts = (np.zeros(5, np.int32), np.zeros(0, np.float32), np.zeros(4, np.float32), np.zeros(4, np.uint8))
    s = bst[:3]
    assert s.params == bst.params and s.params is not bst.params
    assert s.params["base_score"] == 0.375 and s.params["max_depth"] == 3
    assert (s.n_features, s.feature_names, s.feature_types) == (4, ["f_0", "f_1", "f_2", "f_3"], ["c", "q", "q", "q"])
    assert s.attributes() == bst.attributes() == {"note": "kept"}
    assert s.best_iteration is None and s.best_score is None and s._cuts is None and s.handle == 0
    for t, u in zip(bst.get_trees()[:3], s.get_trees()):
        assert set(t) == set(u)
        for k, v in t.items():
            if v is None:
                assert u[k] is None
            else:
                assert np.asarray(v).tobytes() == np.asarray(u[k]).tobytes() and u[k] is not v, k
    assert s.get_trees()[1]["split_cond"][0] == np.inf and E._cat_list(s.get_trees()[0]["cat_bits"][0]) == [1, 3, 200]
    assert s.get_dump(with_stats=True) == bst.get_dump(with_stats=True)[:3]
    assert s.get_dump(dump_format="json") == bst.get_dump(dump_format="json")[:3]
    ref = _load(keep_rounds(bytes(bst.save_raw()), [0, 1, 2]))
    for kind in ("weight", "gain", "cover", "total_gain", "total_cover"):
        assert s.get_score(importance_type=kind) == ref.get_score(importance_type=kind)
    assert s.save_config() == bst.save_config()
    s.set_attr(note="changed")          # the slice is a model of its own
    assert bst.attr("note") == "kept"


def test_vector_leaf_slice_keeps_leaf_vectors():
    bst = _load(xgb_model_file(4, vector=4))
    s = bst[2:]
    assert s.is_vector_leaf and s.params["multi_strategy"] == "multi_output_tree" and s.params["num_target"] == 4
    for t, u in zip(bst.get_trees()[2:], s.get_trees()):
        assert u["leaf_vector"].shape == (3, 4) and u["leaf_vector"].tobytes() == t["leaf_vector"].tobytes()


def test_quantile_and_parallel_params_carry():
    q = _load(xgb_model_file(3, objective="reg:quantileerror", alphas=[0.1, 0.5, 0.9]))[1]
    assert q.num_class == 3 and E.quantile_alpha_text(q.params["quantile_alpha"]) == "[0.100000001, 0.5, 0.899999976]"
    p = _load(xgb_model_file(3, objective="multi:softprob", num_class=3, npt=2))[1:]
    assert p.num_parallel_tree == 2 and p.num_class == 3 and p.num_boosted_rounds() == 2


def test_slice_pickles_and_round_trips(tmp_path):
    raw = xgb_model_file(5, dart=True, objective="multi:softprob", num_class=3)
    s = _load(raw)[1:5:3]
    s.best_iteration, s.best_score = 1, 0.5
    p = pickle.loads(pickle.dumps(s))
    assert bytes(p.save_raw()) == bytes(s.save_raw()) and (p.best_iteration, p.best_score) == (1, 0.5)
    f = str(tmp_path / "slice.json")
    s.save_model(f)
    assert bytes(E.Booster(model_file=f).save_raw()) == bytes(s.save_raw())
    assert bytes(s.copy().save_raw()) == bytes(s.save_raw())


# ----------------------------------------------------------------------------- EarlyStopping
class _Model:
    """What EarlyStopping reads and writes on a model, recording the slices it takes."""

    def __init__(self, rounds=0):
        self.rounds, self.best_iteration, self.best_score, self.sliced = rounds, None, None, []

    def num_boosted_rounds(self):
        return self.rounds

    def __getitem__(self, val):
        self.sliced.append(val)
        return _Model(len(range(*val.indices(self.rounds))))


def _drive(cb, scores, model=None, data="valid", metric="rmse", log=None):
    """Run cb over the rounds of `scores` as train() does; returns (model, the epoch it stopped at or None)."""
    model = model or _Model()
    cb.before_training(model)
    log = log if log is not None else {}
    for epoch, v in enumerate(scores):
        log.setdefault(data, {}).setdefault(metric, []).append(v)
        model.rounds += 1
        if cb.after_iteration(model, epoch, log):
            return model, epoch
    return model, None


def test_stops_after_rounds_without_improvement():
    m, stop = _drive(E.callback.EarlyStopping(3), [5.0, 4.0, 4.0, 4.5, 4.0, 3.0])
    assert stop == 4 and (m.best_iteration, m.best_score) == (1, 4.0)
    m, stop = _drive(E.callback.EarlyStopping(2), [5.0, 4.0, 3.0, 2.0])
    assert stop is None and (m.best_iteration, m.best_score) == (3, 2.0)
    m, stop = _drive(E.callback.EarlyStopping(1), [1.0, 1.0])
    assert stop == 1 and m.best_iteration == 0       # an equal score does not improve


@pytest.mark.parametrize("maximize,scores,best", [
    (False, [1.0, 0.75, 0.7], (2, 0.7)),      # best - 0.25 > 0.75 is false; 0.7 improves
    (True, [1.0, 1.25, 1.3], (2, 1.3)),       # 1.25 - 0.25 > 1.0 is false; 1.3 improves
])
def test_min_delta_boundary(maximize, scores, best):
    m, stop = _drive(E.callback.EarlyStopping(5, maximize=maximize, min_delta=0.25), scores)
    assert stop is None and (m.best_iteration, m.best_score) == best
    m, stop = _drive(E.callback.EarlyStopping(1, maximize=maximize, min_delta=0.25), scores[:2])
    assert stop == 1 and m.best_iteration == 0


def test_min_delta_must_not_be_negative():
    with pytest.raises(ValueError, match="min_delta"):
        E.callback.EarlyStopping(3, min_delta=-1e-9)


@pytest.mark.parametrize("metric,maximized", [("rmse", False), ("logloss", False), ("auc", True), ("aucpr", True),
                                              ("ndcg@5", True), ("map", True), ("pre@3", True), ("mae", False)])
def test_direction_follows_the_metric(metric, maximized):
    scores = [0.5, 0.6, 0.4]
    m, _ = _drive(E.callback.EarlyStopping(5), scores, metric=metric)
    assert m.best_score == (0.6 if maximized else 0.4)
    m, _ = _drive(E.callback.EarlyStopping(5, maximize=not maximized), scores, metric=metric)
    assert m.best_score == (0.4 if maximized else 0.6)


def _log():
    return {"train": {"rmse": [3.0, 2.0, 1.0], "mae": [3.0, 2.0, 1.0]},
            "valid": {"rmse": [3.0, 2.0, 2.5], "mae": [3.0, 3.5, 4.0], "auc": [0.5, 0.7, 0.6]}}


@pytest.mark.parametrize("kw,best", [
    ({}, (1, 0.7)),                                           # the last eval set and its last metric: valid-auc
    ({"metric_name": "rmse"}, (1, 2.0)),
    ({"metric_name": "mae"}, (0, 3.0)),
    ({"data_name": "train"}, (2, 1.0)),                      # train's last metric: mae
    ({"data_name": "train", "metric_name": "rmse"}, (2, 1.0)),
])
def test_named_and_default_metric_and_data(kw, best):
    cb, m, full = E.callback.EarlyStopping(10, **kw), _Model(), _log()
    cb.before_training(m)
    for epoch in range(3):
        log = {d: {k: v[:epoch + 1] for k, v in ms.items()} for d, ms in full.items()}
        assert cb.after_iteration(m, epoch, log) is False
    assert (m.best_iteration, m.best_score) == best


@pytest.mark.parametrize("kw,match", [({"data_name": "test"}, "no eval set named 'test'"),
                                      ({"metric_name": "error"}, "has no metric named 'error'"),
                                      ({"data_name": "train", "metric_name": "auc"},
                                       "'train' has no metric named 'auc'")])
def test_unknown_names_raise(kw, match):
    with pytest.raises(ValueError, match=match):
        E.callback.EarlyStopping(2, **kw).after_iteration(_Model(), 0, _log())


def test_needs_an_eval_set():
    with pytest.raises(ValueError, match="at least one eval set"):
        E.callback.EarlyStopping(2).after_iteration(_Model(), 0, {})


def test_best_iteration_counts_the_rounds_of_xgb_model():
    m, stop = _drive(E.callback.EarlyStopping(2), [3.0, 2.0, 2.5, 2.5], model=_Model(rounds=7))
    assert stop == 3 and (m.best_iteration, m.best_score) == (8, 2.0)


def test_save_best_returns_the_best_rounds():
    cb = E.callback.EarlyStopping(2, save_best=True)
    m, stop = _drive(cb, [3.0, 2.0, 2.5, 2.5])
    out = cb.after_training(m)
    assert m.sliced == [slice(None, 2)] and out.rounds == 2 and (out.best_iteration, out.best_score) == (1, 2.0)
    cb = E.callback.EarlyStopping(2)
    m, _ = _drive(cb, [3.0, 2.0, 2.5, 2.5])
    assert cb.after_training(m) is m and m.sliced == []
    # a real booster: the slice holds the first best_iteration + 1 rounds (DART weights included)
    raw = xgb_model_file(6, dart=True)
    bst = _load(raw)
    cb = E.callback.EarlyStopping(2, save_best=True)
    log = {"valid": {"rmse": []}}
    for epoch, v in enumerate([3.0, 2.0, 1.5, 1.75, 1.6]):
        log["valid"]["rmse"].append(v)
        stop = cb.after_iteration(bst, epoch, log)
    assert stop and (bst.best_iteration, bst.best_score) == (2, 1.5)
    out = cb.after_training(bst)
    assert out is not bst and out.num_boosted_rounds() == 3 and (out.best_iteration, out.best_score) == (2, 1.5)
    assert bytes(out.save_raw()) == bytes(_load(keep_rounds(raw, [0, 1, 2])).save_raw())
    assert bst.num_boosted_rounds() == 6


def test_history_restarts_in_before_training():
    cb = E.callback.EarlyStopping(1)
    m, stop = _drive(cb, [1.0, 2.0])
    assert stop == 1
    m, stop = _drive(cb, [5.0, 4.0, 3.0])      # a second train() call with the same callback
    assert stop is None and (m.best_iteration, m.best_score) == (2, 3.0)


def test_pickles_and_is_the_xgb_callback():
    from xgboost_ray_b200 import xgb
    assert xgb.xgboost.callback.EarlyStopping is E.EarlyStopping
    assert issubclass(E.EarlyStopping, E.TrainingCallback)
    cb = E.callback.EarlyStopping(2, metric_name="rmse", data_name="valid", maximize=False, save_best=True,
                                  min_delta=0.5)
    m, log = _Model(), {}
    cb.before_training(m)
    for epoch, v in enumerate([4.0, 3.0]):
        log.setdefault("valid", {}).setdefault("rmse", []).append(v)
        cb.after_iteration(m, epoch, log)
    p = pickle.loads(pickle.dumps(cb))            # mid-history: the copy continues where the original is
    assert vars(p) == vars(cb)
    for c in (cb, p):
        mm = _Model()
        mm.best_iteration, mm.best_score = m.best_iteration, m.best_score
        seen = dict(log, valid={"rmse": log["valid"]["rmse"] + [2.75]})
        assert c.after_iteration(mm, 2, seen) is False
        seen["valid"]["rmse"].append(2.9)
        assert c.after_iteration(mm, 3, seen) is True
        assert (mm.best_iteration, mm.best_score) == (1, 3.0)
