"""CPU checks of the DART restatement (tests/dart_reference.py) and of the DART model file format."""
import copy
import json

import jsonschema
import numpy as np
import pytest

from tests import dart_reference as R
from tests.model_schema import GBTREE, MODEL, TREE
from tests.test_model_json import XGB_STYLE

DART = {
    "type": "object",
    "properties": {
        "name": {"const": "dart"},
        "gbtree": GBTREE,
        "weight_drop": {"type": "array", "items": {"type": "number"}},
    },
    "required": ["name", "gbtree", "weight_drop"],
    "additionalProperties": False,
}
DART_MODEL = copy.deepcopy(MODEL)
DART_MODEL["properties"]["learner"]["properties"]["gradient_booster"] = DART
assert TREE is GBTREE["properties"]["model"]["properties"]["trees"]["items"]


def test_normalisation_tree_by_hand():
    # eta 0.3, one new tree: lr = 0.3; two trees dropped: factor 2 / 2.3, new weight 1 / 2.3
    w = R.normalize([1.0, 1.0, 1.0], [0, 2], 0.3, 1, "tree")
    lr = float(np.float32(0.3))
    assert w.dtype == np.float32 and w.size == 4
    assert w[0] == np.float32(np.float32(1.0) * np.float32(2 / (2 + lr))) and w[1] == 1.0
    assert w[2] == w[0] and w[3] == np.float32(1 / (2 + lr))


def test_normalisation_forest_by_hand():
    w = R.normalize([0.5, 1.0], [0], 0.3, 1, "forest")
    f = np.float32(1 / (1 + float(np.float32(0.3))))
    assert list(w) == [np.float32(np.float32(0.5) * f), np.float32(1.0), f]


@pytest.mark.parametrize("normalize_type", ["tree", "forest"])
def test_normalisation_several_new_trees(normalize_type):
    # K = 3 classes x num_parallel_tree = 2: six new trees share lr = eta / 6
    w = R.normalize(np.ones(12, np.float32), [1, 4, 7], 0.6, 6, normalize_type)
    lr = float(np.float32(float(np.float32(0.6)) / 6))
    assert w.size == 18
    if normalize_type == "tree":
        f, new = np.float32(3 / (3 + lr)), np.float32(1 / (3 + lr))
    else:
        f = new = np.float32(1 / (1 + lr))
    assert all(w[t] == f for t in (1, 4, 7)) and all(w[12:] == new)
    assert all(w[t] == 1.0 for t in range(12) if t not in (1, 4, 7))


def test_nothing_dropped_gives_weight_one():
    assert list(R.normalize([0.25, 2.0], [], 0.3, 2)) == [0.25, 2.0, 1.0, 1.0]


def test_skip_drop_one_never_drops():
    for r in range(50):
        assert R.drop_set(np.ones(20), r, seed=3, rate_drop=1.0, skip_drop=1.0, one_drop=1) == []


def test_rate_drop_one_drops_all():
    for r in range(20):
        assert R.drop_set(np.ones(15), r, seed=1, rate_drop=1.0) == list(range(15))


@pytest.mark.parametrize("sample_type", ["uniform", "weighted"])
def test_one_drop_yields_exactly_one(sample_type):
    w = np.linspace(0.2, 1.0, 30).astype(np.float32)
    for r in range(40):
        assert len(R.drop_set(w, r, seed=5, rate_drop=0.0, one_drop=1, sample_type=sample_type)) == 1


def test_equal_weights_make_weighted_uniform():
    w = np.full(40, 0.37, np.float32)
    for r in range(30):
        assert (R.drop_set(w, r, seed=9, rate_drop=0.2, sample_type="weighted", one_drop=1)
                == R.drop_set(w, r, seed=9, rate_drop=0.2, sample_type="uniform", one_drop=1))


def test_draw_depends_only_on_seed_round_and_weights():
    w = np.linspace(0.5, 1.5, 25).astype(np.float32)
    a = [R.drop_set(w, r, seed=11, rate_drop=0.3, sample_type="weighted") for r in range(10)]
    assert a == [R.drop_set(w.copy(), r, seed=11, rate_drop=0.3, sample_type="weighted") for r in range(10)]
    assert a != [R.drop_set(w, r, seed=12, rate_drop=0.3, sample_type="weighted") for r in range(10)]
    # the draw of tree t does not depend on how many trees follow it (uniform)
    for r in range(10):
        short = R.drop_set(w[:10], r, seed=11, rate_drop=0.3)
        assert short == [t for t in R.drop_set(w, r, seed=11, rate_drop=0.3) if t < 10]


def test_drop_rate_is_about_right():
    n = sum(len(R.drop_set(np.ones(100), r, seed=0, rate_drop=0.1)) for r in range(100))
    assert 800 < n < 1200


def test_margins_ordered_weighted_sum():
    # two stumps on feature 0 (split bin 1) and a categorical stump on feature 1 (codes {2} go right)
    stump = dict(left=np.array([1, -1, -1]), right=np.array([2, -1, -1]), split_feature=np.array([0, -1, -1]),
                 split_bin=np.array([1, -1, -1]), default_left=np.array([1, 0, 0], np.uint8),
                 value=np.array([0, -0.5, 0.25], np.float32), split_type=np.zeros(3, np.uint8),
                 cat_bits=np.zeros((3, 8), np.uint32))
    cat = dict(stump, split_feature=np.array([1, -1, -1]), split_type=np.array([1, 0, 0], np.uint8),
               cat_bits=np.zeros((3, 8), np.uint32), value=np.array([0, 1.0, 3.0], np.float32))
    cat["cat_bits"][0, 0] = 1 << 2
    bins = np.array([[0, 2], [2, 0], [255, 255]], np.uint8)
    hm = np.array([1, 0], np.uint8)
    w = np.array([0.5, 2.0, 1.0], np.float32)
    m = R.margins([stump, stump, cat], w, bins, hm, np.full(3, 0.1, np.float32))
    # row 0: left, left, code 2 -> right; row 1: right, right, left; row 2: missing -> default left; code 255 -> left
    want = [[0.1 + 0.5 * -0.5 + 2 * -0.5 + 3.0], [0.1 + 0.5 * 0.25 + 2 * 0.25 + 1.0], [0.1 + 0.5 * -0.5 + 2 * -0.5 + 1.0]]
    assert np.allclose(m, want, atol=1e-6)
    d = R.margins([stump, stump, cat], w, bins, hm, np.full(3, 0.1, np.float32), skip=[1])
    assert np.allclose(d[:, 0], m[:, 0] - 2.0 * np.array([-0.5, 0.25, -0.5]), atol=1e-6)


DART_STYLE = copy.deepcopy(XGB_STYLE)
DART_STYLE["learner"]["gradient_booster"] = {"name": "dart", "gbtree": XGB_STYLE["learner"]["gradient_booster"],
                                             "weight_drop": [0.75, 1.25]}


def test_hand_written_dart_file_loads_and_round_trips(tmp_path):
    from xgboost_ray_b200 import engine as E
    jsonschema.validate(DART_STYLE, DART_MODEL)
    f = str(tmp_path / "dart.json")
    json.dump(DART_STYLE, open(f, "w"))
    b = E.Booster(model_file=f)
    assert b.is_dart and b.num_trees() == 2
    assert list(b.get_tree_weights()) == [0.75, 1.25]
    raw = bytes(b.save_raw())
    d = json.loads(raw.decode())
    jsonschema.validate(d, DART_MODEL)
    assert d["learner"]["gradient_booster"]["weight_drop"] == [0.75, 1.25]
    b2 = E.Booster()
    b2.load_model(raw)
    assert bytes(b2.save_raw()) == raw
    cfg = json.loads(b2.save_config())
    assert cfg["learner"]["gradient_booster"]["name"] == "dart"
    assert cfg["learner"]["gradient_booster"]["dart_train_param"]["sample_type"] == "uniform"


def test_weight_count_must_match_trees(tmp_path):
    from xgboost_ray_b200 import engine as E
    bad = copy.deepcopy(DART_STYLE)
    bad["learner"]["gradient_booster"]["weight_drop"] = [1.0]
    with pytest.raises(E.XGBoostError, match="weight_drop"):
        E.Booster().load_model(json.dumps(bad).encode())


def test_booster_kinds():
    from xgboost_ray_b200 import engine as E
    assert E.Booster({"booster": "dart"}).is_dart
    with pytest.raises(E.XGBoostError, match="gblinear"):
        E.Booster({"booster": "gblinear"})


def test_sklearn_takes_the_dart_parameters():
    from xgboost_ray_b200.sklearn import RayXGBRegressor
    r = RayXGBRegressor(booster="dart", rate_drop=0.1, skip_drop=0.5, sample_type="weighted", normalize_type="forest",
                        one_drop=1)
    p = r.get_xgb_params()
    assert p["booster"] == "dart" and p["rate_drop"] == 0.1 and p["one_drop"] == 1
    assert p["sample_type"] == "weighted" and p["normalize_type"] == "forest" and p["skip_drop"] == 0.5
    assert r.get_params()["booster"] == "dart"


@pytest.mark.parametrize("objective,extra", [("reg:squarederror", {}), ("binary:logistic", {"subsample": 0.8}),
                                             ("multi:softprob", {"num_class": 3, "colsample_bynode": 0.6})])
def test_nothing_dropped_is_the_oracle_gbtree_model(oracle, objective, extra):
    """rate_drop = 0: every weight is 1 and fl(1 * v) = v, so the reference grows the oracle's own gbtree model."""
    rng = np.random.RandomState(0)
    X = rng.uniform(0, 10, size=(3000, 6)).astype(np.float32)
    X[rng.uniform(size=X.shape) < 0.03] = np.nan
    z = np.nan_to_num(X[:, 0]) + np.sin(np.nan_to_num(X[:, 1])) * 2 + rng.normal(scale=0.3, size=3000)
    y = {"reg:squarederror": z, "binary:logistic": z > np.median(z),
         "multi:softprob": np.digitize(z, np.quantile(z, [1 / 3, 2 / 3]))}[objective].astype(np.float32)
    params = dict({"objective": objective, "max_depth": 4, "base_score": 0.5, "seed": 3}, **extra)
    ref = R.train(oracle, dict(params, booster="dart", rate_drop=0.0), X, y, 6)
    ob, _ = oracle.train(params, X, y, 6)
    assert all(d == [] for d in ref.drops) and list(ref.weights) == [1.0] * ob.num_trees
    assert ref.num_trees == ob.num_trees
    for i in range(ob.num_trees):
        t, o = ref.bst.tree(i), ob.tree(i)
        for k in ("left", "split_feature", "split_bin", "default_left", "value", "loss_chg"):
            assert np.array_equal(getattr(t, k), getattr(o, k)), (i, k)
    assert ref.margin().tobytes() == ob.margin.tobytes()


def test_dropping_rounds_grow_from_the_drop_margin(oracle):
    """With drops, round r's trees are the oracle's trees for gradients at the drop margin: growing one more oracle round
    by hand from the reference's drop margin gives the same tree."""
    rng = np.random.RandomState(1)
    X = rng.uniform(0, 10, size=(2000, 5)).astype(np.float32)
    y = (X[:, 0] + rng.normal(size=2000)).astype(np.float32)
    params = {"booster": "dart", "objective": "reg:squarederror", "max_depth": 3, "base_score": 0.5, "rate_drop": 0.5,
              "seed": 2}
    ref = R.train(oracle, params, X, y, 8)
    assert sum(1 for d in ref.drops if d) >= 4
    last = ref.drops[-1]
    w7 = R.replay_weights(7, 0.3, 1, seed=2, rate_drop=0.5)[0]
    assert np.array_equal(ref.weights[:8], R.normalize(w7, last, 0.3, 1)[:8])
    m = R.margins(ref.trees()[:7], w7, ref.bins, ref.has_missing, ref.base, skip=last)
    g, h = oracle.gradients("reg:squarederror", m, y)
    cuts = oracle.Cuts.from_data(X, 256)
    solo = oracle.Booster({"objective": "reg:squarederror", "max_depth": 3, "base_score": 0.5, "seed": 2}, cuts)
    for i in range(7):   # the same tree count, so that sampling seeds (none here) and ids line up
        solo.boost(ref.bins, y, custom_g=np.zeros_like(g), custom_h=np.ones_like(h))
    solo.boost(ref.bins, y, custom_g=g, custom_h=h)
    t, o = ref.tree(7), solo.tree(7)
    assert np.array_equal(t.split_feature, o.split_feature) and np.array_equal(t.value, o.value)


def test_a_dart_model_does_not_continue_as_gbtree():
    from xgboost_ray_b200 import engine as E
    src = E.Booster()
    src.load_model(json.dumps(DART_STYLE).encode())
    with pytest.raises(E.XGBoostError, match="DART"):
        E.train({"booster": "gbtree"}, None, num_boost_round=1, xgb_model=src, verbose_eval=False)
