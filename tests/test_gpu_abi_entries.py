"""The C entries of prediction and of the tree record, called through ctypes: each refusal of B2_BoosterPredict,
B2_BoosterPredictContribs, B2_BoosterPredictLeaf and B2_BoosterAddTree matched against its whole message, which refusal
wins when a call breaks two rules, a categorical and a vector-leaf tree added whole through B2_BoosterAddTree in every
prediction mode, and malformed model files refused before any tree walk."""
import ctypes as C
import json

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, F = 8, 3
VECTOR = "\nnum_target=2\nmulti_strategy=multi_output_tree"   # booster() params of a two-target vector-leaf model


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


@pytest.fixture
def handles(eng):
    """Matrices and boosters created by a test, freed when it ends."""
    made = []
    yield made
    for kind, h in reversed(made):
        getattr(eng.lib(), "B2_BoosterFree" if kind == "booster" else "B2_MatrixFree")(h)


def call(eng, fn, *args):
    eng._check(getattr(eng.lib(), fn)(*args))


def features(cols=F):
    X = np.random.RandomState(0).uniform(0, 1, size=(N, cols)).astype(np.float32)
    X[:, 0] = np.arange(N) % 4   # category codes 0..3
    return X


def matrix(eng, handles, cols=F, keep_raw=True, base_margin=None, label=None):
    X = features(cols)
    h = eng._H(0)
    call(eng, "B2_MatrixCreateFromDense", eng._fp(X), N, cols, float("nan"), eng._default_device(), C.byref(h))
    handles.append(("matrix", h.value))
    for field, v in (("base_margin", base_margin), ("label", label)):
        if v is not None:
            v = np.ascontiguousarray(v, np.float32)
            call(eng, "B2_MatrixSetFloatInfo", h.value, field.encode(), eng._fp(v), v.size)
    if not keep_raw:
        call(eng, "B2_MatrixQuantize", h.value, 0, 256, 0, 0)
    return h.value


def booster(eng, handles, extra=""):
    """A prediction-only booster over F features with base_score 0, so that a margin is the sum of the leaves."""
    h = eng._H(0)
    text = "num_feature=%d\nbase_score=0\ndevice=%d%s" % (F, eng._default_device(), extra)
    call(eng, "B2_BoosterCreate", text.encode(), 0, 0, C.byref(h))
    handles.append(("booster", h.value))
    return h.value


def stump(feature, cond, values, right_codes=None, leaf_vector=None):
    """A root split on `feature` with two leaves of `values`, as a tree dict; the leaves cover the same hessian.  With
    right_codes the split is categorical: those category codes go right."""
    t = dict(left=[1, -1, -1], right=[2, -1, -1], parent=[-1, 0, 0], split_feature=[feature, -1, -1],
             split_bin=[-1, -1, -1], split_cond=[cond, 0, 0], default_left=[1, 0, 0], value=[0, values[0], values[1]],
             base_weight=[0, 0, 0], loss_chg=[0, 0, 0], sum_hess=[2.0, 1.0, 1.0], leaf_vector=leaf_vector)
    if right_codes is not None:
        t["split_type"] = np.asarray([1, 0, 0], np.uint8)
        t["cat_bits"] = np.zeros((3, 8), np.uint32)
        for c in right_codes:
            t["cat_bits"][0, c >> 5] |= np.uint32(1 << (c & 31))
    return t


def add_tree(eng, bst, t):
    rec, _arrays = eng.B2Tree.of(t)
    call(eng, "B2_BoosterAddTree", bst, C.byref(rec))


def categorical_stump(eng, handles, right_codes):
    bst = booster(eng, handles)
    add_tree(eng, bst, stump(0, 0.0, (-1.0, 1.0), right_codes=right_codes))
    return bst


def vector_stump(eng, handles, leaf_vec):
    bst = booster(eng, handles, VECTOR)
    add_tree(eng, bst, stump(1, 0.5, (0.0, 0.0), leaf_vector=leaf_vec))
    return bst


def predict(eng, bst, m, out_len, tree_begin=0, tree_end=0):
    out = np.zeros(max(out_len, 1), np.float32)
    call(eng, "B2_BoosterPredict", bst, m, 1, tree_begin, tree_end, eng._fp(out), out_len)
    return out[:out_len]


def contribs(eng, bst, m, out_len, interactions=0, tree_begin=0, tree_end=0):
    out = np.zeros(max(out_len, 1), np.float32)
    call(eng, "B2_BoosterPredictContribs", bst, m, tree_begin, tree_end, interactions, eng._fp(out), out_len)
    return out[:out_len]


def leaf(eng, bst, m, out_len, tree_begin=0, tree_end=0):
    out = np.zeros(max(out_len, 1), np.float32)
    call(eng, "B2_BoosterPredictLeaf", bst, m, tree_begin, tree_end, eng._fp(out), out_len)
    return out[:out_len]


def evaluate(eng, bst, m, metric):
    v = C.c_double(0)
    call(eng, "B2_BoosterEvalSet", bst, m, metric.encode(), C.byref(v))
    return v.value


def refused(eng, fn, *args):
    with pytest.raises(eng.XGBoostError) as e:
        fn(eng, *args)
    return str(e.value)


NO_RAW = "prediction matrix has no raw data on the device (B2_MatrixEnsureRaw)"
MISMATCH = "feature count mismatch: matrix has 4, model has 3"
RANGE = "invalid tree range [2, 1)"
BASE_MARGIN = "base_margin has 16 values, expected 8"


def test_predict_refusals(eng, handles):
    bst = categorical_stump(eng, handles, [1])
    m = matrix(eng, handles)
    assert refused(eng, predict, bst, m, N - 1) == "output buffer has 7 values, expected 8"
    assert refused(eng, predict, bst, matrix(eng, handles, keep_raw=False), N) == NO_RAW
    assert refused(eng, predict, bst, matrix(eng, handles, cols=4), N) == MISMATCH
    assert refused(eng, predict, bst, m, N, 2) == RANGE
    assert refused(eng, predict, bst, matrix(eng, handles, base_margin=np.zeros(2 * N)), N) == BASE_MARGIN


def test_contribs_refusals(eng, handles):
    bst = categorical_stump(eng, handles, [1])
    m = matrix(eng, handles)
    assert refused(eng, contribs, bst, m, N * (F + 1) - 1) == "output buffer has 31 values, expected 32"
    assert refused(eng, contribs, bst, m, N * (F + 1) ** 2 + 1, 1) == "output buffer has 129 values, expected 128"
    assert refused(eng, contribs, bst, matrix(eng, handles, keep_raw=False), N * (F + 1)) == NO_RAW
    assert refused(eng, contribs, bst, matrix(eng, handles, cols=4), N * 5) == MISMATCH
    assert refused(eng, contribs, bst, m, N * (F + 1), 0, 2) == RANGE
    assert refused(eng, contribs, bst, matrix(eng, handles, base_margin=np.zeros(2 * N)), N * (F + 1)) == BASE_MARGIN
    vec = vector_stump(eng, handles, np.zeros((3, 2)))
    assert refused(eng, contribs, vec, m, N * 2 * (F + 1)) == (
        "pred_contribs is not supported for vector-leaf trees (multi_strategy=multi_output_tree)")
    assert refused(eng, contribs, vec, m, N * 2 * (F + 1) ** 2, 1) == (
        "pred_interactions is not supported for vector-leaf trees (multi_strategy=multi_output_tree)")


def test_leaf_refusals(eng, handles):
    bst = categorical_stump(eng, handles, [1])
    m = matrix(eng, handles)
    assert refused(eng, leaf, bst, m, N + 1) == "output buffer has 9 values, expected 8"
    assert refused(eng, leaf, bst, matrix(eng, handles, keep_raw=False), N) == NO_RAW
    assert refused(eng, leaf, bst, matrix(eng, handles, cols=4), N) == MISMATCH
    assert refused(eng, leaf, bst, m, N, 2) == RANGE
    assert refused(eng, leaf, bst, matrix(eng, handles, base_margin=np.zeros(2 * N)), N) == BASE_MARGIN


def test_negative_base_margin_length_sets_none(eng, handles):
    """B2_MatrixSetFloatInfo takes base_margin of length -N (a multiple of N rows) as no base_margin; a later valid
    one is copied in full."""
    bst = categorical_stump(eng, handles, [1])
    m = matrix(eng, handles)
    plain = predict(eng, bst, m, N)
    v = np.full(N, 0.5, np.float32)
    call(eng, "B2_MatrixSetFloatInfo", m, b"base_margin", eng._fp(v), -N)
    np.testing.assert_array_equal(predict(eng, bst, m, N), plain)
    call(eng, "B2_MatrixSetFloatInfo", m, b"base_margin", eng._fp(v), N)
    np.testing.assert_array_equal(predict(eng, bst, m, N), plain + 0.5)


def test_precedence(eng, handles):
    """A call that breaks two rules reports the one its entry checks first."""
    bst = categorical_stump(eng, handles, [1])
    no_raw = matrix(eng, handles, keep_raw=False)
    bad_margin = matrix(eng, handles, base_margin=np.zeros(2 * N))
    # predict: the output length before the matrix, the tree range before the base_margin
    assert refused(eng, predict, bst, no_raw, N + 1) == "output buffer has 9 values, expected 8"
    assert refused(eng, predict, bst, bad_margin, N, 2) == RANGE
    # contributions: the vector-leaf model before the output length, the output length before the matrix
    vec = vector_stump(eng, handles, np.zeros((3, 2)))
    assert refused(eng, contribs, vec, no_raw, 1) == (
        "pred_contribs is not supported for vector-leaf trees (multi_strategy=multi_output_tree)")
    assert refused(eng, contribs, bst, no_raw, 1) == "output buffer has 1 values, expected 32"
    # leaf indices: the matrix and the tree range before the output length (which the range sets)
    assert refused(eng, leaf, bst, no_raw, 1) == NO_RAW
    assert refused(eng, leaf, bst, matrix(eng, handles), 1, 2) == RANGE


def test_categorical_stump_in_every_prediction_mode(eng, handles):
    codes = features()[:, 0].astype(int)
    expect = np.where(np.isin(codes, [1, 2]), 1.0, -1.0).astype(np.float32)
    bst = categorical_stump(eng, handles, [1, 2])
    m = matrix(eng, handles, label=expect)
    shap = np.zeros((N, F + 1), np.float32)
    # leaves of equal cover: the tree's expected value is 0, so feature 0's contribution is the whole prediction
    shap[:, 0] = expect
    np.testing.assert_array_equal(predict(eng, bst, m, N), expect)
    np.testing.assert_allclose(contribs(eng, bst, m, N * (F + 1)).reshape(N, F + 1), shap, atol=1e-6)
    np.testing.assert_array_equal(leaf(eng, bst, m, N), np.where(expect > 0, 2.0, 1.0))
    assert evaluate(eng, bst, m, "rmse") == 0.0


def test_vector_stump_prediction(eng, handles):
    right = features()[:, 1] >= 0.5
    vec = np.asarray([[0, 0], [1, 2], [3, 4]], np.float32)
    bst = vector_stump(eng, handles, vec)
    m = matrix(eng, handles)
    np.testing.assert_array_equal(predict(eng, bst, m, 2 * N).reshape(N, 2), np.where(right[:, None], vec[2], vec[1]))


def blank(n, vector=False):
    """Zeroed arrays for B2_BoosterGetTree to fill, as Booster.get_tree allocates them."""
    t = {k: np.zeros(n, np.int32) for k in ("left", "right", "parent", "split_feature", "split_bin")}
    t.update({k: np.zeros(n, np.float32) for k in ("split_cond", "value", "base_weight", "loss_chg")})
    t.update(default_left=np.zeros(n, np.uint8), sum_hess=np.zeros(n), split_type=np.zeros(n, np.uint8),
             cat_bits=np.zeros((n, 8), np.uint32), leaf_vector=np.zeros((n, 2), np.float32) if vector else None)
    return t


def get_tree(eng, bst, t):
    rec, _arrays = eng.B2Tree.of(t)
    call(eng, "B2_BoosterGetTree", bst, 0, C.byref(rec))
    return t


def test_get_tree_fills_the_record(eng, handles):
    """B2_BoosterGetTree returns a tree as it was added, into buffers of its node count and leaf vector length."""
    vec = np.arange(6, dtype=np.float32).reshape(3, 2)
    cat, cat_tree = categorical_stump(eng, handles, [1, 200]), stump(0, 0.0, (-1.0, 1.0), right_codes=[1, 200])
    vector, vector_tree = vector_stump(eng, handles, vec), stump(1, 0.5, (0.0, 0.0), leaf_vector=vec)
    for bst, want in ((cat, cat_tree), (vector, vector_tree)):
        got = get_tree(eng, bst, blank(3, vector=want["leaf_vector"] is not None))
        for k, v in got.items():
            if v is not None:
                np.testing.assert_array_equal(v, want[k] if want.get(k) is not None else 0, err_msg=k)
    assert refused(eng, get_tree, cat, blank(4)) == "tree buffers have 4 nodes, tree 0 has 3"
    assert refused(eng, get_tree, cat, blank(3, vector=True)) == "leaf vector buffer has 6 values, tree 0 has 0"
    assert refused(eng, get_tree, vector, blank(3)) == "leaf vector buffer has 0 values, tree 0 has 6"


def refused_tree(eng, bst, t):
    """The message B2_BoosterAddTree refuses tree t with; the model keeps the trees it had."""
    before = C.c_int32(0)
    call(eng, "B2_BoosterNumTrees", bst, C.byref(before))
    with pytest.raises(eng.XGBoostError) as e:
        add_tree(eng, bst, t)
    after = C.c_int32(0)
    call(eng, "B2_BoosterNumTrees", bst, C.byref(after))
    assert after.value == before.value
    return str(e.value)


def edited(t, **fields):
    return dict(t, **{k: np.asarray(v) for k, v in fields.items()})


def test_add_tree_refuses_no_nodes(eng, handles):
    bst = booster(eng, handles)
    empty = {k: np.zeros(0) for k in stump(0, 0.5, (1, 2))}
    assert refused_tree(eng, bst, dict(empty, leaf_vector=None)) == "tree 0 has no nodes"


def test_add_tree_refuses_child_outside_the_tree(eng, handles):
    bst = booster(eng, handles)
    t = stump(1, 0.5, (1.0, 2.0))
    assert refused_tree(eng, bst, edited(t, right=[-5, -1, -1])) == "tree 0 node 0 has child -5 outside [0, 3)"
    add_tree(eng, bst, t)   # a refused tree is named by the index it would have had in the model
    assert refused_tree(eng, bst, edited(t, left=[3, -1, -1])) == "tree 1 node 0 has child 3 outside [0, 3)"


def test_add_tree_refuses_a_split_reached_twice(eng, handles):
    bst = booster(eng, handles)
    t = stump(1, 0.5, (1.0, 2.0))
    assert refused_tree(eng, bst, edited(t, left=[0, -1, -1])) == "tree 0 node 0 splits and is reached twice from the root"
    # a shared subtree: both children of the root are split node 1
    shared = dict(left=[1, 2, -1, -1], right=[1, 3, -1, -1], parent=[-1, 0, 1, 1], split_feature=[1, 2, -1, -1],
                  split_bin=[-1] * 4, split_cond=[0.5, 0.5, 0, 0], default_left=[0] * 4, value=[0, 0, 1, 2],
                  base_weight=[0] * 4, loss_chg=[0] * 4, sum_hess=[1.0] * 4)
    assert refused_tree(eng, bst, shared) == "tree 0 node 1 splits and is reached twice from the root"
    # a leaf shared by two splits, and a node the root does not reach (xgboost's deleted nodes), are walked safely
    add_tree(eng, bst, edited(t, right=[1, -1, -1]))
    np.testing.assert_array_equal(predict(eng, bst, matrix(eng, handles), N), np.ones(N, np.float32))


def test_add_tree_refuses_a_feature_outside_the_model(eng, handles):
    bst = booster(eng, handles)
    assert refused_tree(eng, bst, stump(F, 0.5, (1.0, 2.0))) == "tree 0 node 0 splits on feature 3; the model has 3 features"


def test_add_tree_refuses_a_categorical_leaf(eng, handles):
    bst = booster(eng, handles)
    t = stump(0, 0.0, (-1.0, 1.0), right_codes=[1])
    assert refused_tree(eng, bst, edited(t, split_type=np.asarray([1, 0, 1], np.uint8))) == (
        "tree 0 node 2 is a leaf with split_type 1 (categorical)")


def test_add_tree_refuses_a_leaf_vector_on_a_single_output_booster(eng, handles):
    bst = booster(eng, handles)
    assert refused_tree(eng, bst, stump(1, 0.5, (0.0, 0.0), leaf_vector=np.zeros((3, 2)))) == (
        "tree 0 is a vector-leaf tree (multi_strategy=multi_output_tree); this booster grows single-output trees "
        "(multi_strategy=one_output_per_tree, 1 target(s)): a model keeps the strategy it was trained with")


def test_add_tree_refuses_a_missing_leaf_vector(eng, handles):
    bst = booster(eng, handles, VECTOR)
    assert refused_tree(eng, bst, stump(1, 0.5, (1.0, 2.0))) == (
        "tree 0 is a single-output tree (multi_strategy=one_output_per_tree); this booster grows vector-leaf trees "
        "(multi_strategy=multi_output_tree): a model keeps the strategy it was trained with")


def test_add_tree_refuses_a_leaf_vector_of_the_wrong_length(eng, handles):
    bst = booster(eng, handles, VECTOR)
    assert refused_tree(eng, bst, stump(1, 0.5, (0.0, 0.0), leaf_vector=np.zeros(5))) == (
        "tree 0 has a leaf vector of 5 values; it needs 6 (3 nodes x 2 targets)")
    assert refused_tree(eng, bst, stump(1, 0.5, (0.0, 0.0), leaf_vector=np.zeros((3, 3)))) == (
        "tree 0 has a leaf vector of 9 values; it needs 6 (3 nodes x 2 targets)")


@pytest.mark.parametrize("children, message", [
    ({"right_children": [-5, -1, -1]}, "tree 0 node 0 has child -5 outside [0, 3)"),
    ({"left_children": [0, -1, -1]}, "tree 0 node 0 splits and is reached twice from the root"),
])
def test_malformed_model_file_refused(eng, tmp_path, children, message):
    """A model file whose tree walk would leave the tree or never end is refused when the predictor is built, before
    any kernel walks it; so is every later prediction."""
    from tests.model_files import xgb_model_file
    doc = json.loads(xgb_model_file(1, n_features=F))
    doc["learner"]["gradient_booster"]["model"]["trees"][0].update(children)
    path = str(tmp_path / "model.json")
    with open(path, "w") as f:
        json.dump(doc, f)
    bst = eng.Booster(model_file=path)
    for _ in range(2):
        with pytest.raises(eng.XGBoostError) as e:
            bst.predict(eng.DMatrix(features()))
        assert str(e.value) == message
