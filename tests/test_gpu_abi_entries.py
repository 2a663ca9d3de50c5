"""The C entries of prediction, called through ctypes: each refusal of B2_BoosterPredict, B2_BoosterPredictContribs and
B2_BoosterPredictLeaf matched against its whole message, which refusal wins when a call breaks two rules, and that an
edit of an existing tree (B2_BoosterSetTreeCategories, B2_BoosterSetTreeLeafVector) reaches every cached copy of the
model: the device node table, the TreeSHAP paths and the evaluation margins."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, F = 8, 3


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


def add_stump(eng, bst, feature, cond, values):
    """A root split on `feature` with two leaves of `values`; the leaves cover the same hessian."""
    topology = [np.asarray(a, np.int32) for a in ([1, -1, -1], [2, -1, -1], [-1, 0, 0], [feature, -1, -1])]
    cond_a, value_a = np.asarray([cond, 0, 0], np.float32), np.asarray([0, values[0], values[1]], np.float32)
    default_left, hess = np.asarray([1, 0, 0], np.uint8), np.asarray([2.0, 1.0, 1.0], np.float64)
    call(eng, "B2_BoosterAddTree", bst, 3, *(eng._ip(a) for a in topology), None, eng._fp(cond_a), eng._bp(default_left),
         eng._fp(value_a), None, None, hess.ctypes.data_as(eng._DP))


def categorical_stump(eng, handles, right_codes):
    bst = booster(eng, handles)
    add_stump(eng, bst, 0, 0.0, (-1.0, 1.0))
    set_categories(eng, bst, right_codes)
    return bst


def set_categories(eng, bst, right_codes):
    split_type = np.asarray([1, 0, 0], np.uint8)
    bits = np.zeros((3, 8), np.uint32)
    for c in right_codes:
        bits[0, c >> 5] |= np.uint32(1 << (c & 31))
    call(eng, "B2_BoosterSetTreeCategories", bst, 0, eng._bp(split_type), bits.ctypes.data_as(C.POINTER(C.c_uint32)))


def vector_stump(eng, handles, leaf_vec):
    bst = booster(eng, handles, "\nnum_target=2\nmulti_strategy=multi_output_tree")
    add_stump(eng, bst, 1, 0.5, (0.0, 0.0))
    set_leaf_vector(eng, bst, leaf_vec)
    return bst


def set_leaf_vector(eng, bst, leaf_vec):
    v = np.ascontiguousarray(leaf_vec, np.float32).reshape(-1)
    call(eng, "B2_BoosterSetTreeLeafVector", bst, 0, eng._fp(v), v.size)


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


def test_category_edit_reaches_every_cache(eng, handles):
    codes = features()[:, 0].astype(int)
    old, new = [1, 2], [0, 3]
    expect_old = np.where(np.isin(codes, old), 1.0, -1.0).astype(np.float32)
    bst = categorical_stump(eng, handles, old)
    m = matrix(eng, handles, label=expect_old)
    shap = np.zeros((N, F + 1), np.float32)
    # leaves of equal cover: the tree's expected value is 0, so feature 0's contribution is the whole prediction
    shap[:, 0] = expect_old
    np.testing.assert_array_equal(predict(eng, bst, m, N), expect_old)
    np.testing.assert_allclose(contribs(eng, bst, m, N * (F + 1)).reshape(N, F + 1), shap, atol=1e-6)
    np.testing.assert_array_equal(leaf(eng, bst, m, N), np.where(expect_old > 0, 2.0, 1.0))
    assert evaluate(eng, bst, m, "rmse") == 0.0
    set_categories(eng, bst, new)
    expect_new = -expect_old
    shap[:, 0] = expect_new
    np.testing.assert_array_equal(predict(eng, bst, m, N), expect_new)
    np.testing.assert_allclose(contribs(eng, bst, m, N * (F + 1)).reshape(N, F + 1), shap, atol=1e-6)
    np.testing.assert_array_equal(leaf(eng, bst, m, N), np.where(expect_new > 0, 2.0, 1.0))
    assert evaluate(eng, bst, m, "rmse") == pytest.approx(2.0, abs=1e-6)


def test_leaf_vector_edit_reaches_prediction(eng, handles):
    right = features()[:, 1] >= 0.5
    old = np.asarray([[0, 0], [1, 2], [3, 4]], np.float32)
    new = np.asarray([[0, 0], [-5, 6], [7, -8]], np.float32)
    bst = vector_stump(eng, handles, old)
    m = matrix(eng, handles)
    np.testing.assert_array_equal(predict(eng, bst, m, 2 * N).reshape(N, 2), np.where(right[:, None], old[2], old[1]))
    set_leaf_vector(eng, bst, new)
    np.testing.assert_array_equal(predict(eng, bst, m, 2 * N).reshape(N, 2), np.where(right[:, None], new[2], new[1]))
