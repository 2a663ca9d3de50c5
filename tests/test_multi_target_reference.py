"""CPU side of multi-target regression / multi-label classification: the reference of tests/multi_target_reference.py
against the oracle and hand-computed answers, RayDMatrix with a label of several columns (2-D array, DataFrame, list of
columns; the multi-label Parquet cases of xgboost_ray/tests/test_matrix.py:294-341), the model file and the sklearn
label rules."""
import copy
import json

import numpy as np
import pytest

from tests import multi_target_reference as R
from tests import objective_reference as O
from xgboost_ray_b200.matrix import RayDMatrix, RayShardingMode, combine_data

F32 = np.float32


def _data(n=600, f=5, T=3, seed=0, binary=False):
    rng = np.random.RandomState(seed)
    X = rng.uniform(0, 10, (n, f)).astype(F32)
    Y = np.stack([X[:, k] * 0.5 + np.sin(X[:, k + 1]) + rng.normal(0, 0.2, n) for k in range(T)], axis=1).astype(F32)
    if binary:
        Y = (Y > np.median(Y, axis=0)).astype(F32)
    return X, Y


@pytest.mark.parametrize("obj", ["reg:squarederror", "binary:logistic"])
def test_tree_k_of_round_r_is_the_single_target_oracle_model_of_column_k(oracle, obj):
    X, Y = _data(binary=obj == "binary:logistic")
    params = {"objective": obj, "max_depth": 4, "eta": 0.3, "base_score": 0.5}
    ref = R.train(oracle, params, X, Y, 3)
    T = Y.shape[1]
    for k in range(T):
        single, _ = oracle.train(params, X, Y[:, k], 3)
        for r in range(3):
            a, b = ref.tree(r * T + k), single.tree(r)
            for f in ("left", "split_feature", "split_bin", "value", "loss_chg"):
                assert getattr(a, f).tobytes() == getattr(b, f).tobytes(), (k, r, f)


@pytest.mark.parametrize("obj", R.MULTI_TARGET_OBJECTIVES)
def test_gradients_are_the_single_target_sequence_per_column(oracle, obj):
    X, Y = _data(n=300, binary=obj in ("binary:logistic", "binary:logitraw", "reg:logistic"))
    if obj == "reg:squaredlogerror":
        Y = np.abs(Y)
    m = np.random.RandomState(1).normal(0, 1, Y.shape).astype(F32)
    w = np.random.RandomState(2).uniform(0.5, 2, len(Y)).astype(F32)
    params = {"objective": obj, "scale_pos_weight": 1.5}
    g, h, _ = R.column_gradients(params, m, Y, w)
    for k in range(Y.shape[1]):
        if obj in ("reg:squarederror", "binary:logistic"):
            og, oh = oracle.gradients(obj, m[:, k].copy(), Y[:, k], w if obj == "reg:squarederror" else
                                      np.where(Y[:, k] == 1, w * F32(1.5), w).astype(F32))
            og, oh = og.reshape(-1), oh.reshape(-1)
        else:
            og, oh, _ = O.gradients(params, m[:, k], Y[:, k], w)
        assert g[:, k].tobytes() == og.tobytes() and h[:, k].tobytes() == oh.tobytes()


def test_intercept_hand_cases_and_one_column():
    # constant columns: stump_k = c_k exactly, the intercept is the binary32 sum of c_k / T in k order
    Y = np.tile(np.array([1.0, 2.0, 4.5], F32), (8, 1))
    assert R.intercept({"objective": "reg:squarederror"}, Y) == float(F32(F32(F32(1 / 3) + F32(2 / 3)) + F32(1.5)))
    # weights enter the stump of every column the same way
    w = np.array([1, 3] * 4, F32)
    Y2 = np.stack([np.array([0, 4] * 4, F32), np.array([2, 2] * 4, F32)], axis=1)
    assert R.intercept({"objective": "reg:squarederror"}, Y2, w) == float(F32(F32(3.0 / 2) + F32(2.0 / 2)))
    # one column: today's estimate, bit for bit
    X, Y = _data(T=1, seed=3)
    for obj in ("reg:pseudohubererror", "reg:squaredlogerror", "reg:logistic"):
        y = np.abs(Y) if obj == "reg:squaredlogerror" else (Y > np.median(Y)).astype(F32) if obj == "reg:logistic" else Y
        assert F32(R.intercept({"objective": obj}, y)) == F32(O.estimate_base_score({"objective": obj}, y[:, 0]))
    # binary:logistic: the sigmoid of the mean stump
    L = np.array([[1, 0], [1, 0], [1, 1], [0, 1]], F32)
    v = R.intercept({"objective": "binary:logistic"}, L)
    assert 0.5 < v < 0.7


def test_elementwise_metric_formulas():
    m = np.array([[1.0, 2.0], [3.0, 5.0]], F32)
    y = np.array([[1.5, 2.0], [2.0, 4.0]], F32)
    w = np.array([1.0, 3.0], F32)
    # rmse: sqrt(sum_i w_i sum_k d_ik^2 / (T sum w))
    want = np.sqrt((1 * (0.25 + 0) + 3 * (1 + 1)) / (2 * 4.0))
    assert R.metric("rmse", "reg:squarederror", m, y, w) == pytest.approx(want, rel=1e-12)
    assert R.metric("mae", "reg:squarederror", m, y) == pytest.approx((0.5 + 0 + 1 + 1) / 4, rel=1e-12)
    L = np.array([[1, 0], [0, 1]], F32)
    z = np.array([[2.0, -1.0], [0.5, -3.0]], F32)
    assert R.metric("error", "binary:logistic", z, L) == pytest.approx(2 / 4)
    p = 1 / (1 + np.exp(-z.astype(np.float64)))
    ll = -(L * np.log(p) + (1 - L) * np.log(1 - p)).mean()
    assert R.metric("logloss", "binary:logistic", z, L) == pytest.approx(ll, rel=1e-6)


def test_raydmatrix_label_forms_and_shard_reassembly(tmp_path):
    import pandas as pd
    X, Y = _data(n=41)
    df = pd.DataFrame(np.column_stack([X, Y]), columns=["a", "b", "c", "d", "e", "y0", "y1", "y2"])
    for data, label in ((X, Y), (X, pd.DataFrame(Y)), (df, ["y0", "y1", "y2"]), (df, ["y2", "y0"])):
        want = Y if not isinstance(label, list) else df[label].values.astype(F32)
        want_x = X if not isinstance(label, list) else df.drop(columns=label).values.astype(F32)
        for mode in (RayShardingMode.INTERLEAVED, RayShardingMode.BATCH):
            for w in (1, 2, 3):
                m = RayDMatrix(data, label, sharding=mode)
                m.load_data(w)
                parts = [m.get_data(r, w) for r in range(w)]
                assert all(p["label"].ndim == 2 and p["label"].shape[1] == want.shape[1] for p in parts)
                assert np.array_equal(combine_data(mode, [p["label"] for p in parts]), want)
                assert np.array_equal(combine_data(mode, [p["data"] for p in parts]), want_x)
        if isinstance(label, list):
            assert m._columns == ["a", "b", "c", "d", "e"] + [c for c in ["y0", "y1", "y2"] if c not in label]


@pytest.mark.parametrize("two_files", [False, True])
@pytest.mark.parametrize("distributed", [False, True])
def test_parquet_multi_label(tmp_path, two_files, distributed):
    """xgboost_ray/tests/test_matrix.py:294-341: Parquet with four label columns, one file and two files, central and
    distributed loading."""
    import pandas as pd
    rng = np.random.RandomState(4)
    x = rng.uniform(size=(32, 4)).astype(F32)
    multi_y = rng.randint(0, 2, size=(32, 4)).astype(F32)
    df = pd.DataFrame(x, columns=["a", "b", "c", "d"])
    labels = ["label_%d" % k for k in range(4)]
    df[labels] = multi_y
    if two_files:
        files = [str(tmp_path / "data_1.parquet"), str(tmp_path / "data_2.parquet")]
        df[:16].to_parquet(files[0])
        df[16:].to_parquet(files[1])
        src = files
    else:
        src = str(tmp_path / "data.parquet")
        df.to_parquet(src)
    for w in ((1, 2) if (two_files or not distributed) else (1,)):
        m = RayDMatrix(src, labels, distributed=distributed)
        m.load_data(w)
        parts = [m.get_data(r, w) for r in range(w)]
        got_y = np.concatenate([p["label"] for p in parts]) if m.sharding == RayShardingMode.FIXED else \
            combine_data(m.sharding, [p["label"] for p in parts])
        got_x = np.concatenate([np.concatenate(p["data"]) if isinstance(p["data"], list) else p["data"]
                                for p in parts]) if m.sharding == RayShardingMode.FIXED else \
            combine_data(m.sharding, [p["data"] for p in parts])
        order = np.lexsort(got_x.T[::-1])
        ref = np.lexsort(x.T[::-1])
        assert np.array_equal(got_x[order], x[ref]) and np.array_equal(got_y[order], multi_y[ref])


def _multi_target_booster(T, rounds=2, objective="binary:logistic"):
    from xgboost_ray_b200 import engine as E
    bst = E.Booster({"objective": objective, "num_target": T, "base_score": 0.25})
    bst.n_features = 2
    leaf = dict(left=np.array([-1], np.int32), right=np.array([-1], np.int32), parent=np.array([-1], np.int32),
                split_feature=np.array([-1], np.int32), split_bin=np.array([-1], np.int32),
                split_cond=np.zeros(1, np.float32), default_left=np.zeros(1, np.uint8),
                value=np.array([0.5], np.float32), base_weight=np.array([0.7], np.float32),
                loss_chg=np.zeros(1, np.float32), sum_hess=np.array([10.0]), split_type=np.zeros(1, np.uint8),
                cat_bits=np.zeros((1, 8), np.uint32))
    bst._trees = [dict(leaf) for _ in range(rounds * T)]
    return bst


def test_model_file_counts_targets():
    import jsonschema
    from tests.model_schema import MODEL
    from xgboost_ray_b200 import engine as E
    bst = _multi_target_booster(3)
    d = json.loads(bytes(bst.save_raw()).decode())
    jsonschema.validate(d, copy.deepcopy(MODEL))
    L = d["learner"]
    assert L["learner_model_param"]["num_target"] == "3" and L["learner_model_param"]["num_class"] == "0"
    gb = L["gradient_booster"]["model"]
    assert gb["tree_info"] == [0, 1, 2, 0, 1, 2] and gb["iteration_indptr"] == [0, 3, 6]
    assert "num_target" not in json.loads(L["attributes"]["b2.params"])
    back = E.Booster(model_file=bytearray(bst.save_raw()))
    assert back.num_class == 3 and back.num_boosted_rounds() == 2 and back.params["num_target"] == 3
    assert bytes(back.save_raw()) == bytes(bst.save_raw())
    # one target: the file of a single-output model, no num_target parameter carried
    one = E.Booster(model_file=bytearray(_multi_target_booster(1).save_raw()))
    assert one.num_class == 1 and "num_target" not in one.params


def test_classifier_label_rules():
    from xgboost_ray_b200.sklearn import RayXGBClassifier
    X, _ = _data(n=20)
    with pytest.raises(ValueError, match="0 or 1"):
        RayXGBClassifier(n_estimators=1).fit(X, np.full((20, 2), 2.0))
    with pytest.raises(ValueError, match="0 or 1"):
        RayXGBClassifier(n_estimators=1).fit(X, np.full((20, 3), 0.5))
