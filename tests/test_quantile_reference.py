"""CPU checks of reg:quantileerror's reference rules (tests/quantile_reference.py), its model file and its parameters."""
import copy
import json

import jsonschema
import numpy as np
import pytest

from tests import quantile_reference as R
from tests.model_schema import MODEL
from xgboost_ray_b200 import engine as E

F32 = np.float32


def test_unweighted_rule_by_hand():
    assert R.leaf_quantile([], 0.5) is None
    # n = 1: every alpha gives the single value
    for a in (0.01, 0.5, 0.99):
        assert R.leaf_quantile([3.0], a) == F32(3.0)
    # n = 2: alpha <= 1/3 -> min, alpha >= 2/3 -> max, in between x = 3 alpha, j = 0, d = x - 1
    assert R.leaf_quantile([5.0, 1.0], 0.3) == F32(1.0)
    assert R.leaf_quantile([5.0, 1.0], 0.25) == F32(1.0)
    assert R.leaf_quantile([5.0, 1.0], 0.7) == F32(5.0)
    assert R.leaf_quantile([5.0, 1.0], 0.5) == F32(1.0 + (3 * float(F32(0.5)) - 1.0) * 4.0)
    # ties and signed zeros
    assert R.leaf_quantile([2.0, 2.0, 2.0], 0.4) == F32(2.0)
    q = R.leaf_quantile(np.array([-0.0, 0.0, -0.0], F32), 0.5)
    assert q == 0 and not np.signbit(q)


def test_weighted_rule_by_hand():
    r = np.array([4.0, 1.0, 3.0, 2.0], F32)
    # unit weights: first value whose cumulative weight reaches ceil(alpha W)
    m = R.fixed_mass(np.ones(4, F32), R.frexp_exponent(1.0))
    assert R.leaf_quantile(r, 0.5, m) == F32(2.0)
    assert R.leaf_quantile(r, 0.51, m) == F32(3.0)
    assert R.leaf_quantile(r, 0.01, m) == F32(1.0)
    assert R.leaf_quantile(r, 0.99, m) == F32(4.0)
    # a zero weight never carries the cumulative sum over the target
    w = np.array([1.0, 0.0, 1.0, 2.0], F32)
    m = R.fixed_mass(w, R.frexp_exponent(2.0))
    assert R.leaf_quantile(r, 0.3, m) == F32(2.0)     # rows 2.0 (w 2) reach 2 >= ceil(0.3 * 4)
    # fractional weights
    w = np.array([0.25, 0.5, 0.125, 0.125], F32)
    m = R.fixed_mass(w, R.frexp_exponent(0.5))
    assert R.leaf_quantile(r, 0.5, m) == F32(1.0)     # 1.0 has weight 0.5 = half of W = 1
    assert R.leaf_quantile(r, 0.6, m) == F32(2.0)
    # all weights rounding to zero: the minimum
    assert R.leaf_quantile(r, 0.7, np.zeros(4, np.int64)) == F32(1.0)


@pytest.mark.parametrize("seed", range(6))
def test_rules_agree_with_numpy(seed):
    rng = np.random.RandomState(seed)
    n = rng.randint(1, 400)
    r = rng.normal(size=n).astype(F32)
    if seed % 2:
        r = np.round(r, 1).astype(F32)                  # ties
    for a in (0.01, 0.05, 0.1, 0.37, 0.5, 0.9, 0.95, 0.99):
        ref = np.quantile(r.astype(np.float64), float(F32(a)), method="weibull")
        assert abs(float(R.leaf_quantile(r, a)) - ref) <= 1e-6 * max(1.0, abs(ref))
        m = R.fixed_mass(np.ones(n, F32), 1)
        assert R.leaf_quantile(r, a, m) == F32(np.quantile(r, float(F32(a)), method="inverted_cdf"))


@pytest.mark.parametrize("seed", range(4))
def test_fixed_point_and_fp32_sums_agree_for_integer_weights(seed):
    rng = np.random.RandomState(seed)
    n = 300
    r = rng.normal(size=n).astype(F32)
    w = rng.randint(0, 50, size=n).astype(F32)
    e = R.frexp_exponent(w.max())
    keep = w != 0
    W = float(w.sum())
    assert W < 2 ** 24
    checked = 0
    for a in np.linspace(0.02, 0.98, 97):
        # the running fp32 rule compares with fp32(alpha W); where that rounding crosses an integer the exact rule
        # (which compares with alpha W itself) differs by design
        if np.ceil(float(F32(a)) * W) != np.ceil(float(F32(F32(a) * F32(W)))):
            continue
        checked += 1
        assert R.leaf_quantile(r[keep], a, R.fixed_mass(w[keep], e)) == R.weighted_quantile_fp32(r[keep], a, w[keep])
    assert checked >= 48


def test_intercept_is_mean_of_label_quantiles():
    y = np.arange(1, 10, dtype=F32)
    assert R.intercept(y, None, np.array([0.5], F32)) == F32(5.0)
    q1, q9 = R.leaf_quantile(y, 0.1), R.leaf_quantile(y, 0.9)
    assert R.intercept(y, None, np.array([0.1, 0.9], F32)) == F32(F32(F32(0) + q1 + q9) / F32(2))


def test_gradients_and_pinball():
    m = np.array([[0.0, 1.0], [2.0, 2.0]], F32)
    y = np.array([1.0, 2.0], F32)
    g, h = R.gradients(m, y, np.array([1.0, 2.0], F32), np.array([0.25, 0.75], F32))
    assert g.tolist() == [[-0.25, 0.25], [1.5, 0.5]] and h.tolist() == [[1.0, 1.0], [2.0, 2.0]]
    # row 0: u = (1, 0) -> 0.25; row 1: u = (0, 0) -> 0; mean over rows and alphas with weights (1, 2)
    assert R.pinball(m, y, np.array([1.0, 2.0]), [0.25, 0.75]) == pytest.approx(0.25 / 6)


@pytest.mark.parametrize("value,want", [
    (0.5, [0.5]), (0.1, [0.1]), ([0.05, 0.5, 0.95], [0.05, 0.5, 0.95]), ((0.2, 0.8), [0.2, 0.8]),
    (np.array([0.3, 0.7]), [0.3, 0.7]), ("[0.1, 0.5, 0.9]", [0.1, 0.5, 0.9]), ("0.25", [0.25]), (None, [0.5]),
    (np.float32(0.4), [0.4])])
def test_quantile_alpha_forms(value, want):
    assert E.quantile_alphas(value).tobytes() == np.array(want, F32).tobytes()


@pytest.mark.parametrize("value", [0.0, 1.0, -0.1, 1.5, float("nan"), float("inf"), [0.5, 1.0], "abc", [], "[0.2, x]",
                                   [True], 1 - 1e-9])
def test_quantile_alpha_errors(value):
    with pytest.raises(E.XGBoostError, match="quantile_alpha"):
        E.quantile_alphas(value)


def test_quantile_alpha_error_names_the_value():
    with pytest.raises(E.XGBoostError, match="1.5"):
        E.quantile_alphas([0.5, 1.5])


@pytest.mark.parametrize("extra,match", [({"num_class": 3}, "num_class"), ({"booster": "dart"}, "dart"),
                                         ({"num_parallel_tree": 2}, "num_parallel_tree"),
                                         ({"quantile_alpha": 2.0}, "quantile_alpha")])
def test_rejected_combinations(extra, match):
    params = dict({"objective": "reg:quantileerror"}, **extra)
    with pytest.raises(E.XGBoostError, match=match):
        E._check_supported(params)
    E._check_supported({"objective": "reg:squarederror", "num_class": 3})   # other objectives: not this rule


def _quantile_booster(alphas):
    bst = E.Booster({"objective": "reg:quantileerror", "quantile_alpha": alphas, "base_score": 0.25})
    bst.n_features = 2
    leaf = dict(left=np.array([-1], np.int32), right=np.array([-1], np.int32), parent=np.array([-1], np.int32),
                split_feature=np.array([-1], np.int32), split_bin=np.array([-1], np.int32),
                split_cond=np.zeros(1, np.float32), default_left=np.zeros(1, np.uint8),
                value=np.array([0.5], np.float32), base_weight=np.array([0.7], np.float32),
                loss_chg=np.zeros(1, np.float32), sum_hess=np.array([10.0]), split_type=np.zeros(1, np.uint8),
                cat_bits=np.zeros((1, 8), np.uint32))
    bst._trees = [dict(leaf) for _ in range(2 * E.quantile_alphas(alphas).size)]
    return bst


def test_multi_quantile_model_file_against_schema():
    bst = _quantile_booster([0.05, 0.5, 0.95])
    d = json.loads(bytes(bst.save_raw()).decode())
    schema = copy.deepcopy(MODEL)
    schema["properties"]["learner"]["properties"]["objective"]["oneOf"].append(
        {"type": "object",
         "properties": {"name": {"const": "reg:quantileerror"},
                        "reg_quantileerror_param": {"type": "object", "properties": {"quantile_alpha": {"type": "string"}},
                                                    "required": ["quantile_alpha"], "additionalProperties": False}},
         "required": ["name", "reg_quantileerror_param"], "additionalProperties": False})
    jsonschema.validate(d, schema)
    L = d["learner"]
    assert L["learner_model_param"]["num_target"] == "3" and L["learner_model_param"]["num_class"] == "0"
    assert L["objective"]["reg_quantileerror_param"]["quantile_alpha"] == "[0.0500000007, 0.5, 0.949999988]"
    gb = L["gradient_booster"]["model"]
    assert gb["tree_info"] == [0, 1, 2, 0, 1, 2] and gb["iteration_indptr"] == [0, 3, 6]
    # read back: the alphas (bit for bit), the output count and the rounds
    back = E.Booster(model_file=bytearray(bst.save_raw()))
    assert E.quantile_alphas(back.params["quantile_alpha"]).tobytes() == np.array([0.05, 0.5, 0.95], F32).tobytes()
    assert back.num_class == 3 and back.num_boosted_rounds() == 2
    cfg = json.loads(back.save_config())["learner"]["objective"]
    assert cfg == {"name": "reg:quantileerror", "reg_quantileerror_param": {"quantile_alpha": "[0.0500000007, 0.5, 0.949999988]"}}


def test_single_quantile_model_counts_one_target():
    bst = _quantile_booster(0.3)
    L = json.loads(bytes(bst.save_raw()).decode())["learner"]
    assert L["learner_model_param"]["num_target"] == "1" and bst.num_class == 1


def test_param_text_writes_exact_alphas():
    bst = E.Booster({"objective": "reg:quantileerror", "quantile_alpha": "[0.1, 0.9]"})
    text = bst._param_text().decode()
    vals = [float(x) for x in dict(line.split("=", 1) for line in text.split("\n"))["quantile_alpha"].split(",")]
    assert np.array(vals, F32).tobytes() == np.array([0.1, 0.9], F32).tobytes()


def test_sklearn_passes_quantile_alpha():
    from xgboost_ray_b200.sklearn import RayXGBRegressor
    r = RayXGBRegressor(objective="reg:quantileerror", quantile_alpha=[0.1, 0.9])
    assert r.get_xgb_params()["quantile_alpha"] == [0.1, 0.9]
    assert r.get_params()["quantile_alpha"] == [0.1, 0.9]
