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


@pytest.fixture(scope="module")
def built():
    """libb2hist.so: the engine checks the parameters (B2_CheckParams needs no device)."""
    from xgboost_ray_b200 import build
    return build.build()


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


def bits(v):
    return np.array([v], F32).tobytes()


def test_radix_select_by_hand():
    r = np.array([3.0, 1.0, 2.0], F32)
    # n = 3: alpha = 1/(n+1) = 0.25 is the minimum and 3/(n+1) = 0.75 the maximum by equality, with one target
    assert R.radix_select(r, 0.25) == (F32(1.0), None)
    assert R.radix_select(r, 0.75) == (F32(3.0), None)
    # frac = 0: alpha (n + 1) = 2 is an integer, so q is v_1 itself; the targets are 2.0 and 3.0, keys 0xc0000000 and
    # 0xc0400000, which part in the second byte
    assert R.radix_select(r, 0.5) == (F32(2.0), 1)
    assert R.leaf_quantile(r, 0.5) == F32(2.0)
    # -0 and +0 are one key: the targets never split, and the answer is +0
    q, split = R.radix_select(np.array([-0.0, 0.0, -0.0, 0.0], F32), 0.5)
    assert bits(q) == bits(0.0) and split is None
    # weighted: masses 2^31 each (max weight 1) sum to 2^33; alpha = 0.5 puts the target exactly at the end of 2.0's
    # cumulative weight, so 2.0 is picked and not 3.0
    r4 = np.array([4.0, 1.0, 3.0, 2.0], F32)
    m = R.fixed_mass(np.ones(4, F32), R.frexp_exponent(1.0))
    assert m.tolist() == [2 ** 31] * 4
    assert R.radix_select(r4, 0.5, m) == (F32(2.0), None) and R.leaf_quantile(r4, 0.5, m) == F32(2.0)
    assert R.radix_select(r4, np.nextafter(F32(0.5), F32(1)), m)[0] == F32(3.0)
    # half-way masses with max weight 1 (e = 1, scale 2^31): 2^-32 -> 0.5 -> 0 and 3 * 2^-32 -> 1.5 -> 2, ties to even
    w = np.array([1.0, 2.0 ** -32, 3 * 2.0 ** -32, 5 * 2.0 ** -32], F32)
    assert R.fixed_mass(w, R.frexp_exponent(w.max())).tolist() == [2 ** 31, 0, 2, 2]
    # a row of mass 0 is never the answer of the weighted rule, even as the smallest value: W = 2^31 + 4, so alpha =
    # 1e-10 gives the target 1, first reached by 2.0 (mass 2)
    m = R.fixed_mass(w, 1)
    r = np.array([5.0, -1.0, 2.0, 3.0], F32)
    assert R.radix_select(r, 1e-10, m) == (F32(2.0), None) and R.leaf_quantile(r, 1e-10, m) == F32(2.0)
    # every mass 0 (weights 2^-32 where the tree's largest is 1): ceil(alpha W) = 0, the minimum by count
    m0 = R.fixed_mass(np.full(3, 2.0 ** -32, F32), 1)
    assert m0.tolist() == [0, 0, 0]
    assert R.radix_select(r[1:], 0.9, m0) == (F32(-1.0), None) and R.leaf_quantile(r[1:], 0.9, m0) == F32(-1.0)


def weighted_inputs(y, w):
    keep = w != 0
    return y[keep], R.fixed_mass(w[keep], R.frexp_exponent(w.max()))


@pytest.mark.parametrize("n", [1, 2, 3, 4, 255, 256, 257, 20000])
def test_radix_select_is_the_sort_on_boundary_sets(n):
    """The kernel's four-pass selection, replayed, gives leaf_quantile's value bit for bit on every boundary set, and
    each pair set splits its targets in the pass its keys say"""
    rng = np.random.RandomState(n)
    splits = set()
    checked = 0
    for name, y, alphas in R.boundary_sets(n):
        for a in alphas:
            q, split = R.radix_select(y, a)
            assert bits(q) == bits(R.leaf_quantile(y, a)), (name, float(a))
            splits.add(split)
            if name.startswith("pair") and n > 2:
                assert split == int(name[-2]), (name, split)
            for kind in ("int", "half", "pow2"):
                w = R.boundary_weights(kind, n, rng)
                yw, m = weighted_inputs(y, w)
                aw = [a]
                if kind == "pow2":          # no zero weights: yw is y
                    aw.append(R.boundary_alpha(y, w, rng) or a)
                for b in aw:
                    qw, sw = R.radix_select(yw, b, m)
                    assert bits(qw) == bits(R.leaf_quantile(yw, b, m)) and sw is None, (name, kind, float(b))
            checked += 1
    assert checked >= len(R.SPLIT_PAIRS)
    if n > 1:
        assert splits >= {0, 1, 2, 3, None}, splits


def test_weighted_target_on_a_cumulative_boundary():
    rng = np.random.RandomState(5)
    for n in (2, 3, 5, 100, 257):
        y = rng.choice(R.POOL, n)
        w = R.boundary_weights("pow2", n, rng)
        a = R.boundary_alpha(y, w, rng)
        if a is None:
            continue
        m = R.fixed_mass(w, R.frexp_exponent(w.max()))
        yn = np.where(y == 0, F32(0.0), y).astype(F32)
        order = np.argsort(yn, kind="stable")
        cum = np.cumsum(m[order])
        target = int(np.ceil(float(a) * float(cum[-1])))
        i = int(np.nonzero(cum == target)[0][0])          # the target is exactly a cumulative sum
        assert yn[order][i] < yn[order][i + 1]
        assert R.leaf_quantile(y, a, m) == yn[order][i] == R.radix_select(y, a, m)[0]


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
def test_rejected_combinations(built, extra, match):
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
