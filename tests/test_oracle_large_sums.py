"""The exact fixed-point reference (tests/fixed_sums_reference.py) and the CPU oracle's leaf values and base_score past
2^23 rows, where one int64 sum of 40-bit fixed-point values can wrap.  The GPU side is tests/test_gpu_large_sums.py."""
import numpy as np
import pytest

from tests import fixed_sums_reference as R

F = np.float32


# ------------------------------------------------------------------ the reference itself
@pytest.mark.parametrize("scale", [1e-6, 0.37, 1.0, 1.99, 3e4])
def test_fixed_sum_matches_float64_at_small_n(scale):
    rng = np.random.RandomState(int(scale * 1000) % 997)
    v = (rng.normal(size=5001) * scale).astype(F)
    v[7] = F(scale)                       # the maximum itself
    e = R.quant_exponent(v)
    k = np.ldexp(1.0, R.LEAF_BITS - e)
    q = np.rint(v.astype(np.float64) * k)
    assert np.max(np.abs(q)) <= 2.0 ** 40
    assert R.fixed_sum(v, e) == np.sum(q, dtype=np.float64)   # below 2^53: the float64 sum of integers is exact


def test_fixed_sum_on_label_grid_is_the_plain_sum():
    rng = np.random.RandomState(3)
    y = R.grid_labels(rng, 4099, 0, 2048)
    g, h = R.gradients("reg:squarederror", np.zeros(y.size, F), y, np.full(y.size, 1.5, F))
    G, H = R.node_sums(g, h, R.quant_exponent(g), R.quant_exponent(h))
    assert G == np.sum(g, dtype=np.float64) and H == 1.5 * y.size


def test_fixed_sum_past_int64():
    # 2^24 + 2^20 values near -1.99: the exact sum is far beyond what one int64 holds
    _, y = R.root_case(R.N_LARGE)
    e = R.quant_exponent(y)
    assert e == 1
    ks, counts = np.unique(np.rint(y.astype(np.float64) * 1024).astype(np.int64), return_counts=True)
    exact = sum(int(k) * int(c) for k, c in zip(ks, counts)) << (R.LEAF_BITS - e - 10)   # q = k * 2^(39 - 10)
    got = R.fixed_sum(-y, e)
    assert got == -exact and abs(got) > 2 ** 63
    assert R.fixed_sum(np.ones(R.N_LARGE, F), 1) == R.N_LARGE << 39


def test_calc_weight_rules():
    assert R.calc_weight(-4.0, 1.0) == 2.0
    assert R.calc_weight(-4.0, 0.5) == 0.0                                  # below min_child_weight
    assert R.calc_weight(-4.0, 1.0, alpha=1.0) == 1.5                       # L1 shrinks |G| by alpha
    assert R.calc_weight(0.5, 1.0, alpha=1.0) == 0.0
    assert R.calc_weight(-4.0, 1.0, max_delta_step=0.7) == 0.7              # clipped
    assert R.calc_weight(4.0, 1.0, max_delta_step=0.7) == -0.7


# ------------------------------------------------------------------ the oracle at 2^24 + 2^20 rows
def _small_cuts(oracle):
    return oracle.Cuts.from_data(np.zeros((4, 1), F))   # estimate_base_score reads only labels and weights


@pytest.mark.parametrize("n", [R.N_CONTROL, R.N_LARGE])
@pytest.mark.parametrize("objective,weight", [("reg:squarederror", None), ("reg:squarederror", 1.5),
                                              ("binary:logistic", None)])
def test_oracle_base_score_exact(oracle, objective, weight, n):
    y, _ = R.intercept_case(objective, n)
    w = None if weight is None else np.full(n, weight, F)
    g, h = R.gradients(objective, np.zeros(n, F), y, w)
    G, H = R.node_sums(g, h, R.quant_exponent(g), R.quant_exponent(h))
    want = R.intercept(objective, G, H)
    bst = oracle.Booster({"objective": objective, "max_depth": 1}, _small_cuts(oracle))
    got = F(bst.estimate_base_score(y, w))
    assert got.view(np.uint32) == want.view(np.uint32), (got, want)


def test_oracle_root_leaf_exact(oracle):
    X, y = R.root_case(R.N_LARGE)
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.0}
    bst, _ = oracle.train(params, X, y, 1)
    t = bst.tree(0)
    assert t.n_nodes == 1
    g, h = R.gradients("reg:squarederror", np.zeros(y.size, F), y)
    G, H = R.node_sums(g, h, R.quant_exponent(g), R.quant_exponent(h))
    want = R.leaf_value(G, H)
    assert t.value[0].view(np.uint32) == want.view(np.uint32), (t.value[0], want)
    assert np.all(bst.margin[:, 0] == want)


def test_oracle_skewed_leaves_exact(oracle):
    X, y = R.skewed_case(R.N_LARGE)
    params = {"objective": "reg:squarederror", "max_depth": 1, "eta": 0.3, "base_score": 0.0}
    bst, _ = oracle.train(params, X, y, 1)
    t = bst.tree(0)
    assert t.n_nodes == 3 and t.split_feature[0] == 0
    g, h = R.gradients("reg:squarederror", np.zeros(y.size, F), y)
    eg, eh = R.quant_exponent(g), R.quant_exponent(h)
    side = X[:, 0] != 0
    for nid, rows in ((t.left[0], ~side), (t.right[0], side)):
        G, H = R.node_sums(g[rows], h[rows], eg, eh)
        want = R.leaf_value(G, H)
        assert t.value[nid].view(np.uint32) == want.view(np.uint32), (nid, int(rows.sum()), t.value[nid], want)
        assert t.sum_hess[nid] == rows.sum()
