"""Exact reference of the 40-bit fixed-point sums behind leaf values and the estimated base_score (DESIGN.md §2
items 4 and 5), valid at any row count.

A row adds q = rint(v * 2^(40 - e)) to its leaf's sum, with e the frexp exponent of the tree's max |g| (or |h|), so
|q| <= 2^40 and a plain int64 sum can wrap past 2^23 rows.  Here the sums are Python integers: every chunk of 2^20
rows is summed in int64 (at most 2^60 in magnitude) and the chunk sums are added as Python ints.  No float
accumulation anywhere; the only roundings are the ones the engine makes too (the exact sum to double, then the IEEE
double / binary32 operations of calc_weight, eta and the link).

With labels on a 2^-10 grid every q is exact, so these sums also equal the plain mathematical sums of g and h.
"""
import numpy as np

from tests.objective_reference import sigmoid_

F = np.float32
LEAF_BITS = 40
_CHUNK = 1 << 20


def quant_exponent(v):
    """frexp exponent of max |v| (binary32), 0 for an all-zero array: the engine's quant_exponent_kernel."""
    vmax = F(np.max(np.abs(np.asarray(v, F)))) if np.size(v) else F(0.0)
    bits = int(vmax.view(np.uint32))
    return 0 if bits == 0 else ((bits >> 23) & 0xff) - 126


def fixed_sum(v, e):
    """sum over rows of rint(v * 2^(40 - e)) as an exact Python int."""
    v = np.asarray(v, F)
    k = np.ldexp(1.0, LEAF_BITS - e)
    total = 0
    for i in range(0, v.size, _CHUNK):
        q = np.rint(v[i:i + _CHUNK].astype(np.float64) * k)   # binary32 * 2^k is exact in float64; |q| <= 2^40
        total += int(q.astype(np.int64).sum())
    return total


def node_sums(g, h, eg, eh):
    """(G, H) in float64 from the exact fixed-point sums: float(int) rounds correctly, the power-of-two scale is exact."""
    return float(fixed_sum(g, eg)) / np.ldexp(1.0, LEAF_BITS - eg), float(fixed_sum(h, eh)) / np.ldexp(1.0, LEAF_BITS - eh)


def calc_weight(G, H, min_child_weight=1.0, reg_lambda=1.0, alpha=0.0, max_delta_step=0.0):
    """b2_calc_weight (common.cuh): xgboost's CalcWeight in float64."""
    if H < min_child_weight or H <= 0.0:
        return 0.0
    t = G
    if alpha != 0.0:
        t = G - alpha if G > alpha else (G + alpha if G < -alpha else 0.0)
    dw = -t / (H + reg_lambda)
    if max_delta_step != 0.0 and abs(dw) > max_delta_step:
        dw = float(np.copysign(max_delta_step, dw))
    return dw


def leaf_value(G, H, eta=0.3, **kw):
    """binary32 leaf value: weight rounded to binary32, times eta in binary32 (leaf_values_kernel)."""
    return F(F(calc_weight(G, H, **kw)) * F(eta))


def intercept(objective, G, H):
    """base_score from the stump -G/H at margin 0 (0 when H <= 1e-6), through the link (estimate_base_score)."""
    stump = F(0.0) if H <= 1e-6 else F(-G / H)
    if objective == "binary:logistic":
        return F(sigmoid_(np.array([stump], F))[0])
    return stump


def gradients(objective, margin, label, weight=None):
    """binary32 gradient pairs of reg:squarederror / binary:logistic (gradient_scalar_kernel, scale_pos_weight 1)."""
    m = np.asarray(margin, F)
    y = np.asarray(label, F)
    w = np.ones_like(y) if weight is None else np.asarray(weight, F)
    if objective == "reg:squarederror":
        return ((m - y) * w).astype(F), w.astype(F)
    p = sigmoid_(m)
    hh = np.maximum(p * (F(1.0) - p), F(1e-16))
    return ((p - y) * w).astype(F), (hh * w).astype(F)


# ---- inputs past the int64 limit of one fixed-point sum.  Labels sit on a 2^-10 grid, so every q is exact.
N_LARGE = (1 << 24) + (1 << 20)   # past 2^24: H of a unit-hessian node wraps int64, and G near 2^e wraps past 2^23
N_CONTROL = 1 << 20               # no sum comes near 2^63


def grid_labels(rng, n, lo, hi):
    """labels k / 1024 with k uniform in [lo, hi)"""
    return (rng.randint(lo, hi, size=n) / 1024.0).astype(F)


def intercept_case(objective, n, seed=0):
    """(label, weight) for the base_score tests: squared error labels in [0, 2) (mean near 1), logistic labels 70 % ones"""
    rng = np.random.RandomState(seed)
    if objective == "binary:logistic":
        return (rng.uniform(size=n) < 0.7).astype(F), None
    return grid_labels(rng, n, 0, 2048), None


def root_case(n, seed=1):
    """one constant feature (no split exists: the root is the only leaf) and labels in [1.981, 1.990]: with base_score 0
    every g = -y sits just below -2^e (e = 1), so q_g is close to -2^40 and G wraps int64 past about 2^23 rows"""
    rng = np.random.RandomState(seed)
    return np.zeros((n, 1), F), grid_labels(rng, n, 2029, 2039)


def skewed_case(n, seed=2):
    """one binary feature with about 5 % ones; labels near 1.99 on the 95 % side and near 0.5 on the other, so the
    root splits once and the large leaf holds more than 2^24 rows at N_LARGE"""
    rng = np.random.RandomState(seed)
    x = (rng.uniform(size=n) < 0.05).astype(F)
    y = np.where(x == 0, grid_labels(rng, n, 2029, 2039), grid_labels(rng, n, 500, 520)).astype(F)
    return x.reshape(n, 1), y
