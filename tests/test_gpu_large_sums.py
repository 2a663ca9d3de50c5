"""Leaf values and the estimated base_score past 2^23 rows, against the exact fixed-point reference
(tests/fixed_sums_reference.py).

A row adds up to 2^40 to a 40-bit fixed-point sum, so one int64 sum wraps past 2^23 rows of gradients near the
maximum and past 2^24 rows of a unit hessian.  These tests drive every writer of the leaf sums (the streaming
leaf_accumulate_kernel, the gathering leaf_sums_kernel, final_assign_kernel at the last split level, the unfused leaf
pass, the NCCL and peer-memory exchanges) and the intercept's sum_fixed_kernel with a node of 2^24 + 2^20 rows.

Tolerance: none.  The engine turns the exact integer sums into correctly rounded doubles and then runs the same IEEE
double / binary32 operations as the reference (calc_weight, times eta, the link), so leaf values, margins and
base_score must be equal bit for bit.  A wrapped sum is off by 2^64 units and gives a different value.

Device memory: at most 12 features x 2^24 rows of bins plus a few per-row arrays, about 2 GB."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import fixed_sums_reference as R

pytestmark = pytest.mark.gpu

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SQ = "reg:squarederror"


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def _bits(x):
    return np.asarray(x, F).view(np.uint32)


def _train(eng, params, X, y, weight=None, rounds=1):
    dm = eng.DMatrix(X, label=y, weight=weight)
    return eng.train(params, dm, num_boost_round=rounds, verbose_eval=False), dm


def _sq_sums(y, rows=None, eg=None, eh=None):
    """(G, H) of reg:squarederror at margin 0 over `rows`, quantised with the exponents of all rows"""
    g, h = R.gradients(SQ, np.zeros(y.size, F), y)
    eg = R.quant_exponent(g) if eg is None else eg
    eh = R.quant_exponent(h) if eh is None else eh
    if rows is not None:
        g, h = g[rows], h[rows]
    return R.node_sums(g, h, eg, eh)


# ------------------------------------------------------------------ intercept (sum_fixed_kernel + allreduce)
@pytest.mark.parametrize("n", [R.N_CONTROL, R.N_LARGE])
@pytest.mark.parametrize("objective,weight", [(SQ, None), (SQ, 1.5), ("binary:logistic", None)])
def test_base_score_exact(eng, objective, weight, n):
    y, _ = R.intercept_case(objective, n)
    w = None if weight is None else np.full(n, weight, F)
    g, h = R.gradients(objective, np.zeros(n, F), y, w)
    G, H = R.node_sums(g, h, R.quant_exponent(g), R.quant_exponent(h))
    want = R.intercept(objective, G, H)
    bst, _ = _train(eng, {"objective": objective, "max_depth": 1}, np.zeros((n, 1), F), y, w)
    got = F(bst.params["base_score"])
    assert _bits(got) == _bits(want), (got, want)


# ------------------------------------------------------------------ the root as the only leaf
def _check_root_leaf(bst, dm, y):
    G, H = _sq_sums(y)
    want = R.leaf_value(G, H)
    t = bst.get_trees()[0]
    assert len(t["left"]) == 1
    assert _bits(t["value"][0]) == _bits(want), (t["value"][0], want)
    m = bst.predict(dm, output_margin=True, training=True)
    assert np.array_equal(_bits(m), np.broadcast_to(_bits(F(0.0) + want), m.shape))   # base_score 0 + leaf


# max_depth 6: leaf_accumulate_kernel (streaming) sums the leaf; 12: leaf_sums_kernel (gathering) at the last level
@pytest.mark.parametrize("depth", [6, 12])
def test_root_leaf_exact(eng, depth):
    X, y = R.root_case(R.N_LARGE)
    bst, dm = _train(eng, {"objective": SQ, "max_depth": depth, "eta": 0.3, "base_score": 0.0}, X, y)
    _check_root_leaf(bst, dm, y)


def test_root_leaf_exact_unfused_leaf_pass():
    """B2_LEAF_FUSED=0: the leaf sums come from leaf_sums_kernel after the last level.  The flag is read once per
    process, so this runs in a process of its own."""
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "from xgboost_ray_b200 import engine as E\n"
        "from tests import fixed_sums_reference as R\n"
        "from tests.test_gpu_large_sums import _check_root_leaf, _train\n"
        "X, y = R.root_case(R.N_LARGE)\n"
        "bst, dm = _train(E, {'objective': 'reg:squarederror', 'max_depth': 6, 'eta': 0.3, 'base_score': 0.0}, X, y)\n"
        "_check_root_leaf(bst, dm, y)\n"
        "print('unfused ok')\n") % ROOT
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, B2_LEAF_FUSED="0"), capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and "unfused ok" in r.stdout, (r.stdout[-500:], r.stderr[-2500:])


# ------------------------------------------------------------------ one skewed split
def _check_skewed(bst, dm, X, y):
    t = bst.get_trees()[0]
    assert len(t["left"]) == 3 and t["split_feature"][0] == 0
    side = X[:, 0] != 0
    want = np.zeros(y.size, F)
    model = json.loads(bytes(bst.save_raw()))["learner"]["gradient_booster"]["model"]["trees"][0]
    assert model["sum_hessian"][0] == y.size
    for nid, rows in ((t["left"][0], ~side), (t["right"][0], side)):
        G, H = _sq_sums(y, rows)
        v = R.leaf_value(G, H)
        assert _bits(t["value"][nid]) == _bits(v), (int(nid), int(rows.sum()), t["value"][nid], v)
        assert model["sum_hessian"][nid] == rows.sum()   # histogram sums: exact row counts
        want[rows] = F(0.0) + v
    m = bst.predict(dm, output_margin=True, training=True)
    assert np.array_equal(_bits(m), _bits(want))


# max_depth 1: final_assign_kernel writes the leaf index, leaf_accumulate_kernel sums;
# max_depth 12: both children stop at level 1 and leaf_sums_kernel sums them at the last level
@pytest.mark.parametrize("depth", [1, 12])
def test_skewed_split_leaves_exact(eng, depth):
    X, y = R.skewed_case(R.N_LARGE)
    assert (X[:, 0] == 0).sum() > (1 << 24)
    bst, dm = _train(eng, {"objective": SQ, "max_depth": depth, "eta": 0.3, "base_score": 0.0}, X, y)
    _check_skewed(bst, dm, X, y)


def test_skewed_split_two_rounds_against_oracle(eng, oracle):
    from tests.test_gpu_parity import assert_same_model
    X, y = R.skewed_case(R.N_LARGE)
    params = {"objective": SQ, "max_depth": 1, "eta": 0.3, "base_score": 0.0}
    ebst, dm = _train(eng, params, X, y, rounds=2)
    obst, _ = oracle.train(params, X, y, 2)
    assert_same_model(ebst, obst, leaf_tol=0.0)
    m = ebst.predict(dm, output_margin=True, training=True)
    assert np.array_equal(_bits(m), _bits(obst.margin[:, 0]))


# ------------------------------------------------------------------ final_assign_kernel<kSums> at the last split level
CHAIN_LEVELS = 12       # = max_depth: one indicator per split level 0..11
CHAIN_GROUP = 4096      # rows of each peeled-off group


def chain_case(n):
    """12 indicator features; indicator k marks its own 4096 rows, whose label is 0.5 (the rest: near 1.99).  Each level
    peels one group off the large node, so the node split at level 11 -- by final_assign_kernel adding the leaf sums
    itself, above the streaming depth -- still holds n - 11 * 4096 > 2^24 rows."""
    X = np.zeros((n, CHAIN_LEVELS), F)
    y = R.grid_labels(np.random.RandomState(4), n, 2029, 2039)
    group = np.full(n, -1, np.int32)
    for k in range(CHAIN_LEVELS):
        rows = slice(k * CHAIN_GROUP, (k + 1) * CHAIN_GROUP)
        X[rows, k] = 1.0
        y[rows] = 0.5
        group[rows] = k
    return X, y, group


def test_chain_tree_last_level_sums_exact(eng):
    from xgboost_ray_b200 import engine
    assert CHAIN_LEVELS > engine.lib().b2_leaf_acc_max_depth()   # the gathering path, not the streaming pass
    X, y, group = chain_case(R.N_LARGE)
    bst, dm = _train(eng, {"objective": SQ, "max_depth": CHAIN_LEVELS, "eta": 0.3, "base_score": 0.0}, X, y)
    t = bst.get_trees()[0]
    assert len(t["left"]) == 2 * CHAIN_LEVELS + 1                   # a chain: 12 splits, 13 leaves
    depth = np.zeros(len(t["left"]), np.int32)
    for nid in range(1, len(t["left"])):
        depth[nid] = depth[t["parent"][nid]] + 1
    assert depth.max() == CHAIN_LEVELS
    g, h = R.gradients(SQ, np.zeros(y.size, F), y)
    eg, eh = R.quant_exponent(g), R.quant_exponent(h)
    want = np.zeros(y.size, F)
    for k in range(-1, CHAIN_LEVELS):
        rows = group == k
        G, H = R.node_sums(g[rows], h[rows], eg, eh)
        want[rows] = F(0.0) + R.leaf_value(G, H)   # base_score 0 + leaf
    assert (group == -1).sum() > (1 << 24)
    m = bst.predict(dm, output_margin=True, training=True)
    bad = np.flatnonzero(_bits(m) != _bits(want))
    assert bad.size == 0, (bad.size, group[bad[:3]], m[bad[:3]], want[bad[:3]])


# ------------------------------------------------------------------ two GPUs: only the cross-rank sum exceeds int64
def _ngpu():
    from xgboost_ray_b200 import engine
    return engine.device_count()


@pytest.mark.timeout(600)
@pytest.mark.parametrize("exchange", ["p2p", "nccl"])
def test_two_gpu_cross_rank_leaf_sum_exact(exchange, monkeypatch):
    """2^23 + 2^19 rows per rank, every label 1.0 and base_score 0: g = -1 and h = 1 on every row, so each rank's
    sums stay below 2^63 and only their total passes it."""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    import xgboost_ray_b200.main as M
    from xgboost_ray_b200 import RayDMatrix, RayParams, train
    M.shutdown_actors()                       # the exchange kind is read by the actor processes when they start
    if exchange == "nccl":
        monkeypatch.setenv("B2_EXCHANGE", "nccl")
    else:
        monkeypatch.delenv("B2_EXCHANGE", raising=False)
    n = R.N_LARGE
    x = np.zeros((n, 1), F)
    y = np.ones(n, F)
    params = {"objective": SQ, "max_depth": 6, "eta": 0.3, "base_score": 0.0}
    b1 = train(params, RayDMatrix(x, y), num_boost_round=1, ray_params=RayParams(num_actors=1))
    b2 = train(params, RayDMatrix(x, y), num_boost_round=1, ray_params=RayParams(num_actors=2))
    M.shutdown_actors()
    assert b1.get_dump(dump_format="json", with_stats=True) == b2.get_dump(dump_format="json", with_stats=True)
    want = R.leaf_value(-float(n), float(n))
    for b in (b1, b2):
        v = b.get_trees()[0]["value"]
        assert len(v) == 1 and _bits(v[0]) == _bits(want), (v, want)
