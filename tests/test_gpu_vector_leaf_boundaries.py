"""Vector-leaf trees (multi_strategy="multi_output_tree", DESIGN.md §2 item 19) against tests/multi_output_reference.py
at the shapes where the shared tree steps change layout or path:

  feature layout  F = 31 / 32 / 33 / 100 / 480 / 512 / 513 / 1000, i.e. G = ceil(F / 32) = 1 / 1 / 2 / 4 / 15 / 16 / 17 /
                  32 feature groups: the pair-plan histogram (G <= 16) and the one-group-per-CTA histogram (G > 16), the
                  split scan at 8 * G CTAs per node with the winner in the last group, the child totals past group 0
  quantisation    hist_qbits 8 / 12 / 20 / 24 with hist_chunk_rows default / 64 / 4096 (each target's histogram through
                  the shared-memory window separately), max_bin 2 and 16
  depth           max_depth 1, 11 (the last streaming leaf pass), 12 and 14 (assign_leaves once per target), a gamma-
                  pruned ragged tree at depth 10
  target count    T = 2 / 16 (fused |g|, |h| maxima, CUDA-graph capture and replays of both round parities) and 17 / 64
                  (separate maxima, direct launches), 6 to 8 rounds
  graph replay    the model bytes of 10 rounds equal those of a run with B2_GRAPH=0 (graphs off)
  sampling        subsample 0.5 / 0.8 alone and with colsample_by* and feature_weights, distinct targets
  per-target scale one tree with targets whose exponents are 0 (all-zero pairs), -148 (subnormal g), past 60
                  (g, h * 2^60)
  prediction      held-out rows with NaN, a non-NaN missing, ±inf and values at split conditions: output margins for
                  iteration_range (0, 0), (0, 2), (2, 5) and pred_leaf, bit for bit against the reference walk
  large sums      2^24 + 2^20 rows (and the 2^20 control) in one leaf, each target's value from its exact 40-bit sums
                  (tests/fixed_sums_reference.py), and the multi-target intercept

Trees, split conditions and loss_chg are compared exactly, leaf vectors within 1e-5, train margins bit for bit.

Device memory: the level histograms take 2 * T * 2^(D-1) * G * 128 KiB.  The largest cases are max_depth 14 at T = 2 and
G = 1 (4 GiB of histograms, as test_gpu_multi_output.py's depth-14 case) and the 2^24 + 2^20-row cases at max_depth 12
(1 GiB of histograms plus about 0.6 GiB of per-row arrays); every other case stays under 1.1 GiB of histograms.  On an
H100 80GB HBM3 (700 W power limit) the whole file took 151 s, reference growth included, and the device memory of the
test process peaked at 11,555 MiB: the engine keeps freed buffers for reuse, so the process holds what earlier cases
allocated (the depth-14 case added 4.1 GiB, the 2^24 + 2^20-row cases 2.8 GiB)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import fixed_sums_reference as FS
from tests import multi_output_reference as MO
from tests import multi_target_reference as MT

pytestmark = pytest.mark.gpu
F32 = np.float32
VEC = {"multi_strategy": "multi_output_tree"}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def layout_data(n, F, T, seed, nan_frac=0.05):
    """uniform [0, 10) with NaN, a constant column (1) and an all-missing column (F - 2); target k leans on the last
    feature (the last group), one in the middle and one near the front"""
    rng = np.random.RandomState(seed)
    X = rng.uniform(0, 10, size=(n, F)).astype(F32)
    X[rng.uniform(size=X.shape) < nan_frac] = np.nan
    X[:, 1] = 2.5
    X[:, F - 2] = np.nan
    Z = np.nan_to_num(X, nan=5.0)
    cols = [Z[:, F - 1] * (1.0 + 0.3 * k) + np.sin(Z[:, (F // 2 + k) % F]) + 0.2 * Z[:, (3 * k + 3) % F]
            + rng.normal(0, 0.3, n) for k in range(T)]
    return X, np.stack(cols, 1).astype(F32)


def run(eng, params, X, Y, rounds, weight=None, feature_weights=None, missing=None):
    """train on the GPU and with the reference; trees exactly, leaf vectors within 1e-5, train margins bit for bit"""
    d = eng.DMatrix(X, label=Y, weight=weight, multi_target=True)
    if feature_weights is not None:
        d.set_info(feature_weights=feature_weights)
    bst = eng.train(dict(params, **VEC), d, num_boost_round=rounds, verbose_eval=False)
    ref = MO.train(params, X, Y, rounds, weight=weight, feature_weights=feature_weights)
    assert F32(bst.params["base_score"]) == F32(ref.base_score)
    MO.assert_engine_matches(bst, ref)
    m = bst.predict(d, training=True, output_margin=True)
    assert m.shape == Y.shape and m.tobytes() == ref.margin.tobytes()
    return bst, ref, d


def split_features(bst):
    return np.concatenate([t["split_feature"][t["split_feature"] >= 0] for t in bst.get_trees()])


def max_depth_reached(bst):
    out = 0
    for t in bst.get_trees():
        d = np.zeros(len(t["left"]), np.int64)
        for nid in range(1, len(t["left"])):
            d[nid] = d[t["parent"][nid]] + 1
        out = max(out, int(d.max()))
    return out


# ------------------------------------------------------------------ feature layout
@pytest.mark.parametrize("F,T,depth", [(31, 4, 8), (32, 3, 8), (33, 4, 8), (100, 3, 8), (480, 3, 6), (512, 4, 6),
                                       (513, 3, 6), (1000, 3, 5)])
def test_feature_layout(eng, F, T, depth):
    X, Y = layout_data(8000 if F <= 513 else 6000, F, T, seed=F)
    bst, ref, _ = run(eng, {"objective": "reg:squarederror", "max_depth": depth, "eta": 0.3}, X, Y, 3)
    sf = split_features(bst)
    G = (F + 31) // 32
    assert (sf >= 32 * (G - 1)).any(), "no split on a feature of the last group"
    assert not np.isin(sf, [1, F - 2]).any()                    # the constant and the all-missing column
    assert any(t["default_left"][t["split_feature"] >= 0].any() for t in bst.get_trees())


# ------------------------------------------------------------------ quantisation: hist_qbits x chunking, max_bin
@pytest.mark.parametrize("chunk", [None, 64, 4096])
@pytest.mark.parametrize("qbits", [8, 12, 20, 24])
def test_qbits_and_chunking(eng, qbits, chunk):
    X, Y = layout_data(20000, 12, 3, seed=qbits)
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "hist_qbits": qbits}
    if chunk is not None:
        params["hist_chunk_rows"] = chunk
    run(eng, params, X, Y, 3)


@pytest.mark.parametrize("max_bin", [2, 16])
def test_few_bins(eng, max_bin):
    X, Y = layout_data(10000, 12, 3, seed=50 + max_bin)
    w = np.random.RandomState(max_bin).uniform(0.5, 2.0, len(Y)).astype(F32)
    run(eng, {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "max_bin": max_bin}, X, Y, 3, weight=w)


# ------------------------------------------------------------------ depth
@pytest.mark.parametrize("depth,T", [(1, 3), (11, 3), (12, 3), (14, 2)])
def test_depth(eng, depth, T):
    X, Y = layout_data(20000, 12, T, seed=100 + depth)
    bst, _, _ = run(eng, {"objective": "reg:squarederror", "max_depth": depth, "eta": 0.3, "min_child_weight": 0.5},
                    X, Y, 3)
    assert max_depth_reached(bst) == depth


def test_gamma_pruned_ragged_tree(eng):
    X, Y = layout_data(20000, 12, 3, seed=7)
    bst, ref, _ = run(eng, {"objective": "reg:squarederror", "max_depth": 10, "eta": 0.3, "gamma": 30.0}, X, Y, 3)
    nodes = [t.n_nodes for t in ref._trees]
    assert max_depth_reached(bst) >= 6 and all(n < 2 ** 11 - 1 for n in nodes)
    # ragged: leaves at several depths
    t = bst.get_trees()[0]
    d = np.zeros(len(t["left"]), np.int64)
    for nid in range(1, len(t["left"])):
        d[nid] = d[t["parent"][nid]] + 1
    assert len(set(d[t["split_feature"] < 0].tolist())) >= 3


# ------------------------------------------------------------------ target count: fused maxima and graphs vs direct
@pytest.mark.parametrize("T,rounds", [(2, 8), (16, 7), (17, 6), (64, 6)])
def test_target_count(eng, T, rounds):
    X, Y = layout_data(6000, 12, T, seed=200 + T)
    run(eng, {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3}, X, Y, rounds)


# ------------------------------------------------------------------ graph replay: same bytes as direct launches
_CHILD = """
import sys
sys.path.insert(0, {root!r})
import numpy as np
from xgboost_ray_b200 import engine as eng
from tests.test_gpu_vector_leaf_boundaries import layout_data, VEC
X, Y = layout_data(6000, 12, 4, seed=300)
bst = eng.train(dict({{"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3}}, **VEC),
                eng.DMatrix(X, label=Y, multi_target=True), num_boost_round=10, verbose_eval=False)
open({out!r}, "wb").write(bytes(bst.save_raw()))
"""


def test_graph_replay_matches_direct_launches(eng, tmp_path, capfd):
    if os.environ.get("B2_GRAPH", "1") in ("", "0"):
        pytest.skip("CUDA graphs are switched off in this process")
    X, Y = layout_data(6000, 12, 4, seed=300)
    bst, _, _ = run(eng, {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3}, X, Y, 10)
    err = capfd.readouterr().err
    assert "CUDA graph capture of the tree failed" not in err
    out = tmp_path / "direct.json"
    env = dict(os.environ, B2_GRAPH="0")
    r = subprocess.run([sys.executable, "-c", _CHILD.format(root=ROOT, out=str(out))], env=env, cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert bytes(bst.save_raw()) == out.read_bytes()


# ------------------------------------------------------------------ row sampling with distinct targets
@pytest.mark.parametrize("cols", [False, True], ids=["rows", "rows+cols"])
@pytest.mark.parametrize("subsample", [0.5, 0.8])
def test_subsample(eng, subsample, cols):
    X, Y = layout_data(10000, 40, 3, seed=int(subsample * 10) + cols)
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "subsample": subsample, "seed": 17}
    fw = None
    if cols:
        params.update(colsample_bytree=0.8, colsample_bylevel=0.8, colsample_bynode=0.7)
        fw = np.linspace(0.2, 3.0, X.shape[1]).astype(F32)
    run(eng, params, X, Y, 4, feature_weights=fw)


# ------------------------------------------------------------------ per-target quantisation scale
def test_per_target_exponents(eng):
    X, Y = layout_data(8000, 12, 4, seed=400)
    n = len(Y)
    tiny = F32(np.ldexp(1.0, -149))

    def grads(margin):
        r = (margin - Y).astype(F32)
        g = np.zeros_like(r)
        h = np.zeros_like(r)
        # target 0: all zero (exponents 0); target 1: g in {-1, 0, 1} * 2^-149 (exponent -148), h = 1;
        # target 2: (g, h) * 2^60 (exponents 62 and 61); target 3: ordinary squared error
        g[:, 1] = (np.sign(r[:, 1]) * tiny).astype(F32)
        h[:, 1] = 1.0
        g[:, 2] = (r[:, 2] * F32(2.0 ** 60)).astype(F32)
        h[:, 2] = F32(2.0 ** 60)
        g[:, 3], h[:, 3] = r[:, 3], 1.0
        return g, h

    params = dict({"max_depth": 7, "eta": 0.3, "base_score": 0.0}, **VEC)
    d = eng.DMatrix(X, label=Y, multi_target=True)
    bst = eng.train(params, d, num_boost_round=3, obj=lambda p, dm: grads(np.asarray(p, F32).reshape(n, 4)),
                    verbose_eval=False)
    ref = MO.train(params, X, Y, 3, gradients=grads)
    MO.assert_engine_matches(bst, ref)
    assert bst.predict(d, training=True, output_margin=True).tobytes() == ref.margin.tobytes()
    g, h = grads(np.zeros_like(Y))
    eg = [FS.quant_exponent(g[:, k]) for k in range(4)]
    eh = [FS.quant_exponent(h[:, k]) for k in range(4)]
    assert eg[:2] == [0, -148] and eg[2] > 60 and eh == [0, 1, 61, 1], (eg, eh)
    lv = np.concatenate([t.leaf_vector for t in ref._trees])
    assert (lv[:, 0] == 0).all() and (lv[:, 2] != 0).any() and (lv[:, 3] != 0).any()


# ------------------------------------------------------------------ raw-value prediction and pred_leaf
def held_out(ref, n, F, seed, missing):
    """rows with NaN, ±inf, every split condition (and its two neighbours) in its feature and, for a non-NaN
    missing, that value (with -0.0 for missing = 0.0)"""
    X, _ = layout_data(n, F, 1, seed)
    rng = np.random.RandomState(seed)
    X[rng.uniform(size=X.shape) < 0.03] = np.inf
    X[rng.uniform(size=X.shape) < 0.03] = -np.inf
    i = 0
    for t in ref._trees:
        for nid in np.nonzero(t.split_feature >= 0)[0]:
            c = F32(t.split_cond[nid])
            for v in (c, np.nextafter(c, F32(-np.inf)), np.nextafter(c, F32(np.inf))):
                X[i % n, t.split_feature[nid]] = v
                i += 1
    if not np.isnan(missing):
        X[rng.uniform(size=X.shape) < 0.05] = missing
        if missing == 0.0:
            X[rng.uniform(size=X.shape) < 0.03] = F32(-0.0)
    return X


@pytest.mark.parametrize("missing", [np.nan, -999.0, 0.0])
def test_predict_held_out(eng, missing):
    X, Y = layout_data(8000, 20, 3, seed=500)
    bst, ref, _ = run(eng, {"objective": "reg:squarederror", "max_depth": 7, "eta": 0.3, "base_score": 0.25}, X, Y, 5)
    Xt = held_out(ref, 4000, 20, 501, missing)
    d = eng.DMatrix(Xt, missing=missing)
    for ir in (None, (0, 2), (2, 5)):
        kw = {} if ir is None else {"iteration_range": ir}
        got = bst.predict(d, output_margin=True, **kw)
        want = MO.predict_margin(ref, Xt, missing=missing, iteration_range=ir)
        assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32)), ir
        leaf = bst.predict(d, pred_leaf=True, **kw)
        assert np.array_equal(np.asarray(leaf).astype(np.int64), MO.pred_leaf(ref, Xt, missing, ir)), ir


# ------------------------------------------------------------------ 40-bit leaf sums and the intercept past 2^24 rows
def _bits(x):
    return np.asarray(x, F32).view(np.uint32)


@pytest.mark.parametrize("n", [FS.N_CONTROL, FS.N_LARGE])
@pytest.mark.parametrize("depth", [6, 12])
def test_root_leaf_sums_exact(eng, depth, n):
    """X constant: the root is the only leaf.  With base_score 0 every g = -y sits just below -2^1, so a target's G is
    near -2^40 per row and wraps one int64 past 2^23 rows"""
    X, y1 = FS.root_case(n, seed=1)
    _, y2 = FS.root_case(n, seed=2)
    Y = np.stack([y1, y2], 1)
    params = {"objective": "reg:squarederror", "max_depth": depth, "eta": 0.3, "base_score": 0.0}
    d = eng.DMatrix(X, label=Y, multi_target=True)
    bst = eng.train(dict(params, **VEC), d, num_boost_round=1, verbose_eval=False)
    t = bst.get_trees()[0]
    assert len(t["left"]) == 1
    want = []
    for y in (y1, y2):
        g, h = FS.gradients("reg:squarederror", np.zeros(n, F32), y)
        G, H = FS.node_sums(g, h, FS.quant_exponent(g), FS.quant_exponent(h))
        want.append(FS.leaf_value(G, H))
    assert np.array_equal(_bits(t["leaf_vector"][0]), _bits(want)), (t["leaf_vector"][0], want)
    m = bst.predict(d, output_margin=True, training=True)
    assert np.array_equal(_bits(m), np.broadcast_to(_bits(F32(0.0) + np.array(want, F32)), m.shape))


@pytest.mark.parametrize("n", [FS.N_CONTROL, FS.N_LARGE])
def test_intercept_exact(eng, n):
    rng = np.random.RandomState(5)
    Y = np.stack([FS.grid_labels(rng, n, 0, 2048), FS.grid_labels(rng, n, 1024, 4096)], 1)
    params = {"objective": "reg:squarederror", "max_depth": 1}
    bst = eng.train(dict(params, **VEC), eng.DMatrix(np.zeros((n, 1), F32), label=Y, multi_target=True),
                    num_boost_round=1, verbose_eval=False)
    want = F32(MT.intercept(params, Y))
    assert _bits(F32(bst.params["base_score"])) == _bits(want), (bst.params["base_score"], want)
