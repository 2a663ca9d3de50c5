"""tests/multi_output_reference.py against the oracle and against hand-computed answers (CPU only).

  * T = 1 with min_child_weight = 0: the vector rules are the oracle's scalar tree, bit for bit;
  * Y = [y, y]: the oracle's topology, loss_chg exactly doubled, every leaf vector (v, v);
  * a hand-computed two-target example, and a target below min_child_weight getting weight 0 in a child."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import multi_output_reference as R
from tests.test_gpu_parity import make_data

F32 = np.float32


def data(n=3000, f=8, seed=0, nan_frac=0.05):
    X = make_data(n, f, seed, "uniform", nan_frac)
    Z = np.nan_to_num(X, nan=5.0)
    y = (Z[:, 0] * 0.7 + np.sin(Z[:, 1]) + np.random.RandomState(seed).normal(0, 0.3, n)).astype(F32)
    return X, y


CASES = [
    ({"objective": "reg:squarederror"}, False),
    ({"objective": "binary:logistic", "max_delta_step": 0.7}, True),
    ({"objective": "reg:squarederror", "reg_alpha": 0.5, "gamma": 0.2}, True),
    ({"objective": "reg:squarederror", "colsample_bytree": 0.8, "colsample_bylevel": 0.8, "colsample_bynode": 0.7,
      "seed": 3}, False),
]


def same_tree(o, r):
    for k in ("left", "right", "split_feature", "split_bin", "default_left"):
        assert np.array_equal(getattr(o, k), getattr(r, k)), k
    inner = o.split_feature >= 0
    assert np.array_equal(o.split_cond[inner].view(np.uint32), r.split_cond[inner].view(np.uint32))


@pytest.mark.parametrize("extra,weighted", CASES)
def test_one_target_is_the_oracle_tree(extra, weighted):
    X, y = data(seed=len(extra))
    if extra["objective"] == "binary:logistic":
        y = (y > np.median(y)).astype(F32)
    w = np.random.RandomState(1).uniform(0.5, 2.0, len(y)).astype(F32) if weighted else None
    params = dict({"max_depth": 5, "eta": 0.3, "min_child_weight": 0, "base_score": 0.5}, **extra)
    obst, _ = O.train(params, X, y, 3, weight=w)
    ref = R.train(params, X, y[:, None], 3, weight=w)
    for i in range(3):
        o, r = obst.tree(i), ref.tree(i)
        same_tree(o, r)
        assert np.array_equal(o.loss_chg, r.loss_chg)
        leaf = o.split_feature < 0
        assert np.array_equal(o.value[leaf], r.leaf_vector[leaf, 0])
    assert np.array_equal(obst.margin.reshape(-1), ref.margin[:, 0])


@pytest.mark.parametrize("extra,weighted", CASES[:2])
def test_duplicated_targets_double_the_oracle(extra, weighted):
    X, y = data(seed=7)
    if extra["objective"] == "binary:logistic":
        y = (y > np.median(y)).astype(F32)
    w = np.random.RandomState(2).uniform(0.5, 2.0, len(y)).astype(F32) if weighted else None
    params = dict({"max_depth": 6, "eta": 0.3, "min_child_weight": 0, "gamma": 0, "base_score": 0.5}, **extra)
    obst, _ = O.train(params, X, y, 3, weight=w)
    ref = R.train(params, X, np.stack([y, y], 1), 3, weight=w)
    for i in range(3):
        o, r = obst.tree(i), ref.tree(i)
        # (5e-7, 1e-6] is where doubling would cross the expand threshold: this seed has no such loss_chg
        assert not np.any((o.loss_chg > 5e-7) & (o.loss_chg <= 1e-6))
        same_tree(o, r)
        assert np.array_equal(r.loss_chg, F32(2) * o.loss_chg)
        leaf = o.split_feature < 0
        assert np.array_equal(r.leaf_vector[leaf, 0], o.value[leaf])
        assert np.array_equal(r.leaf_vector[leaf, 1], o.value[leaf])


SAMPLED = [
    {"subsample": 0.5, "seed": 11},
    {"subsample": 0.8, "colsample_bynode": 0.6, "seed": 4},
]


@pytest.mark.parametrize("extra", SAMPLED)
def test_one_target_subsampled_is_the_oracle_tree(extra):
    X, y = data(n=4000, seed=9)
    params = dict({"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "min_child_weight": 0,
                   "base_score": 0.5}, **extra)
    obst, _ = O.train(params, X, y, 4)
    ref = R.train(params, X, y[:, None], 4)
    for i in range(4):
        o, r = obst.tree(i), ref.tree(i)
        same_tree(o, r)
        assert np.array_equal(o.loss_chg, r.loss_chg)
        leaf = o.split_feature < 0
        assert np.max(np.abs(o.value[leaf] - r.leaf_vector[leaf, 0])) <= 1e-6
    assert np.max(np.abs(obst.margin.reshape(-1) - ref.margin[:, 0])) <= 1e-6
    # the draw drops rows: a tree without it is a different tree
    full = R.train(dict(params, subsample=1.0), X, y[:, None], 1)
    assert full.tree(0).n_nodes != ref.tree(0).n_nodes or not np.array_equal(full.tree(0).loss_chg, ref.tree(0).loss_chg)


def test_row_draw_keeps_the_fraction():
    keep = R.row_keep(7, 3, 0, 200000, 0.3)
    assert abs(keep.mean() - 0.3) < 0.005
    assert not np.array_equal(keep, R.row_keep(7, 4, 0, 200000, 0.3))   # a new draw per tree
    assert R.row_keep(7, 3, 0, 1000, 1.0).all()


def held_out_rows(trees, n=3000, f=8, seed=31):
    """rows with NaN, +-inf and every split condition of the trees placed in its feature (and next to it)"""
    X, _ = data(n=n, f=f, seed=seed, nan_frac=0.05)
    rng = np.random.RandomState(seed)
    X[rng.uniform(size=X.shape) < 0.03] = np.inf
    X[rng.uniform(size=X.shape) < 0.03] = -np.inf
    i = 0
    for t in trees:
        for nid in np.nonzero(t.split_feature >= 0)[0]:
            c = F32(t.split_cond[nid])
            for v in (c, np.nextafter(c, F32(-np.inf)), np.nextafter(c, F32(np.inf))):
                X[i % n, t.split_feature[nid]] = v
                i += 1
    return X


@pytest.mark.parametrize("missing", [np.nan, -999.0])
def test_one_target_predict_is_the_oracle_predict(missing):
    X, y = data(n=4000, seed=12)
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "min_child_weight": 0, "base_score": 0.5}
    obst, _ = O.train(params, X, y, 4)
    ref = R.train(params, X, y[:, None], 4)
    Xt = held_out_rows([ref.tree(i) for i in range(4)])
    if not np.isnan(missing):
        Xt[np.random.RandomState(2).uniform(size=Xt.shape) < 0.05] = missing
    want = obst.predict_margin(Xt, missing=missing)
    got = R.predict_margin(ref, Xt, missing=missing)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    for b, e in ((0, 2), (2, 4)):
        assert np.array_equal(R.predict_margin(ref, Xt, missing=missing, iteration_range=(b, e)).view(np.uint32),
                              obst.predict_margin(Xt, missing=missing, tree_begin=b, tree_end=e).view(np.uint32))
    leaves = R.pred_leaf(ref, Xt, missing=missing)
    assert leaves.shape == (len(Xt), 4)
    assert all((ref.tree(i).split_feature[leaves[:, i]] < 0).all() for i in range(4))


def test_duplicated_targets_subsampled_double_inside_the_reference():
    X, y = data(seed=17)
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "min_child_weight": 0, "gamma": 0,
              "base_score": 0.5, "subsample": 0.6, "seed": 8}
    one = R.train(params, X, y[:, None], 3)
    two = R.train(params, X, np.stack([y, y], 1), 3)
    for i in range(3):
        o, r = one.tree(i), two.tree(i)
        assert not np.any((o.loss_chg > 5e-7) & (o.loss_chg <= 1e-6))
        same_tree(o, r)
        assert np.array_equal(r.loss_chg, F32(2) * o.loss_chg)
        assert np.array_equal(r.leaf_vector[:, 0], o.leaf_vector[:, 0])
        assert np.array_equal(r.leaf_vector[:, 1], o.leaf_vector[:, 0])
    assert np.array_equal(two.margin[:, 0], one.margin[:, 0]) and np.array_equal(two.margin[:, 1], one.margin[:, 0])


def test_hand_computed_two_targets():
    # one feature, four rows with values 0..3; target 0 wants the split 0|123, target 1 the split 012|3; summed, the
    # first of the two tied best candidates wins (hand computation below); squared error at margin 0, lambda = 0, eta = 1
    X = np.array([[0.0], [1.0], [2.0], [3.0]], F32)
    Y = np.array([[-3.0, 0.0], [1.0, 0.0], [1.0, 0.0], [1.0, 4.0]], F32)
    params = {"objective": "reg:squarederror", "max_depth": 1, "eta": 1.0, "lambda": 0.0, "min_child_weight": 0,
              "base_score": 0.0}
    ref = R.train(params, X, Y, 1)
    t = ref.tree(0)
    # g = -y, h = 1, w = -G/H.  Parent gains: t0 G=0 -> 0; t1 G=-4,H=4 -> 4.  Candidates (left = rows <= bin):
    #   bin 0: t0 L(3,1) R(-3,3) -> 9+3 = 12; t1 L(0,1) R(-4,3) -> 16/3; total 12 + 16/3 - 4 = 13.333
    #   bin 1: t0 L(2,2) R(-2,2) -> 2+2 = 4;  t1 L(0,2) R(-4,2) -> 8;    total 12 - 4 = 8
    #   bin 2: t0 L(1,3) R(-1,1) -> 1/3+1;    t1 L(0,3) R(-4,1) -> 16;   total 17.333 - 4 = 13.333
    # bins 0 and 2 tie at 40/3 in fp32; the earlier candidate wins
    assert t.split_feature[0] == 0 and t.split_bin[0] == 0
    assert t.loss_chg[0] == F32(12.0 + 16.0 / 3.0 - 4.0)
    assert np.array_equal(t.leaf_vector[t.left[0]], F32([-3.0, 0.0]))
    assert np.array_equal(t.leaf_vector[t.right[0]], F32([1.0, 4.0 / 3.0]))


def test_target_below_min_child_weight_gets_weight_zero():
    # target 1's hessians are 0.1 per row: with min_child_weight = 1, a child with fewer than 10 rows has H_1 < 1, so
    # target 1 adds 0 to the gain there and its leaf value is 0
    X = np.arange(40, dtype=F32)[:, None]
    y0 = np.where(np.arange(40) < 5, -5.0, 1.0).astype(F32)
    y1 = np.linspace(-1, 1, 40).astype(F32)

    def grads(margin):
        g = np.stack([margin[:, 0] - y0, F32(0.1) * (margin[:, 1] - y1)], 1).astype(F32)
        h = np.stack([np.ones(40, F32), np.full(40, 0.1, F32)], 1)
        return g, h

    params = {"max_depth": 1, "eta": 1.0, "min_child_weight": 1.0, "base_score": 0.0}
    ref = R.train(params, X, np.zeros((40, 2), F32), 1, gradients=grads)
    t = ref.tree(0)
    assert t.split_bin[0] == 4            # the 5 rows of target 0's step go left
    assert t.leaf_vector[t.left[0], 1] == 0.0
    assert t.leaf_vector[t.right[0], 1] != 0.0
    assert t.leaf_vector[t.left[0], 0] != 0.0
