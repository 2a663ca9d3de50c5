"""GPU tests of the split scan (eval_splits_kernel: one CTA per 4 feature slots of a node) and of the level decision
taken by the scan's last CTA, against the CPU oracle.

The scan grid is the level's upper bound of nodes; CTAs past the real node count only take their ticket, and the CTA
that completes the grid resets the counter and decides.  A level whose nodes all stop, a level with no node at all and
many graph-replayed trees in a row must all leave the counter at zero for the next level and the next tree."""
import numpy as np
import pytest

from tests.test_gpu_parity import assert_same_model, make_data, run_both

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def regression_data(n, f, seed, nan_frac=0.0):
    X = make_data(n, f, seed, "uniform", nan_frac)
    rng = np.random.RandomState(seed + 1)
    Z = np.nan_to_num(X, nan=5.0)
    y = (Z[:, : min(f, 6)].sum(axis=1) + np.sin(Z[:, 0]) * 3 + rng.normal(scale=0.5, size=n)).astype(np.float32)
    return X, y


def split_counts(bst):
    return [int(np.sum(t["split_feature"] >= 0)) for t in bst.get_trees()]


# feature counts around the 4-slot CTA: fewer than 4, not a multiple of 4, one full group, a partial last group
@pytest.mark.parametrize("f", [1, 3, 5, 32, 37, 70])
def test_scan_feature_counts(eng, oracle, f):
    X, y = regression_data(20000, f, 2)
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5}
    ebst, obst, _ = run_both(eng, oracle, params, X, y, 3)
    assert_same_model(ebst, obst)


def test_levels_that_stop_early(eng, oracle):
    # gamma prunes most nodes: the upper-bound grid has CTAs past the real node count, and trees stop before max_depth,
    # so later levels have no node at all; six graph-replayed trees must keep deciding correctly
    X, y = regression_data(30000, 20, 4)
    params = {"objective": "reg:squarederror", "max_depth": 8, "eta": 0.3, "base_score": 0.5, "gamma": 400.0}
    ebst, obst, _ = run_both(eng, oracle, params, X, y, 6)
    assert_same_model(ebst, obst)
    counts = split_counts(ebst)
    assert min(counts) < 2 ** 8 - 1, counts    # some level did not split every node
    assert max(counts) > 0, counts


def test_no_split_at_root(eng, oracle):
    # min_child_weight above the total hessian: the root's level decides that nothing splits
    X, y = regression_data(5000, 12, 6)
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5, "min_child_weight": 1e5}
    ebst, obst, _ = run_both(eng, oracle, params, X, y, 3)
    assert_same_model(ebst, obst)
    assert split_counts(ebst) == [0, 0, 0]


def test_graph_replayed_trees(eng, oracle):
    X, y = regression_data(40000, 100, 9)
    params = {"objective": "reg:squarederror", "max_depth": 8, "eta": 0.3, "base_score": 0.5}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 8)
    assert_same_model(ebst, obst)
    m = ebst.predict(dm, output_margin=True, training=True)
    assert np.max(np.abs(m - obst.margin[:, 0])) <= 1e-5


def test_missing_values_both_directions(eng, oracle):
    X, y = regression_data(30000, 24, 12, nan_frac=0.15)
    # rows missing on feature 0 get a high label: the missing rows go right at some splits and left at others
    y = y + np.where(np.isnan(X[:, 0]), 20.0, 0.0).astype(np.float32) - np.where(np.isnan(X[:, 1]), 20.0, 0.0).astype(np.float32)
    params = {"objective": "reg:squarederror", "max_depth": 7, "eta": 0.3, "base_score": 0.5}
    ebst, obst, _ = run_both(eng, oracle, params, X, y, 4)
    assert_same_model(ebst, obst)
    dl = np.concatenate([t["default_left"][t["split_feature"] >= 0] for t in ebst.get_trees()])
    assert dl.min() == 0 and dl.max() == 1


def test_colsample_bynode_with_stored_siblings(eng, oracle):
    # siblings are stored at levels 1 .. depth - 2 with every slot, including features the node did not sample
    X, y = regression_data(30000, 70, 13)
    params = {"objective": "reg:squarederror", "max_depth": 7, "eta": 0.3, "base_score": 0.5, "seed": 3,
              "colsample_bynode": 0.4}
    ebst, obst, _ = run_both(eng, oracle, params, X, y, 4)
    assert_same_model(ebst, obst)
