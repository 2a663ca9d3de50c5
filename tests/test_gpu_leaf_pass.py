"""GPU tests of the leaf pass and of the sibling subtraction inside the split scan, against the CPU oracle.

The leaf sums come from a streaming pass over (leaf index, gradient pair) in row order up to the depth whose per-leaf
accumulators fit in shared memory, and from the gathering path above it; both must give the oracle's trees.  Sibling
histograms are formed in eval_splits_kernel and stored only for levels whose nodes are parents of the next level; with
column sampling, the stored sibling must still cover the features the level did not sample."""
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


def regression_data(n, f, seed):
    X = make_data(n, f, seed, "uniform")
    rng = np.random.RandomState(seed + 1)
    y = (X[:, : min(f, 6)].sum(axis=1) + np.sin(X[:, 0]) * 3 + rng.normal(scale=0.5, size=n)).astype(np.float32)
    return X, y


# depth 11 is the deepest tree summed by the streaming pass, 12 takes the gathering path
@pytest.mark.parametrize("depth", [1, 2, 11, 12])
def test_leaf_pass_depths(eng, oracle, depth):
    X, y = regression_data(30000, 16, 3)
    params = {"objective": "reg:squarederror", "max_depth": depth, "eta": 0.3, "base_score": 0.5, "hist_qbits": 18}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 3)
    assert_same_model(ebst, obst)
    m = ebst.predict(dm, output_margin=True, training=True)
    assert np.max(np.abs(m - obst.margin[:, 0])) <= 1e-5


def test_leaf_pass_multiclass(eng, oracle):
    n, f = 20000, 12
    X = make_data(n, f, 8, "uniform")
    y = np.clip((X[:, 0] + X[:, 1]) / 7.0, 0, 2).astype(np.int32).astype(np.float32)
    params = {"objective": "multi:softprob", "num_class": 3, "max_depth": 5, "eta": 0.3, "base_score": 0.5}
    ebst, obst, dm = run_both(eng, oracle, params, X, y, 3)
    assert_same_model(ebst, obst)
    m = ebst.predict(dm, output_margin=True, training=True).reshape(n, 3)
    assert np.max(np.abs(m - obst.margin)) <= 1e-5


def test_sibling_subtraction_with_column_sampling(eng, oracle):
    # a feature left out at level d can be scanned at level d + 1, whose parents are the siblings stored at level d
    X, y = regression_data(20000, 40, 11)
    params = {"objective": "reg:squarederror", "max_depth": 6, "eta": 0.3, "base_score": 0.5, "seed": 5,
              "colsample_bylevel": 0.5, "colsample_bynode": 0.6}
    ebst, obst, _ = run_both(eng, oracle, params, X, y, 4)
    assert_same_model(ebst, obst)
