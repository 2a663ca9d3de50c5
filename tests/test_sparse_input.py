"""scipy.sparse input without a GPU: the canonical CSR form DMatrix uploads, the RayDMatrix shards of a sparse matrix and
their /dev/shm hand-off, the densify rule the device applies to a tile, and the tile row count.

The dense twin of a sparse matrix is the same matrix with NaN in every cell it does not store; every result on a sparse
matrix must equal the result on its twin."""
import numpy as np
import pytest
import scipy.sparse as sp

from xgboost_ray_b200 import engine as E
from xgboost_ray_b200.main import _attach_shared
from xgboost_ray_b200.matrix import RayDMatrix, RayShardingMode, csr_take_rows


def twin(X):
    """Dense float32 copy with NaN in every absent cell (stored values, stored 0.0 and stored NaN kept)."""
    c = sp.coo_matrix(X)
    out = np.full(c.shape, np.nan, np.float32)
    out[c.row, c.col] = c.data.astype(np.float32)
    return out


def densify(c, r0, rows):
    """NumPy statement of csr_densify_kernel: rows [r0, r0 + rows) of a canonical CSR, NaN where a row stores nothing,
    stored bits copied unchanged."""
    out = np.full((rows, c.shape[1]), np.nan, np.float32)
    for i in range(rows):
        b, e = c.indptr[r0 + i], c.indptr[r0 + i + 1]
        out[i, c.indices[b:e]] = c.values[b:e]
    return out


def sample(n=300, f=9, density=0.2, seed=0):
    rng = np.random.RandomState(seed)
    X = sp.random(n, f, density=density, random_state=rng, format="csr", dtype=np.float64)
    X.data[::7] = 0.0          # stored zeros are values
    X.data[3::11] = np.nan     # stored NaN is missing
    return X


def same(a, b):
    return (a.shape == b.shape and np.array_equal(a.indptr, b.indptr) and np.array_equal(a.indices, b.indices)
            and np.array_equal(a.values.view(np.uint32), b.values.view(np.uint32)))


def test_canonical_form_of_every_input_format():
    X = sample()
    ref = E.canonical_csr(X)
    assert ref.indptr.dtype == np.int64 and ref.indices.dtype == np.int32 and ref.values.dtype == np.float32
    assert ref.shape == X.shape and ref.nnz == X.nnz
    int32_ptr = X.copy()
    int32_ptr.indptr = int32_ptr.indptr.astype(np.int32)
    for other in (X.tocsc(), X.tocoo(), sp.csr_array(X), sp.coo_array(X), int32_ptr, X.astype(np.float32)):
        assert same(E.canonical_csr(other), ref)
    assert np.array_equal(densify(ref, 0, X.shape[0]), twin(X), equal_nan=True)


def test_shuffled_columns_are_sorted_on_a_copy():
    X = sample(seed=3)
    ref = E.canonical_csr(X)
    shuffled = X.copy()
    rng = np.random.RandomState(5)
    for i in range(X.shape[0]):
        b, e = shuffled.indptr[i], shuffled.indptr[i + 1]
        p = b + rng.permutation(e - b)
        shuffled.indices[b:e], shuffled.data[b:e] = shuffled.indices[p].copy(), shuffled.data[p].copy()
    shuffled.has_sorted_indices = False
    before = (shuffled.indptr.copy(), shuffled.indices.copy(), shuffled.data.copy())
    assert same(E.canonical_csr(shuffled), ref)
    for a, b in zip(before, (shuffled.indptr, shuffled.indices, shuffled.data)):
        assert np.array_equal(a, b, equal_nan=True)   # the caller's matrix is untouched


def test_shape_keeps_trailing_absent_columns_and_empty_rows():
    X = sp.csr_matrix((np.array([1.0, 2.0]), np.array([0, 1]), np.array([0, 0, 2, 2])), shape=(3, 6))
    c = E.canonical_csr(X)
    assert c.shape == (3, 6)
    assert np.array_equal(densify(c, 0, 3), twin(X), equal_nan=True)
    empty = E.canonical_csr(sp.csr_matrix((4, 3), dtype=np.float32))
    assert empty.nnz == 0 and np.isnan(densify(empty, 0, 4)).all()


@pytest.mark.parametrize("fmt", ["csr", "coo", "csc"])
def test_duplicate_entry_is_refused_naming_row_and_column(fmt):
    rows, cols = np.array([0, 2, 2, 3]), np.array([1, 4, 4, 0])
    X = sp.coo_matrix((np.ones(4), (rows, cols)), shape=(5, 6))
    if fmt == "csr":   # built from raw arrays: scipy keeps the duplicate
        X = sp.csr_matrix((np.ones(4), np.array([1, 4, 4, 0]), np.array([0, 1, 1, 3, 4, 4])), shape=(5, 6))
    elif fmt == "csc":
        X = sp.csc_matrix((np.ones(4), np.array([3, 0, 2, 2]), np.array([0, 1, 2, 2, 2, 4, 4])), shape=(5, 6))
    with pytest.raises(E.XGBoostError, match="row 2 stores column 4 twice"):
        E.canonical_csr(X)


def test_densify_rule_keeps_stored_bits_and_values():
    vals = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, np.finfo(np.float32).max, -np.finfo(np.float32).max,
                     np.float32(1e-45), -999.0], np.float32)
    X = sp.csr_matrix((vals, np.arange(9) % 4, np.array([0, 4, 8, 8, 9])), shape=(4, 5))
    c = E.canonical_csr(X)
    d = densify(c, 0, 4)
    t = twin(X)
    assert np.array_equal(d.view(np.uint32), t.view(np.uint32))   # -0.0 stays -0.0, the subnormal stays
    assert np.array_equal(densify(c, 1, 3), t[1:4], equal_nan=True)


@pytest.mark.parametrize("f,rows", [(1, 67108864), (100, 670976), (4300, 15488)])
def test_tile_rows_rule(f, rows):
    r = E.raw_tile_rows(f)
    assert r == rows and r % 128 == 0 and r * 4 * f <= E.RAW_TILE_BYTES < (r + 128) * 4 * f
    assert E.raw_tile_rows(10 ** 7) == 128   # never below 128 rows


def test_csr_take_rows_equals_twin_rows():
    X = sample(n=101, f=5, seed=8)
    c = E.canonical_csr(X)
    t = twin(X)
    for rows in (slice(3, 40), slice(1, 101, 4), np.array([5, 0, 99, 5, 17]), slice(50, 50)):
        s = csr_take_rows(c, rows)
        assert np.array_equal(densify(s, 0, s.shape[0]), t[rows], equal_nan=True)


def _shard_twin(shared):
    A = _attach_shared(shared["data"])
    assert isinstance(A, sp.csr_matrix)
    return twin(A)


@pytest.mark.parametrize("mode", [RayShardingMode.INTERLEAVED, RayShardingMode.BATCH])
def test_ray_dmatrix_shards_densify_to_twin_shards(mode):
    X = sample(n=257, f=11, seed=2)
    rng = np.random.RandomState(0)
    y, w = rng.rand(257).astype(np.float32), rng.rand(257).astype(np.float32)
    m = RayDMatrix(X, y, weight=w, num_actors=3, sharding=mode)
    d = RayDMatrix(twin(X), y, weight=w, num_actors=3, sharding=mode)
    try:
        for r in range(3):
            s, t = m.get_shared(r), d.get_data(r)
            assert s["data"][0] == "csr" and all(x[0] == "shm" for x in s["data"][1:4])
            assert np.array_equal(_shard_twin(s), t["data"], equal_nan=True)
            assert np.array_equal(_attach_shared(s["label"]), t["label"])
            assert np.array_equal(_attach_shared(s["weight"]), t["weight"])
        assert m._columns == ["f%d" % i for i in range(11)]
    finally:
        m.unload_data()
        d.unload_data()


def test_ray_dmatrix_qid_groups_are_row_gathers():
    X = sample(n=200, f=6, seed=4)
    rng = np.random.RandomState(1)
    qid = np.sort(rng.randint(0, 30, size=200))[rng.permutation(200)]   # unsorted: the rows are gathered by qid
    y = rng.randint(0, 3, size=200).astype(np.float32)
    m = RayDMatrix(X, y, qid=qid, num_actors=2, sharding=RayShardingMode.BATCH)
    d = RayDMatrix(twin(X), y, qid=qid, num_actors=2, sharding=RayShardingMode.BATCH)
    try:
        for r in range(2):
            s, t = m.get_shared(r), d.get_data(r)
            assert np.array_equal(_shard_twin(s), t["data"], equal_nan=True)
            assert np.array_equal(_attach_shared(s["qid"]), t["qid"])
            assert np.array_equal(_attach_shared(s["label"]), t["label"])
        assert all(np.array_equal(a, b) for a, b in zip(m._row_index, d._row_index))
    finally:
        m.unload_data()
        d.unload_data()


def test_ray_dmatrix_refuses_named_columns_and_unsupported_inputs():
    X = sample()
    with pytest.raises(ValueError, match="`label` names the column"):
        RayDMatrix(X, "target", num_actors=1)
    with pytest.raises(ValueError, match="LIBSVM"):
        RayDMatrix("train.libsvm", num_actors=1)
    with pytest.raises(ValueError, match="list of scipy.sparse row blocks"):
        RayDMatrix([X[:10], X[10:]], num_actors=1)


def test_dmatrix_refuses_sparse_inputs_out_of_scope():
    pd = pytest.importorskip("pandas")
    X = sample()
    with pytest.raises(E.XGBoostError, match="SparseDtype"):
        E.DMatrix(pd.DataFrame.sparse.from_spmatrix(X))
    with pytest.raises(E.XGBoostError, match="list of sparse row blocks"):
        E.DMatrix([X[:10], X[10:]])

    class It:
        def __init__(self):
            self.done = False

        def reset(self):
            self.done = False

        def next(self, input_data):
            if self.done:
                return 0
            input_data(data=X)
            self.done = True
            return 1

    with pytest.raises(E.XGBoostError, match="DataIter batch"):
        E.DMatrix(It())


def test_sparse_detection_does_not_import_scipy():
    import subprocess
    import sys
    code = ("import sys, numpy as np; from xgboost_ray_b200 import engine, data_sources; "
            "assert not engine.is_sparse(np.zeros((2, 2))); data_sources.resolve_data_source(np.zeros((2, 2))); "
            "assert 'scipy.sparse' not in sys.modules and 'scipy' not in sys.modules")
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.run([sys.executable, "-c", code], check=True, cwd=root)
