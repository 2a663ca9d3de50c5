"""DMatrix(bin_layout=...) and RayDMatrix(bin_layout=...): the argument is checked before anything reaches a device."""
import numpy as np
import pytest
import scipy.sparse as sp

from xgboost_ray_b200 import engine


@pytest.mark.parametrize("bad", ["columnar", "CSR", "", None, 2])
def test_unknown_layout_is_refused(bad):
    with pytest.raises(engine.XGBoostError, match="bin_layout must be one of 'auto', 'dense', 'csr'"):
        engine.DMatrix(sp.csr_matrix(np.eye(4, dtype=np.float32)), bin_layout=bad)


@pytest.mark.parametrize("data", [np.zeros((6, 3), np.float32), [np.zeros((2, 3), np.float32)] * 3])
def test_csr_layout_needs_sparse_input(data):
    with pytest.raises(engine.XGBoostError, match='bin_layout="csr" needs a scipy.sparse matrix'):
        engine.DMatrix(data, bin_layout="csr")


def test_ray_dmatrix_checks_the_layout():
    from xgboost_ray_b200 import RayDMatrix
    with pytest.raises(engine.XGBoostError, match="bin_layout"):
        RayDMatrix(sp.csr_matrix(np.eye(4, dtype=np.float32)), np.zeros(4, np.float32), bin_layout="sparse")
    m = RayDMatrix(sp.csr_matrix(np.eye(4, dtype=np.float32)), np.zeros(4, np.float32), bin_layout="csr")
    from xgboost_ray_b200.main import _matrix_meta
    assert _matrix_meta(m)["bin_layout"] == "csr"
