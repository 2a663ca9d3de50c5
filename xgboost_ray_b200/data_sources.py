"""Data-source adapters for RayDMatrix: numpy, pandas, scipy.sparse, CSV, Parquet (single file or list of files).

Mirrors the adapter registry of the reference (xgboost_ray/data_sources/__init__.py:13-24,
data_source.py:22-155, numpy.py:13-33, pandas.py:8-30, csv.py:9-47, parquet.py:9-48).  The
third-party distributed-dataframe sources (Modin, Dask, Petastorm, Ray Datasets, object store,
__partitioned__) are out of scope on a single 8xH100 box (SURVEY.md 2 #14).

Unlike the reference every adapter loads straight into a float32 C-contiguous numpy block plus
named side columns -- that is what the device upload wants -- instead of a pandas frame.
"""
import os
from enum import Enum
from typing import Any, List, Optional, Sequence

import numpy as np


class RayFileType(Enum):
    """Known file types (xgboost_ray/data_sources/data_source.py:14-19)."""
    CSV = 1
    PARQUET = 2
    PETASTORM = 3


class LoadedFrame:
    """Column-named float32 table: `values` [n, c] C-contiguous and `columns` names."""

    def __init__(self, values: np.ndarray, columns: List[str], feature_types: Optional[List[str]] = None):
        self.values = np.ascontiguousarray(values, dtype=np.float32)
        self.columns = [str(c) for c in columns]
        # per column 'c' (pandas `category` dtype, stored as its codes) or 'q'; None = all numeric
        self.feature_types = list(feature_types) if feature_types is not None and "c" in feature_types else None

    def __len__(self):
        return self.values.shape[0]

    def column(self, name):
        return self.values[:, self.columns.index(str(name))]

    def drop(self, names):
        keep = [i for i, c in enumerate(self.columns) if c not in set(map(str, names))]
        types = [self.feature_types[i] for i in keep] if self.feature_types else None
        return LoadedFrame(self.values[:, keep], [self.columns[i] for i in keep], types)


def _from_pandas(df, ignore=None, indices=None):
    if ignore:
        df = df[[c for c in df.columns if c not in set(ignore)]]
    if indices is not None:
        df = df.iloc[indices]
    if not hasattr(df, "to_numpy"):
        return LoadedFrame(np.asarray(df), list(df.columns))
    is_cat = [str(dt) == "category" for dt in df.dtypes]
    if not any(is_cat):
        return LoadedFrame(df.to_numpy(dtype=np.float32, na_value=np.nan), list(df.columns))
    # xgboost's pandas adapter (xgb.DMatrix(df, enable_categorical=True), reached through main.py:437): a `category`
    # column is its integer codes, code -1 (NaN) is a missing value; the column is typed 'c'
    out = np.empty((len(df), len(df.columns)), np.float32)
    for j, (c, cat) in enumerate(zip(df.columns, is_cat)):
        if cat:
            codes = df[c].cat.codes.to_numpy().astype(np.float32)
            codes[codes < 0] = np.nan
            out[:, j] = codes
        else:
            out[:, j] = df[c].to_numpy(dtype=np.float32, na_value=np.nan)
    return LoadedFrame(out, list(df.columns), ["c" if cat else "q" for cat in is_cat])


class DataSource:
    supports_central_loading = True
    supports_distributed_loading = False
    needs_partitions = True

    @staticmethod
    def is_data_type(data: Any, filetype: Optional[RayFileType] = None) -> bool:
        return False

    @staticmethod
    def get_filetype(data: Any) -> Optional[RayFileType]:
        return None

    @staticmethod
    def load_data(data, ignore=None, indices=None, **kwargs) -> LoadedFrame:
        raise NotImplementedError

    @staticmethod
    def get_n(data: Any) -> int:
        return len(data)


class Numpy(DataSource):
    @staticmethod
    def is_data_type(data, filetype=None):
        return isinstance(data, np.ndarray)

    @staticmethod
    def load_data(data, ignore=None, indices=None, **kwargs):
        a = data if data.ndim == 2 else data.reshape(-1, 1)
        if indices is not None:
            a = a[indices]
        fr = LoadedFrame(a, ["f%d" % i for i in range(a.shape[1])])
        return fr.drop(ignore) if ignore else fr


class Pandas(DataSource):
    @staticmethod
    def is_data_type(data, filetype=None):
        try:
            import pandas as pd
        except ImportError:
            return False
        return isinstance(data, (pd.DataFrame, pd.Series))

    @staticmethod
    def load_data(data, ignore=None, indices=None, **kwargs):
        import pandas as pd
        if isinstance(data, pd.Series):
            data = data.to_frame()
        return _from_pandas(data, ignore, indices)


def _is_path_like(data, ext):
    if isinstance(data, str):
        return data.endswith(ext)
    if isinstance(data, (list, tuple)) and data and all(isinstance(d, str) for d in data):
        return all(d.endswith(ext) for d in data)
    return False


def _paths(data, indices=None) -> List[str]:
    paths = [data] if isinstance(data, str) else list(data)
    if indices is not None:
        paths = [paths[i] for i in indices]
    out = []
    for p in paths:
        if os.path.isdir(p):
            out.extend(sorted(os.path.join(p, f) for f in os.listdir(p) if not f.startswith(".")))
        else:
            out.append(p)
    return out


class CSV(DataSource):
    supports_distributed_loading = True
    needs_partitions = False

    @staticmethod
    def is_data_type(data, filetype=None):
        return filetype == RayFileType.CSV or _is_path_like(data, ".csv")

    @staticmethod
    def get_filetype(data):
        return RayFileType.CSV if _is_path_like(data, ".csv") else None

    @staticmethod
    def load_data(data, ignore=None, indices=None, **kwargs):
        import pandas as pd
        frames = [pd.read_csv(p, **kwargs) for p in _paths(data, indices)]
        return _from_pandas(pd.concat(frames, ignore_index=True) if len(frames) > 1 else frames[0], ignore)

    @staticmethod
    def get_n(data):
        return 1 if isinstance(data, str) else len(data)


class Parquet(DataSource):
    supports_distributed_loading = True
    needs_partitions = False

    @staticmethod
    def is_data_type(data, filetype=None):
        return filetype == RayFileType.PARQUET or _is_path_like(data, ".parquet")

    @staticmethod
    def get_filetype(data):
        return RayFileType.PARQUET if _is_path_like(data, ".parquet") else None

    @staticmethod
    def load_data(data, ignore=None, indices=None, **kwargs):
        import pyarrow.parquet as pq
        cols = kwargs.pop("columns", None)
        tables = [pq.read_table(p, columns=cols) for p in _paths(data, indices)]
        names = tables[0].column_names
        blocks = []
        for t in tables:
            blocks.append(np.column_stack([t.column(c).to_numpy(zero_copy_only=False).astype(np.float32, copy=False)
                                           for c in names]) if t.num_rows else np.zeros((0, len(names)), np.float32))
        fr = LoadedFrame(np.concatenate(blocks, axis=0) if len(blocks) > 1 else blocks[0], names)
        return fr.drop(ignore) if ignore else fr

    @staticmethod
    def get_n(data):
        return 1 if isinstance(data, str) else len(data)


class Sparse(DataSource):
    """A scipy.sparse matrix or array (CSR, CSC, COO), loaded centrally.  RayDMatrix keeps it in CSR form and shards
    it by rows; it is never densified on the host."""
    needs_partitions = True

    @staticmethod
    def is_data_type(data, filetype=None):
        from xgboost_ray_b200.engine import is_sparse
        return is_sparse(data)

    @staticmethod
    def load_data(data, ignore=None, indices=None, **kwargs):
        from xgboost_ray_b200.engine import canonical_csr
        if ignore:
            raise ValueError("`ignore` names columns, but a scipy.sparse matrix has none (got %r)" % (ignore,))
        return canonical_csr(data)

    @staticmethod
    def get_n(data):
        return data.shape[0]


data_sources = [Numpy, Pandas, Sparse, CSV, Parquet]


def resolve_data_source(data, filetype=None):
    if _is_path_like(data, ".libsvm") or _is_path_like(data, ".svm"):
        raise ValueError("LIBSVM text files are not supported (%r): load them with "
                         "sklearn.datasets.load_svmlight_file and pass the scipy.sparse matrix" % (data,))
    if isinstance(data, (list, tuple)) and data and any(Sparse.is_data_type(d) for d in data):
        raise ValueError("a list of scipy.sparse row blocks is not supported: pass one matrix (scipy.sparse.vstack)")
    for src in data_sources:
        if src.is_data_type(data, filetype):
            return src
    raise ValueError(
        "Unknown data source type: %s with FileType: %s.\nFIX THIS by passing a numpy array, a pandas "
        "DataFrame/Series, a scipy.sparse matrix, or CSV / Parquet file name(s) (Modin/Dask/Petastorm/Ray datasets are out of scope "
        "of the single-node H100 build)." % (type(data), filetype))
