"""ctypes binding of libb2hist.so + the `xgboost`-shaped objects the actor code uses.

This module is the import seam the reference keeps in ``xgboost_ray/xgb.py:1-11``: the names
``DMatrix``, ``QuantileDMatrix``, ``DeviceQuantileDMatrix``, ``Booster``, ``train``,
``collective.CommunicatorContext`` and ``callback.TrainingCallback`` are what
``xgboost_ray/main.py`` uses from the ``xgboost`` package (sites main.py:386, 418, 437, 724,
745-752, 804; session.py:73), re-implemented on top of the sm_90a engine (include/b2hist.h).

There is NO CPU fallback: if the CUDA extension is not built or no H100 is visible, the first
compute call raises ``XGBoostError``.
"""
import ast
import base64
import ctypes as C
import json
import numbers
import operator
import os
import sys
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libb2hist.so")


class XGBoostError(RuntimeError):
    """Engine error (same role as xgboost.core.XGBoostError, caught at main.py:770-772)."""


B2Error = XGBoostError

_lib = None
_lib_lock = threading.Lock()

_FP = C.POINTER(C.c_float)
_IP = C.POINTER(C.c_int32)
_BP = C.POINTER(C.c_uint8)
_DP = C.POINTER(C.c_double)
_LP = C.POINTER(C.c_int64)
_H = C.c_uint64
_FLT_MAX = np.finfo(np.float32).max


class B2Tree(C.Structure):
    """One tree as B2_BoosterAddTree takes it and B2_BoosterGetTree fills it (include/b2hist.h).  Its arrays are named
    as the keys of a tree dict; each is a void pointer here (a typed ctypes pointer costs microseconds per array, per
    tree, to make) and DTYPES gives its element type."""
    DTYPES = {"left": np.int32, "right": np.int32, "parent": np.int32, "split_feature": np.int32, "split_bin": np.int32,
              "split_cond": np.float32, "default_left": np.uint8, "value": np.float32, "base_weight": np.float32,
              "loss_chg": np.float32, "sum_hess": np.float64, "split_type": np.uint8, "cat_bits": np.uint32,
              "leaf_vector": np.float32}
    _fields_ = [("n_nodes", C.c_int32)] + [(k, C.c_void_p) for k in DTYPES] + [("leaf_vector_len", C.c_int64)]
    OPTIONAL = ("split_type", "cat_bits", "leaf_vector")   # NULL when the tree dict has none

    @classmethod
    def of(cls, t):
        """The record of tree dict t, and the arrays it points into (which must outlive its use)."""
        arrays = [None if k in cls.OPTIONAL and t.get(k) is None else np.ascontiguousarray(t[k], dt)
                  for k, dt in cls.DTYPES.items()]
        vec = arrays[-1]
        return cls(arrays[0].size, *[None if a is None else a.ctypes.data for a in arrays],
                   0 if vec is None else vec.size), arrays


# name -> (restype, argtypes); every symbol declared in include/b2hist.h
ABI = {
    "B2_GetLastError": (C.c_char_p, []),
    "B2_GetVersion": (C.c_int, []),
    "B2_CheckParams": (C.c_int, [C.c_char_p]),
    "B2_DeviceCount": (C.c_int, [C.POINTER(C.c_int)]),
    "B2_GetUniqueId": (C.c_int, [_BP]),
    "B2_CommCreate": (C.c_int, [_BP, C.c_int, C.c_int, C.c_int, C.POINTER(_H)]),
    "B2_CommRank": (C.c_int, [_H, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "B2_CommAllReduce": (C.c_int, [_H, _DP, C.c_int32, C.c_int32]),
    "B2_CommAbort": (C.c_int, [_H]),
    "B2_CommFree": (C.c_int, [_H]),
    "B2_MatrixCreateFromDense": (C.c_int, [_FP, C.c_int64, C.c_int32, C.c_float, C.c_int, C.POINTER(_H)]),
    "B2_MatrixCreate": (C.c_int, [C.c_int64, C.c_int32, C.c_float, C.c_int, C.POINTER(_H)]),
    "B2_MatrixCreateFromCSR": (C.c_int, [_LP, _IP, _FP, C.c_int64, C.c_int32, C.c_int64, C.c_float, C.c_int,
                                         C.POINTER(_H)]),
    "B2_MatrixCreateFromProcessInterleaved": (C.c_int, [C.c_int64, C.c_uint64, C.c_int64, C.c_int32, C.c_int32, _H,
                                                        C.c_float, C.c_int, C.POINTER(_H)]),
    "B2_MatrixCreateFromProcess": (C.c_int, [C.c_int64, C.c_uint64, C.c_int64, C.c_int64, C.c_int32, C.c_float, C.c_int,
                                             C.POINTER(_H)]),
    "B2_MatrixSetRows": (C.c_int, [_H, C.c_int64, _FP, C.c_int64]),
    "B2_MatrixSetFloatInfo": (C.c_int, [_H, C.c_char_p, _FP, C.c_int64]),
    "B2_MatrixSetLabel": (C.c_int, [_H, _FP, C.c_int64, C.c_int32]),
    "B2_MatrixSetGroups": (C.c_int, [_H, _IP, C.c_int64]),
    "B2_MatrixSetFeatureTypes": (C.c_int, [_H, _BP, C.c_int32]),
    "B2_MatrixGetFeatureTypes": (C.c_int, [_H, _BP]),
    "B2_MatrixNumRow": (C.c_int, [_H, C.POINTER(C.c_int64)]),
    "B2_MatrixNumCol": (C.c_int, [_H, C.POINTER(C.c_int32)]),
    "B2_MatrixQuantize": (C.c_int, [_H, _H, C.c_int32, _H, C.c_int32]),
    "B2_MatrixQuantizeWithCuts": (C.c_int, [_H, _H, _IP, _FP, _FP, _BP, C.c_int32, C.c_int32]),
    "B2_MatrixEnsureRaw": (C.c_int, [_H, _FP]),
    "B2_MatrixEnsureRawCSR": (C.c_int, [_H, _LP, _IP, _FP]),
    "B2_MatrixSlice": (C.c_int, [_H, _LP, C.c_int64, C.POINTER(_H)]),
    "B2_MatrixDeviceBytes": (C.c_int, [_H, C.POINTER(C.c_int64)]),
    "B2_MatrixCutsSize": (C.c_int, [_H, _IP]),
    "B2_MatrixGetCuts": (C.c_int, [_H, _IP, _FP, _FP, _BP]),
    "B2_MatrixGetBins": (C.c_int, [_H, _BP]),
    "B2_MatrixSetBinLayout": (C.c_int, [_H, C.c_int32]),
    "B2_MatrixFree": (C.c_int, [_H]),
    "B2_BoosterCreate": (C.c_int, [C.c_char_p, _H, _H, C.POINTER(_H)]),
    "B2_BoosterSetParam": (C.c_int, [_H, C.c_char_p]),
    "B2_BoosterUpdateOneIter": (C.c_int, [_H, C.c_int32]),
    "B2_BoosterBoostOneIter": (C.c_int, [_H, _FP, _FP, C.c_int64]),
    "B2_BoosterRefreshOneIter": (C.c_int, [_H, _FP, _FP, C.c_int64]),
    "B2_BoosterGetGradients": (C.c_int, [_H, _FP, _FP, C.c_int64]),
    "B2_BoosterEvalSet": (C.c_int, [_H, _H, C.c_char_p, _DP]),
    "B2_BoosterPredict": (C.c_int, [_H, _H, C.c_int32, C.c_int32, C.c_int32, _FP, C.c_int64]),
    "B2_BoosterPredictContribs": (C.c_int, [_H, _H, C.c_int32, C.c_int32, C.c_int32, _FP, C.c_int64]),
    "B2_BoosterPredictLeaf": (C.c_int, [_H, _H, C.c_int32, C.c_int32, _FP, C.c_int64]),
    "B2_BoosterGetTrainMargin": (C.c_int, [_H, C.c_int32, _FP, C.c_int64]),
    "B2_BoosterResetTrainMargin": (C.c_int, [_H]),
    "B2_BoosterGetBaseScore": (C.c_int, [_H, _FP, _IP]),
    "B2_BoosterNumTargets": (C.c_int, [_H, _IP]),
    "B2_BoosterNumTrees": (C.c_int, [_H, _IP]),
    "B2_BoosterTreeNumNodes": (C.c_int, [_H, C.c_int32, _IP]),
    "B2_BoosterGetTree": (C.c_int, [_H, C.c_int32, C.POINTER(B2Tree)]),
    "B2_BoosterAddTree": (C.c_int, [_H, C.POINTER(B2Tree)]),
    "B2_BoosterGetTreeWeights": (C.c_int, [_H, _FP, C.c_int64]),
    "B2_BoosterSetTreeWeights": (C.c_int, [_H, _FP, C.c_int64]),
    "B2_BoosterGetTimers": (C.c_int, [_H, C.c_int32, C.c_char_p, C.c_int64]),
    "B2_BoosterCancel": (C.c_int, [_H]),
    "B2_BoosterFree": (C.c_int, [_H]),
    "B2_HistBuildRaw": (C.c_int, [_BP, C.c_int64, C.c_int32, _IP, _IP, _IP, C.c_int64, C.c_int32, C.c_int32, C.c_int,
                                  C.POINTER(C.c_int64), _FP]),
    "B2_HistBuildRawCSR": (C.c_int, [_LP, _IP, _BP, C.c_int64, C.c_int32, _IP, _IP, _IP, C.c_int64, C.c_int32, C.c_int,
                                     C.POINTER(C.c_int64), _FP]),
    "B2_QuantizeRaw": (C.c_int, [_FP, _FP, C.c_int64, C.c_int32, C.c_int, _IP, _IP]),
}


def lib():
    """Load libb2hist.so (built by ``python -m xgboost_ray_b200.build``).  Fails loudly."""
    global _lib
    with _lib_lock:
        if _lib is None:
            if not os.path.exists(_LIB_PATH):
                raise XGBoostError(
                    "CUDA extension %s is missing: run `python -m xgboost_ray_b200.build` "
                    "(there is no CPU fallback)" % _LIB_PATH)
            L = C.CDLL(_LIB_PATH)
            for name, (res, args) in ABI.items():
                fn = getattr(L, name)
                fn.restype = res
                fn.argtypes = args
            _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise XGBoostError(lib().B2_GetLastError().decode("utf-8", "replace"))


def device_count():
    n = C.c_int(0)
    _check(lib().B2_DeviceCount(C.byref(n)))
    return n.value


def _default_device():
    return int(os.environ.get("B2_DEVICE", "0"))


def _f32c(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _fp(a):
    return a.ctypes.data_as(_FP) if a is not None else None


def _ip(a):
    return a.ctypes.data_as(_IP) if a is not None else None


def _bp(a):
    return a.ctypes.data_as(_BP) if a is not None else None


# ----------------------------------------------------------------------------- communicator
class _CollectiveState(threading.local):
    def __init__(self):
        self.handle = 0
        self.rank = 0
        self.world = 1


_coll = _CollectiveState()


def get_unique_id():
    """Driver side: the NCCL unique id that takes the `rabit_args` slot (main.py:273-283)."""
    buf = (C.c_uint8 * 128)()
    _check(lib().B2_GetUniqueId(buf))
    return bytes(buf)


class CommunicatorContext:
    """Actor side: enter/exit the NCCL communicator (replaces xgboost.collective.CommunicatorContext
    used by _RabitContext, main.py:308-324 / :724).  args: b2_uid (bytes), b2_rank, b2_world."""

    def __init__(self, **args):
        self.args = args
        self.handle = 0

    def __enter__(self):
        world = int(self.args.get("b2_world", 1))
        rank = int(self.args.get("b2_rank", 0))
        if world > 1:
            uid = self.args["b2_uid"]
            buf = (C.c_uint8 * 128).from_buffer_copy(uid)
            h = _H(0)
            _check(lib().B2_CommCreate(buf, rank, world, int(self.args.get("b2_device", _default_device())),
                                       C.byref(h)))
            self.handle = h.value
        self.rank, self.world = rank, world
        _coll.handle, _coll.rank, _coll.world = self.handle, rank, world
        return self

    def activate(self):
        """Make an already entered communicator the current one of THIS thread (an actor keeps a healthy communicator
        across train() calls; every call trains on a fresh thread and the collective state is thread-local)."""
        _coll.handle, _coll.rank, _coll.world = self.handle, self.rank, self.world
        return self

    def abort(self):
        if self.handle:
            lib().B2_CommAbort(self.handle)

    def __exit__(self, *exc):
        if self.handle:
            lib().B2_CommFree(self.handle)
            self.handle = 0
        _coll.handle, _coll.rank, _coll.world = 0, 0, 1
        return False


class collective:  # namespace shim: xgb.collective.get_rank() (session.py:73)
    CommunicatorContext = CommunicatorContext

    @staticmethod
    def get_rank():
        return _coll.rank

    @staticmethod
    def get_world_size():
        return _coll.world

    @staticmethod
    def allreduce(data, op="sum"):
        """xgb.collective.allreduce over the actors' communicator (float64; op: sum / max / min)."""
        a = np.ascontiguousarray(np.asarray(data, np.float64)).copy()
        flat = a.reshape(-1)
        _check(lib().B2_CommAllReduce(_coll.handle, flat.ctypes.data_as(_DP), flat.size, {"sum": 0, "max": 1, "min": 2}[op]))
        return a


# ----------------------------------------------------------------------------- sparse input
def is_sparse(data):
    """True for a scipy.sparse matrix or array.  scipy is never imported here: a caller holding one has imported it."""
    sp = sys.modules.get("scipy.sparse")
    return sp is not None and sp.issparse(data)


class CSRArrays:
    """The canonical CSR form of a sparse input: int64 `indptr` [n+1], int32 `indices` and float32 `values` [nnz], the
    columns of every row strictly increasing, and the input's `shape` (trailing columns that store nothing count)."""

    def __init__(self, indptr, indices, values, shape):
        self.indptr, self.indices, self.values = indptr, indices, values
        self.shape = (int(shape[0]), int(shape[1]))
        self.ndim = 2

    @property
    def nnz(self):
        return int(self.indices.size)


RAW_TILE_BYTES = 256 << 20   # host.h kRawTileBytes


def raw_tile_rows(n_cols):
    """Rows of one dense tile the device densifies from a CSR matrix of n_cols columns (host.h raw_tile_rows): at most
    RAW_TILE_BYTES of float32, a multiple of 128 rows, at least 128."""
    return max(RAW_TILE_BYTES // (4 * int(n_cols)) // 128 * 128, 128)


def _cast(a, dtype):
    """`a` C-contiguous with `dtype`; the array itself when it already is (no copy)."""
    return np.ascontiguousarray(a, dtype=dtype)


def canonical_csr(X):
    """CSR / CSC / COO (matrix or array) -> CSRArrays.  The caller's matrix is never modified: a conversion or a sort
    of the columns works on a copy.  A (row, column) stored twice is refused (a COO matrix is converted without summing
    its duplicates, so they are refused too)."""
    if X.ndim != 2:
        raise XGBoostError("DMatrix data must be 2-dimensional, got a sparse input of shape %s" % (X.shape,))
    n, f = X.shape
    if X.format == "coo":
        row, col = np.asarray(X.row, np.int64), np.asarray(X.col, np.int64)
        order = np.lexsort((col, row))
        indptr = np.zeros(n + 1, np.int64)
        np.cumsum(np.bincount(row, minlength=n), out=indptr[1:])
        indices, values = _cast(col[order], np.int32), _cast(np.asarray(X.data)[order], np.float32)
    else:
        X = X.tocsr()   # CSC: a transposed copy; CSR: the matrix itself
        indptr, indices, values = _cast(X.indptr, np.int64), _cast(X.indices, np.int32), _cast(X.data, np.float32)
        if indptr.size != n + 1 or indices.size != int(indptr[-1]) or values.size != indices.size:
            raise XGBoostError("sparse input: inconsistent CSR arrays (%d row pointers, %d columns, %d values for %d rows)"
                               % (indptr.size, indices.size, values.size, n))
        step = _row_steps(indptr, indices)
        if step.size and step.min() < 0:   # unsorted columns within a row: sort a copy
            Xs = X.sorted_indices()
            indices, values = _cast(Xs.indices, np.int32), _cast(Xs.data, np.float32)
    step = _row_steps(indptr, indices)
    if step.size and step.min() <= 0:
        k = int(np.flatnonzero(step <= 0)[0])
        r = int(np.searchsorted(indptr, k, side="right")) - 1
        raise XGBoostError("sparse input: row %d stores column %d twice" % (r, int(indices[k])))
    if indices.size and (int(indices.min()) < 0 or int(indices.max()) >= f):
        raise XGBoostError("sparse input: a column index is outside [0, %d)" % f)
    return CSRArrays(indptr, indices, values, (n, f))


def _row_steps(indptr, indices):
    """indices[k + 1] - indices[k] for the consecutive entries k, k + 1 of one row (positions that end a row hold 1)."""
    if indices.size < 2:
        return np.zeros(0, np.int64)
    step = np.diff(indices.astype(np.int64))
    ends = indptr[1:-1]
    ends = ends[(ends > 0) & (ends < indices.size)] - 1
    step[ends] = 1
    return step


# ----------------------------------------------------------------------------- DMatrix
# DMatrix(bin_layout=...): how a quantised matrix keeps its bins (B2_MatrixSetBinLayout, DESIGN.md 2 item 26)
BIN_LAYOUTS = {"auto": 0, "dense": 1, "csr": 2}


def bin_layout_code(bin_layout):
    if not isinstance(bin_layout, str) or bin_layout not in BIN_LAYOUTS:
        raise XGBoostError("bin_layout must be one of %s, got %r" % (", ".join(map(repr, BIN_LAYOUTS)), bin_layout))
    return BIN_LAYOUTS[bin_layout]


class DMatrix:
    """Device matrix.  Float data is uploaded at construction; quantisation (GPU sketch + binning)
    happens when a Booster first trains on it, because cuts are global over the communicator.

    multi_target=True accepts a label of shape (n, T), T > 1: multi-target regression or multi-label classification,
    one tree per column and round.  Without it a label of several columns is refused, so that a label of the wrong
    shape (one-hot classes, a target passed twice) is not trained as T independent outputs.  RayDMatrix and the sklearn
    estimators, whose users ask for several label columns explicitly, set it for them.

    bin_layout chooses how the quantised bins are kept on the device.  "dense": two n x F byte copies.  "csr" (a
    scipy.sparse input only): one byte per stored entry, next to the CSR's column indices, so that a sparse matrix whose
    dense bins would not fit the GPU still trains; the model is byte-identical to the dense layout's.  "auto" (the
    default) takes "csr" only when the two dense copies would exceed half of the device's memory."""

    def __init__(self, data, label=None, weight=None, base_margin=None, missing=None, feature_names=None,
                 feature_types=None, nthread=None, enable_categorical=False, max_bin=None, ref=None,
                 device=None, label_lower_bound=None, label_upper_bound=None, qid=None, group=None, multi_target=False,
                 bin_layout="auto", **kwargs):
        layout = bin_layout_code(bin_layout)
        if is_sparse(data):
            data = canonical_csr(data)
        elif hasattr(data, "values") and not isinstance(data, np.ndarray):  # pandas
            dtypes = list(data.dtypes) if hasattr(data, "columns") else [getattr(data, "dtype", None)]
            if any(str(dt).startswith("Sparse") for dt in dtypes):
                raise XGBoostError("pandas columns with a SparseDtype are not supported: pass "
                                   "scipy.sparse.csr_matrix(df.sparse.to_coo()) instead")
            if feature_names is None and hasattr(data, "columns"):
                feature_names = [str(c) for c in data.columns]
            cat_cols = [str(dt) == "category" for dt in data.dtypes] if hasattr(data, "columns") else []
            if any(cat_cols):
                # xgboost's pandas adapter: category dtype -> codes, -1 (NaN) -> missing; needs enable_categorical
                if not enable_categorical:
                    raise XGBoostError("DataFrame has `category` columns: pass enable_categorical=True")
                cols = []
                for c, is_c in zip(data.columns, cat_cols):
                    if is_c:
                        codes = data[c].cat.codes.to_numpy().astype(np.float32)
                        codes[codes < 0] = np.nan
                        cols.append(codes)
                    else:
                        cols.append(data[c].to_numpy().astype(np.float32))
                if feature_types is None:
                    feature_types = ["c" if is_c else "q" for is_c in cat_cols]
                data = np.stack(cols, axis=1) if cols else np.zeros((len(data), 0), np.float32)
            else:
                data = data.values
        blocks = None
        remote = data if (hasattr(data, "pid") and hasattr(data, "row_stride") and hasattr(data, "addr")) else None
        if remote is not None or isinstance(data, CSRArrays):     # rows of another process (matrix.RemoteBlock) / CSR
            pass
        elif hasattr(data, "next") and hasattr(data, "reset"):       # xgboost.DataIter protocol (matrix.py:127-196)
            blocks, label, weight, base_margin = _drain_data_iter(data, label, weight, base_margin)
        elif isinstance(data, (list, tuple)) and data and all(hasattr(b, "shape") for b in data):
            if any(is_sparse(b) for b in data):
                raise XGBoostError("a list of sparse row blocks is not supported: pass one scipy.sparse matrix "
                                   "(scipy.sparse.vstack(blocks))")
            blocks = [np.asarray(b.values if hasattr(b, "values") and not isinstance(b, np.ndarray) else b) for b in data]
        if remote is not None or isinstance(data, CSRArrays):
            pass
        elif blocks is not None:
            blocks = [b.reshape(-1, 1) if b.ndim == 1 else b for b in blocks]
            if len({b.shape[1] for b in blocks}) != 1:
                raise XGBoostError("all row blocks of a DMatrix must have the same number of columns")
            data = _BlockList([_f32c(b) for b in blocks])
        else:
            data = np.asarray(data)
            if data.ndim == 1:
                data = data.reshape(-1, 1)
            if data.ndim != 2:
                raise XGBoostError("DMatrix data must be 2-dimensional")
            data = _f32c(data)
        if layout == BIN_LAYOUTS["csr"] and not isinstance(data, CSRArrays):
            raise XGBoostError('bin_layout="csr" needs a scipy.sparse matrix: this DMatrix holds dense rows')
        self._host = data
        self.bin_layout = bin_layout
        self.missing = float("nan") if missing is None else float(missing)
        self.device = _default_device() if device is None else int(device)
        self.feature_names = list(feature_names) if feature_names is not None else None
        self.feature_types = list(feature_types) if feature_types is not None else None
        self.enable_categorical = bool(enable_categorical)
        self.max_bin = max_bin
        self.ref = ref
        self._quantized = False
        self._has_raw = True
        self.multi_target = bool(multi_target)
        self._label = None
        self._weight = None
        self._base_margin = None
        self._group_sizes = None
        h = _H(0)
        n, f = self._host.shape
        self.ingest = "host"
        inter = getattr(remote, "interleave", None) if remote is not None else None
        if (inter is not None and _coll.handle and _coll.world == inter[3] and n * f > 0
                and os.environ.get("B2_INTERLEAVED_INGEST", "0") not in ("", "0")):
            # INTERLEAVED shard and every rank of the communicator builds its shard of the same matrix right now: each
            # rank reads one contiguous block from the driver, the rows are redistributed over NVLink.  Opt-in
            # (B2_INTERLEAVED_INGEST=1): validated on 2 GPUs, where it shortens the upload (0.108 vs 0.128 s for 10M x 100)
            # but not yet the whole call; the default stays the strided host read (DESIGN.md 6)
            _check(lib().B2_MatrixCreateFromProcessInterleaved(remote.pid, inter[0], inter[1], f, inter[2], _coll.handle,
                                                               self.missing, self.device, C.byref(h)))
            self.handle = h.value
            self.ingest = "nvlink-redistributed"
        elif remote is not None:
            # the shard lives in the driver process: read it straight into the pinned upload buffers
            _check(lib().B2_MatrixCreateFromProcess(remote.pid, remote.addr, remote.row_stride, n, f, self.missing, self.device,
                                                    C.byref(h)))
            self.handle = h.value
        elif isinstance(self._host, CSRArrays):
            # the device keeps the CSR: absent entries are missing; the sketch and the tree walks read its stored entries
            c = self._host
            _check(lib().B2_MatrixCreateFromCSR(c.indptr.ctypes.data_as(_LP), _ip(c.indices), _fp(c.values), n, f, c.nnz,
                                                self.missing, self.device, C.byref(h)))
            self.handle = h.value
        elif isinstance(self._host, _BlockList):
            # several row blocks (multi-file shard / DataIter): one device allocation, each block uploaded at its row
            # offset -- the host never concatenates them
            _check(lib().B2_MatrixCreate(n, f, self.missing, self.device, C.byref(h)))
            self.handle = h.value
            self._upload_blocks()
        else:
            _check(lib().B2_MatrixCreateFromDense(_fp(self._host), n, f, self.missing, self.device, C.byref(h)))
            self.handle = h.value
        if layout != BIN_LAYOUTS["auto"]:
            _check(lib().B2_MatrixSetBinLayout(self.handle, layout))
        if self.feature_types is not None:
            if len(self.feature_types) != f:
                raise XGBoostError("feature_types has %d entries for %d features" % (len(self.feature_types), f))
            is_cat = np.array([1 if str(t) == "c" else 0 for t in self.feature_types], np.uint8)
            if is_cat.any():
                if not enable_categorical:
                    raise XGBoostError("feature_types marks categorical features: pass enable_categorical=True")
                _check(lib().B2_MatrixSetFeatureTypes(self.handle, _bp(is_cat), f))
        self.set_info(label=label, weight=weight, base_margin=base_margin, label_lower_bound=label_lower_bound,
                      label_upper_bound=label_upper_bound, qid=qid, group=group)

    # -- info
    def set_info(self, label=None, weight=None, base_margin=None, feature_weights=None,
                 label_lower_bound=None, label_upper_bound=None, qid=None, group=None, **kw):
        if qid is not None or group is not None:
            self._set_groups(qid, group, weighted=weight is not None or self._weight is not None)
        elif weight is not None and self._group_sizes is not None:
            raise XGBoostError("sample weights on a matrix with query groups (per-group weights) are not supported")
        # the survival bounds are stored for every objective and read by survival:aft only, as in xgboost
        for field, v in (("label", label), ("weight", weight), ("base_margin", base_margin),
                         ("feature_weights", feature_weights), ("label_lower_bound", label_lower_bound),
                         ("label_upper_bound", label_upper_bound)):
            if v is None:
                continue
            if hasattr(v, "values") and not isinstance(v, np.ndarray):
                v = v.values
            a = np.asarray(v)
            if field == "label" and a.ndim == 2 and a.shape[1] > 1:
                # T label columns: multi-target regression / multi-label classification, one tree per column and round
                if not self.multi_target:
                    raise XGBoostError("label has shape %s: a label of several columns (multi-target regression, "
                                       "multi-label classification) needs DMatrix(..., multi_target=True)" % (a.shape,))
                a = _f32c(a)
                _check(lib().B2_MatrixSetLabel(self.handle, _fp(a), a.shape[0], a.shape[1]))
                self._label = a
                continue
            if field == "label" and a.ndim > 2:
                raise XGBoostError("label must be 1- or 2-dimensional, got shape %s" % (a.shape,))
            a = _f32c(a.reshape(-1))
            _check(lib().B2_MatrixSetFloatInfo(self.handle, field.encode(), _fp(a), a.size))
            setattr(self, "_" + field, a)

    def _set_groups(self, qid, group, weighted):
        """Query groups from `qid` (one id per row, non-decreasing: a group is a run of equal ids) or from `group`
        (the sizes of consecutive groups), as xgboost's DMatrix takes them."""
        if qid is not None and group is not None:
            raise XGBoostError("pass either qid or group, not both")
        if weighted:
            raise XGBoostError("sample weights on a matrix with query groups (per-group weights) are not supported")
        n = self.num_row()
        if qid is not None:
            q = np.asarray(qid.values if hasattr(qid, "values") and not isinstance(qid, np.ndarray) else qid).reshape(-1)
            if q.size != n:
                raise XGBoostError("qid has %d values for %d rows" % (q.size, n))
            if q.size and np.any(q[1:] < q[:-1]):
                raise XGBoostError("qid must be sorted in non-decreasing order (sort the rows by qid first)")
            starts = np.flatnonzero(np.r_[True, q[1:] != q[:-1]]) if q.size else np.zeros(0, np.int64)
            sizes = np.diff(np.r_[starts, q.size])
        else:
            sizes = np.asarray(group, np.int64).reshape(-1)
            if np.any(sizes < 1) or int(sizes.sum()) != n:
                raise XGBoostError("group sizes must be >= 1 and sum to the row count %d" % n)
        if sizes.size and sizes.max() > np.iinfo(np.int32).max:
            raise XGBoostError("a query group has more than 2^31 - 1 rows")
        sizes = np.ascontiguousarray(sizes, np.int32)
        _check(lib().B2_MatrixSetGroups(self.handle, _ip(sizes), sizes.size))
        self._group_sizes = sizes

    def get_group(self):
        return self._group_sizes.copy() if self._group_sizes is not None else np.zeros(0, np.int32)

    def set_group(self, group):
        self.set_info(group=group)

    def set_label(self, label):
        self.set_info(label=label)

    def set_weight(self, weight):
        self.set_info(weight=weight)

    def set_base_margin(self, margin):
        self.set_info(base_margin=margin)

    def get_label(self):
        """(n,) labels, or (n, T) for a label of T > 1 columns."""
        return self._label if self._label is not None else np.zeros(0, np.float32)

    def get_weight(self):
        return self._weight if self._weight is not None else np.zeros(0, np.float32)

    def get_base_margin(self):
        return self._base_margin if self._base_margin is not None else np.zeros(0, np.float32)

    def num_row(self):
        return self._host.shape[0]

    def num_col(self):
        return self._host.shape[1]

    # -- engine side
    def _upload_blocks(self):
        at = 0
        for b in self._host.blocks:
            _check(lib().B2_MatrixSetRows(self.handle, at, _fp(b), b.shape[0]))
            at += b.shape[0]

    def _ensure_quantized(self, max_bin, keep_raw=False, cuts=None):
        """GPU sketch + binning.  `cuts` = (ptrs, vals, mins, has_missing) freezes the cut points instead of sketching
        (restart of an interrupted training with the cuts of its first attempt)."""
        if self._quantized:
            return
        mb = int(self.max_bin or max_bin or 256)
        if cuts is not None:
            ptrs, vals, mins, hm = (np.ascontiguousarray(cuts[0], np.int32), _f32c(cuts[1]), _f32c(cuts[2]),
                                    np.ascontiguousarray(cuts[3], np.uint8))
            if ptrs.size != self.num_col() + 1:
                raise XGBoostError("frozen cuts are for %d features, the matrix has %d" % (ptrs.size - 1, self.num_col()))
            _check(lib().B2_MatrixQuantizeWithCuts(self.handle, _coll.handle, _ip(ptrs), _fp(vals), _fp(mins), _bp(hm), mb,
                                                   1 if keep_raw else 0))
        else:
            ref_h = 0
            if self.ref is not None:
                self.ref._ensure_quantized(max_bin, keep_raw=True)
                ref_h = self.ref.handle
            _check(lib().B2_MatrixQuantize(self.handle, _coll.handle, mb, ref_h, 1 if keep_raw else 0))
        self._quantized = True
        self._has_raw = bool(keep_raw)

    def _ensure_raw(self):
        if not self._has_raw:
            if isinstance(self._host, _SliceRows):   # a slice: its host rows, taken out of the parent's once
                self._host = self._host.rows()
            if isinstance(self._host, CSRArrays):
                c = self._host
                _check(lib().B2_MatrixEnsureRawCSR(self.handle, c.indptr.ctypes.data_as(_LP), _ip(c.indices), _fp(c.values)))
                self._has_raw = True
                return
            if isinstance(self._host, _BlockList):   # rare (predicting on a block-built training matrix): one host copy
                self._host = np.concatenate(self._host.blocks, axis=0)
            elif not isinstance(self._host, np.ndarray):   # rows of another process: fetch them once
                self._host = _f32c(np.asarray(self._host))
            _check(lib().B2_MatrixEnsureRaw(self.handle, _fp(self._host)))
            self._has_raw = True

    def device_bytes(self):
        """Device bytes this matrix owns (raw values dense or CSR, bins, cuts and info arrays)."""
        out = C.c_int64(0)
        _check(lib().B2_MatrixDeviceBytes(self.handle, C.byref(out)))
        return out.value

    def get_cuts(self):
        tot = C.c_int32(0)
        _check(lib().B2_MatrixCutsSize(self.handle, C.byref(tot)))
        f = self.num_col()
        ptrs = np.zeros(f + 1, np.int32)
        vals = np.zeros(max(tot.value, 1), np.float32)
        mins = np.zeros(f, np.float32)
        hm = np.zeros(f, np.uint8)
        _check(lib().B2_MatrixGetCuts(self.handle, _ip(ptrs), _fp(vals), _fp(mins), _bp(hm)))
        return ptrs, vals[:tot.value], mins, hm

    def get_bins(self):
        out = np.zeros(self._host.shape, np.uint8)
        _check(lib().B2_MatrixGetBins(self.handle, _bp(out)))
        return out

    def slice(self, rindex, allow_groups=False):
        """xgboost's DMatrix.slice: a new DMatrix of rows `rindex` of this one, in that order (duplicates allowed).

        The rows are gathered on the device from this matrix's device data (B2_MatrixSlice), dense values as dense and
        CSR as CSR, with the label, weights, base_margin and survival bounds of those rows; missing, the feature names
        and types and feature_weights are copied.  The slice is unquantised: it is sketched with its own cuts when it is
        trained or evaluated, as xgboost re-sketches a slice, so it gives the cuts, bins, models and predictions of
        ``DMatrix(X[rindex], label=y[rindex], ...)``.  This matrix is not changed; when its raw values are no longer on
        the device (quantised without them) they are uploaded again first, as evaluation does.  The slice's host rows
        are taken out of this matrix's host data only if a later call needs them.

        A matrix with query groups is sliced only with allow_groups=True; the slice then has no groups until
        set_group is called.  A QuantileDMatrix is not sliced, as in xgboost."""
        if isinstance(self, QuantileDMatrix):
            raise XGBoostError("slice: a QuantileDMatrix / DeviceQuantileDMatrix cannot be sliced (xgboost does not "
                               "slice them either): slice a DMatrix of the same data")
        if self._group_sizes is not None and not allow_groups:
            raise XGBoostError("slice: the matrix has query groups; pass allow_groups=True and give the slice its "
                               "groups with set_group")
        n = self.num_row()
        idx = slice_rows(rindex, n)
        self._ensure_raw()
        h = _H(0)
        _check(lib().B2_MatrixSlice(self.handle, idx.ctypes.data_as(_LP), idx.size, C.byref(h)))
        out = DMatrix.__new__(DMatrix)
        out.handle = h.value

        def rows(a):   # a per-row host array ([n] or [n][k], base_margin flattened) at the slice's rows
            if a is None or a.size == 0:
                return a
            b = a.reshape(n, -1)[idx]
            return b if a.ndim == 2 else b.reshape(-1)

        out.__dict__.update(
            _host=_SliceRows(self._host, idx), missing=self.missing, device=self.device,
            feature_names=None if self.feature_names is None else list(self.feature_names),
            feature_types=None if self.feature_types is None else list(self.feature_types),
            enable_categorical=self.enable_categorical, max_bin=self.max_bin, ref=None, _quantized=False,
            _has_raw=True, multi_target=self.multi_target, _label=rows(self._label), _weight=rows(self._weight),
            _base_margin=rows(self._base_margin), _group_sizes=None, ingest="slice", bin_layout=self.bin_layout)
        for field in ("_label_lower_bound", "_label_upper_bound"):
            if field in self.__dict__:
                setattr(out, field, rows(getattr(self, field)))
        if "_feature_weights" in self.__dict__:
            out._feature_weights = self._feature_weights
        return out

    def __del__(self):
        try:
            if getattr(self, "handle", 0):
                lib().B2_MatrixFree(self.handle)
                self.handle = 0
        except Exception:
            pass


class _BlockList:
    """Row blocks of one shard, presented with the little of the ndarray surface DMatrix needs."""

    def __init__(self, blocks):
        self.blocks = blocks
        self.shape = (sum(b.shape[0] for b in blocks), blocks[0].shape[1])


def slice_rows(rindex, n):
    """The row indices of DMatrix.slice as int64, checked: at least one, every one an integer in [0, n)."""
    a = np.asarray(rindex).reshape(-1)
    if a.size == 0:
        raise XGBoostError("slice: rindex is empty (a slice needs at least one row)")
    if a.dtype == bool or not np.issubdtype(a.dtype, np.integer):
        vals = a.tolist()   # name the first value that is not even integral (else the first: its type is not int)
        bad = [i for i, v in enumerate(vals) if isinstance(v, bool) or not (
            isinstance(v, numbers.Integral) or (isinstance(v, float) and v.is_integer()))]
        i = bad[0] if bad else 0
        raise XGBoostError("slice: rindex[%d] = %r is not an integer" % (i, vals[i]))
    a = np.ascontiguousarray(a, np.int64)
    out = np.flatnonzero((a < 0) | (a >= n))
    if out.size:
        i = int(out[0])
        raise XGBoostError("slice: rindex[%d] = %d is outside [0, %d)" % (i, int(a[i]), n))
    return a


class _SliceRows:
    """The host rows of a slice: its parent's host data and the row indices, turned into rows only when a call needs
    them (a slice's values live on the device; the host rows serve a re-upload after they were freed there)."""

    def __init__(self, host, idx):
        if isinstance(host, _SliceRows):   # a slice of a slice indexes the first parent
            host, idx = host.host, host.idx[idx]
        self.host, self.idx = host, idx
        self.shape = (idx.size, host.shape[1])

    def rows(self):
        h, idx = self.host, self.idx
        if isinstance(h, CSRArrays):
            lens = np.diff(h.indptr)[idx]
            indptr = np.zeros(idx.size + 1, np.int64)
            np.cumsum(lens, out=indptr[1:])
            pos = np.repeat(h.indptr[idx] - indptr[:-1], lens) + np.arange(indptr[-1], dtype=np.int64)
            return CSRArrays(indptr, h.indices[pos], h.values[pos], self.shape)
        if isinstance(h, _BlockList):
            h = np.concatenate(h.blocks, axis=0)
        return _f32c(np.asarray(h)[idx])


def _drain_data_iter(it, label, weight, base_margin):
    """Pull every batch out of an xgboost.DataIter-style object: `it.next(input_data)` calls `input_data(data=...,
    label=..., weight=..., base_margin=...)` once per batch and returns 0 at the end (matrix.py:166-196)."""
    got = {"data": [], "label": [], "weight": [], "base_margin": []}

    def input_data(data=None, label=None, weight=None, base_margin=None, **kw):
        if is_sparse(data):
            raise XGBoostError("a DataIter batch that is a scipy.sparse matrix is not supported: pass the whole matrix "
                               "to DMatrix as one scipy.sparse matrix")
        got["data"].append(np.asarray(data.values if hasattr(data, "values") and not isinstance(data, np.ndarray) else data))
        for k, v in (("label", label), ("weight", weight), ("base_margin", base_margin)):
            if v is not None:
                a = np.asarray(v.values if hasattr(v, "values") and not isinstance(v, np.ndarray) else v)
                got[k].append(a if k == "label" and a.ndim == 2 else a.reshape(-1))   # a 2-D label keeps its columns

    it.reset()
    while it.next(input_data):
        pass
    if not got["data"]:
        raise XGBoostError("the data iterator produced no batch")
    cat = lambda k, given: given if given is not None else (np.concatenate(got[k]) if got[k] else None)  # noqa: E731
    return got["data"], cat("label", label), cat("weight", weight), cat("base_margin", base_margin)


class QuantileDMatrix(DMatrix):
    """Same device object; kept as a distinct name for RayQuantileDMatrix (main.py:380-386)."""


DeviceQuantileDMatrix = QuantileDMatrix


# ----------------------------------------------------------------------------- callbacks
class TrainingCallback:
    """xgboost.callback.TrainingCallback protocol (compat/__init__.py:12-41)."""

    def before_training(self, model):
        return model

    def after_training(self, model):
        return model

    def before_iteration(self, model, epoch, evals_log):
        return False

    def after_iteration(self, model, epoch, evals_log):
        return False


class EarlyStopException(Exception):
    def __init__(self, best_iteration):
        super().__init__()
        self.best_iteration = best_iteration


class LearningRateScheduler(TrainingCallback):
    """xgboost.callback.LearningRateScheduler: a learning rate per boosting round.

    learning_rates: a sequence of rates, or a callable that takes the epoch and returns the rate.  After round `epoch`
    the callback calls ``model.set_param("learning_rate", rate)`` with rate ``learning_rates[epoch]`` (or
    ``learning_rates(epoch)``), so rate i applies from round i + 1 and the first round trains with the params' eta.
    That is the after_iteration hook xgboost 1.3-2.x uses as far as recalled; it could not be checked against
    xgboost's source.  Epochs restart at 0 in every train() call, also when it continues from xgb_model.

    Actors receive their callbacks pickled: a sequence is stored as a tuple of floats, so the callback pickles; a
    callable must be picklable itself (a module-level function, not a lambda)."""

    def __init__(self, learning_rates):
        if callable(learning_rates):
            self.learning_rates = learning_rates
        elif isinstance(learning_rates, (list, tuple, np.ndarray)):
            self.learning_rates = tuple(float(r) for r in np.asarray(learning_rates, np.float64).reshape(-1))
        else:
            raise TypeError("learning_rates must be a sequence of rates or a callable of the epoch, got %r"
                            % (type(learning_rates).__name__,))

    def after_iteration(self, model, epoch, evals_log):
        rates = self.learning_rates
        model.set_param("learning_rate", rates(epoch) if callable(rates) else rates[epoch])
        return False


class EarlyStopping(TrainingCallback):
    """xgboost.callback.EarlyStopping: stop training once `rounds` rounds in a row have not improved a metric.

    It watches metric `metric_name` of the eval set `data_name`; by default the last eval set of `evals` and its last
    metric.  An unknown name raises ValueError naming it.  `maximize` defaults to the direction train(...,
    early_stopping_rounds=) uses for the metric.  A round improves when `score - min_delta > best` (maximising) or
    `best - min_delta > score` (minimising), so an equal score does not improve.  After every improving round the
    model's best_iteration and best_score are set; best_iteration counts the model's rounds, those of xgb_model
    included.  With save_best=True, after_training returns ``model[: best_iteration + 1]`` carrying both attributes
    again.  These rules are recalled from xgboost 2.x's callback.py, not checked against its source (DESIGN.md 2
    item 23).  Under cv() the history holds (mean, std) pairs and the mean is watched.

    The history starts again in before_training, so one instance can serve several train() calls.  Actors receive the
    callback pickled; every rank sees the same allreduced metric values and stops at the same round.  An actor restart
    re-sends the callbacks, so the history starts again at the checkpoint's round."""

    def __init__(self, rounds, metric_name=None, data_name=None, maximize=None, save_best=False, min_delta=0.0):
        if min_delta < 0:
            raise ValueError("min_delta must be >= 0, got %r" % (min_delta,))
        self.rounds = int(rounds)
        self.metric_name, self.data_name, self.maximize = metric_name, data_name, maximize
        self.save_best, self.min_delta = bool(save_best), float(min_delta)
        self.starting_round, self.best, self.stale = 0, None, 0

    def before_training(self, model):
        self.starting_round, self.best, self.stale = model.num_boosted_rounds(), None, 0
        return model

    def after_iteration(self, model, epoch, evals_log):
        if not evals_log:
            raise ValueError("EarlyStopping needs at least one eval set (evals=)")
        data = self.data_name if self.data_name is not None else list(evals_log)[-1]
        if data not in evals_log:
            raise ValueError("EarlyStopping: no eval set named %r (eval sets: %s)" % (data, ", ".join(evals_log)))
        log = evals_log[data]
        metric = self.metric_name if self.metric_name is not None else list(log)[-1]
        if metric not in log:
            raise ValueError("EarlyStopping: eval set %r has no metric named %r (metrics: %s)"
                             % (data, metric, ", ".join(log)))
        score = log[metric][-1]
        score = float(score[0] if isinstance(score, tuple) else score)   # cv() logs (mean, std): the mean is watched
        mx = self.maximize if self.maximize is not None else _maximized(metric)
        if self.best is None or (score - self.min_delta > self.best if mx else self.best - self.min_delta > score):
            self.best, self.stale = score, 0
            model.best_iteration, model.best_score = self.starting_round + epoch, score
        else:
            self.stale += 1
        return self.stale >= self.rounds

    def after_training(self, model):
        if not self.save_best or model.best_iteration is None:
            return model
        best_iteration, best_score = model.best_iteration, model.best_score
        model = model[: best_iteration + 1]
        model.best_iteration, model.best_score = best_iteration, best_score
        return model


class callback:  # namespace shim: xgb.callback.TrainingCallback, LearningRateScheduler, EarlyStopping
    TrainingCallback = TrainingCallback
    LearningRateScheduler = LearningRateScheduler
    EarlyStopping = EarlyStopping


# ----------------------------------------------------------------------------- Booster
# Everything the Python side knows about an objective, in one place: its default eval metric, the margin -> prediction
# transform, and the parameter block of xgboost 2.x's JSON model ({json key: default}; "num_class" is the model's class
# count).  The engine (csrc/engine.cu) owns the gradients.
class _Objective:
    def __init__(self, metric, transform, block=None, block_params=None):
        self.metric, self.transform, self.block, self.block_params = metric, transform, block, block_params or {}

    def default_metric(self, params):
        if self.metric == "tweedie-nloglik":   # the metric carries the objective's variance power in its name
            return "tweedie-nloglik@%g" % float(params.get("tweedie_variance_power", 1.5))
        if self.metric in ("ndcg", "map"):     # ranking: ndcg / map at the objective's pair cut-off
            return "%s@%d" % (self.metric, int(params.get("lambdarank_num_pair_per_sample", 32)))
        return self.metric


_REG_LOSS = ("reg_loss_param", {"scale_pos_weight": 1})
_SOFTMAX = ("softmax_multiclass_param", {"num_class": None})
# xgboost 2.x writes every lambdarank parameter as a string; lambdarank_bias_norm only matters with lambdarank_unbiased
_LAMBDARANK = ("lambdarank_param", {"lambdarank_pair_method": "topk", "lambdarank_num_pair_per_sample": "32",
                                    "lambdarank_unbiased": "0", "lambdarank_bias_norm": "2", "ndcg_exp_gain": "1"})
_OBJECTIVES = {
    "reg:squarederror": _Objective("rmse", None, *_REG_LOSS),
    "reg:linear": _Objective("rmse", None, *_REG_LOSS),
    "reg:logistic": _Objective("rmse", "sigmoid", *_REG_LOSS),
    "binary:logistic": _Objective("logloss", "sigmoid", *_REG_LOSS),
    "binary:logitraw": _Objective("logloss", None, *_REG_LOSS),
    "reg:squaredlogerror": _Objective("rmsle", None, *_REG_LOSS),
    "reg:pseudohubererror": _Objective("mphe", None, "pseudo_huber_param", {"huber_slope": 1}),
    "count:poisson": _Objective("poisson-nloglik", "exp", "poisson_regression_param", {"max_delta_step": 0.7}),
    "reg:gamma": _Objective("gamma-nloglik", "exp"),
    "reg:tweedie": _Objective("tweedie-nloglik", "exp", "tweedie_regression_param", {"tweedie_variance_power": 1.5}),
    "survival:aft": _Objective("aft-nloglik", "exp", "aft_loss_param",
                               {"aft_loss_distribution": "normal", "aft_loss_distribution_scale": 1}),
    "rank:pairwise": _Objective("ndcg", None, *_LAMBDARANK),
    "rank:ndcg": _Objective("ndcg", None, *_LAMBDARANK),
    "rank:map": _Objective("map", None, *_LAMBDARANK),           # binary relevance; ndcg_exp_gain is kept, unused
    # one output per alpha; the block's value is the alphas' list string (quantile_alpha_text)
    "reg:quantileerror": _Objective("quantile", None, "reg_quantileerror_param", {"quantile_alpha": "[0.5]"}),
    "multi:softprob": _Objective("mlogloss", "softmax", *_SOFTMAX),
    "multi:softmax": _Objective("mlogloss", "softmax", *_SOFTMAX),
}


def quantile_alphas(value):
    """reg:quantileerror's quantile_alpha in any form xgboost takes -> float32 array of the alphas.

    value: a number, a list / tuple / numpy array of numbers, or a string such as "0.5" or "[0.1, 0.5, 0.9]"; None gives
    xgboost's default [0.5].  Every alpha must be finite with 0 < alpha < 1 (as a float32), else XGBoostError names it."""
    if value is None:
        return np.array([0.5], np.float32)
    if isinstance(value, (bytes, bytearray)):
        value = value.decode()
    if isinstance(value, str):
        try:
            value = ast.literal_eval(value.strip())
        except (ValueError, SyntaxError) as e:
            raise XGBoostError("quantile_alpha=%r does not parse as a number or a list of numbers (%s)" % (value, e))
    items = list(np.ravel(np.asarray(value, dtype=object))) if isinstance(value, (list, tuple, np.ndarray)) else [value]
    if not items:
        raise XGBoostError("quantile_alpha must hold at least one alpha")
    out = []
    for a in items:
        if isinstance(a, (bool, np.bool_, str, bytes)) or not isinstance(a, (int, float, np.integer, np.floating)):
            raise XGBoostError("quantile_alpha: %r is not a number" % (a,))
        f = np.float32(a)
        if not (np.isfinite(f) and 0 < f < 1):
            raise XGBoostError("quantile_alpha: %r is outside (0, 1); every alpha must satisfy 0 < alpha < 1" % (a,))
        out.append(f)
    return np.array(out, np.float32)


def quantile_alpha_text(alphas):
    """The alphas as the model and save_config write them: "[0.1, 0.5, 0.9]" (9 significant digits: exact float32)."""
    return "[" + ", ".join(_num_str(a) for a in quantile_alphas(alphas)) + "]"


def _objective(name):
    o = _OBJECTIVES.get(name)
    if o is None:
        raise XGBoostError("unsupported objective '%s' (supported: %s)" % (name, ", ".join(sorted(_OBJECTIVES))))
    return o


_ENGINE_KEYS = ("objective", "num_class", "max_depth", "eta", "learning_rate", "gamma", "min_split_loss",
                "min_child_weight", "lambda", "reg_lambda", "alpha", "reg_alpha", "base_score", "hist_qbits",
                "hist_chunk_rows", "profile", "max_cat_to_onehot", "max_cat_threshold", "scale_pos_weight",
                "max_delta_step", "subsample", "colsample_bytree", "colsample_bylevel", "colsample_bynode", "seed",
                "random_state", "num_parallel_tree", "huber_slope", "tweedie_variance_power", "aft_loss_distribution",
                "aft_loss_distribution_scale", "lambdarank_pair_method", "lambdarank_num_pair_per_sample",
                "lambdarank_unbiased", "ndcg_exp_gain", "booster", "rate_drop", "skip_drop", "sample_type",
                "normalize_type", "one_drop", "quantile_alpha", "num_target", "multi_strategy", "process_type",
                "updater", "refresh_leaf")
# xgboost's parameter aliases among the engine's keys
_ALIASES = {"eta": ("learning_rate",), "learning_rate": ("eta",), "gamma": ("min_split_loss",),
            "min_split_loss": ("gamma",), "lambda": ("reg_lambda",), "reg_lambda": ("lambda",), "alpha": ("reg_alpha",),
            "reg_alpha": ("alpha",), "seed": ("random_state",), "random_state": ("seed",)}
# booster=dart's parameters with xgboost's defaults (save_config's dart_train_param)
_DART_DEFAULTS = {"rate_drop": 0.0, "skip_drop": 0.0, "sample_type": "uniform", "normalize_type": "tree", "one_drop": 0}

# xgboost parameters that change the trained model and that this engine does not implement (its parameter parser
# ignores them as unknown keys): a value different from the neutral one is an error, never silently ignored (a drop-in
# must not train a different model quietly)
_UNSUPPORTED_NEUTRAL = {
    "sampling_method": ("uniform",), "max_leaves": (0,), "grow_policy": ("depthwise",),
    "monotone_constraints": (None, "", "()", (), []),
}


def is_update_mode(params):
    """process_type='update': the rounds refresh the trees of xgb_model instead of growing new ones."""
    return (params.get("process_type") or "default") == "update"


def _engine_text(params, extra=None):
    """The params text of B2_BoosterCreate / B2_CheckParams: the engine's keys of `params` (None: not given), then
    `extra`.  quantile_alpha goes as "a,b,c" with each float32 alpha written exactly."""
    p = {k: params[k] for k in _ENGINE_KEYS if params.get(k) is not None}
    if "quantile_alpha" in p:
        p["quantile_alpha"] = ",".join(repr(float(a)) for a in quantile_alphas(p["quantile_alpha"]))
    if extra:
        p.update(extra)
    return "\n".join("%s=%s" % (k, v) for k, v in p.items()).encode()


def _check_python_forms(params):
    """The checks only Python can make: max_bin's range, and the keys the engine ignores, in their Python forms."""
    mb = params.get("max_bin")
    if mb is not None and not 2 <= int(mb) <= 256:
        raise XGBoostError("parameter max_bin=%r is not supported by the H100 hist engine: the bin matrix is uint8, "
                           "max_bin must be in [2, 256]" % (mb,))
    for k, neutral in _UNSUPPORTED_NEUTRAL.items():
        if k in params and params[k] is not None:
            v = params[k]
            if isinstance(v, (list, tuple)) and k == "monotone_constraints" and all(int(x) == 0 for x in v):
                continue
            if isinstance(v, str) and k == "monotone_constraints" and set(v) <= set("(), 0"):
                continue
            if v not in neutral:
                raise XGBoostError("parameter %s=%r is not supported by the H100 hist engine (supported: %s)"
                                   % (k, v, ", ".join(repr(x) for x in neutral[:4])))


def _check_supported(params):
    """Every parameter rule, without a device: the Python-only checks, then the engine's (params.cu) on its text."""
    _check_python_forms(params)
    _check(lib().B2_CheckParams(_engine_text(params)))


def interaction_sets(value, n_features, feature_names=None):
    """xgboost's interaction_constraints in any accepted form -> list of sorted feature-index sets.

    value: a string such as "[[0, 1], [2, 3, 4]]", or a list / tuple of iterables of integer indices (numpy integers
    included) or of feature names (resolved against feature_names).  Duplicates inside a set are dropped, empty sets are
    ignored; None, "", "[]" and [] give [] (no constraints).  A bad entry raises XGBoostError naming it."""
    if value is None:
        return []
    if isinstance(value, str):
        if not value.strip():
            return []
        try:
            value = ast.literal_eval(value.strip())
        except (ValueError, SyntaxError) as e:
            raise XGBoostError("interaction_constraints=%r does not parse as a list of feature sets (%s)" % (value, e))
    if isinstance(value, (str, bytes)) or not isinstance(value, (list, tuple)):
        raise XGBoostError("interaction_constraints must be a list of feature sets, got %r" % (value,))
    names = {str(n): i for i, n in enumerate(feature_names)} if feature_names is not None else {}
    sets = []
    for s in value:
        if isinstance(s, (str, bytes)) or not hasattr(s, "__iter__"):
            raise XGBoostError("interaction_constraints: %r is not a set of features" % (s,))
        idx = set()
        for f in s:
            if isinstance(f, str):
                if f not in names:
                    raise XGBoostError("interaction_constraints: unknown feature name %r" % (f,))
                f = names[f]
            elif isinstance(f, (bool, np.bool_)) or not isinstance(f, (int, np.integer)):
                raise XGBoostError("interaction_constraints: %r is not an integer feature index" % (f,))
            f = int(f)
            if not 0 <= f < n_features:
                raise XGBoostError("interaction_constraints: feature index %d is outside [0, %d)" % (f, n_features))
            idx.add(f)
        if idx:
            sets.append(sorted(idx))
    return sets


def _params_dict(params):
    return {} if params is None else dict(params)


def _model_document(raw):
    """The document of a model file: JSON when, after optional whitespace, `{` is followed by `"`, `}` or whitespace;
    UBJSON when `{` is followed by a key length, `$`, `#` or no-op marker."""
    i = len(raw) - len(raw.lstrip(b" \t\r\n"))
    if raw[i:i + 1] == b"{":
        nxt = raw[i + 1:i + 2]
        if nxt in (b'"', b"}", b" ", b"\t", b"\r", b"\n"):
            return json.loads(raw.decode())
        if nxt and nxt in b"iUIlL$#N":
            from xgboost_ray_b200 import ubjson
            return ubjson.loads(raw, i)
    raise XGBoostError("not a JSON or UBJSON model; the deprecated binary format is not supported")


def _exact_covers(text):
    """The "b2.sum_hessian" attribute of a UBJSON model: tree -> its float64 covers."""
    out = {}
    try:
        for ti, b in json.loads(text or "[]"):
            out[int(ti)] = np.frombuffer(base64.b64decode(b, validate=True), "<f8").astype(np.float64)
    except (ValueError, TypeError) as e:
        raise XGBoostError("model attribute b2.sum_hessian is malformed: %s" % e)
    return out


def _covers(sum_hessian, exact):
    """A tree's covers: the file's sum_hessian, or the exact float64 covers of b2.sum_hessian where those round to the
    file's values node for node (a tool that rewrote the trees without the attribute leaves its covers in charge)."""
    h = np.asarray(sum_hessian, np.float64)
    if exact is not None and exact.shape == h.shape and \
            np.array_equal(exact.astype(np.float32), h.astype(np.float32)):
        return exact
    return h


class Booster:
    def __init__(self, params=None, cache=(), model_file=None):
        self.params = _params_dict(params)
        self.handle = 0
        self._train = None
        self._trees = []          # list of dict of numpy arrays (host copy for pickling / dumps)
        self._weights = None      # booster=dart: float32 weight of every tree in self._trees (None = all 1)
        self._cuts = None         # (ptrs, vals, mins, has_missing) of the matrix this model was trained on; travels with
        #                           pickles (checkpoints) so that a restarted training quantises with the SAME cuts
        self._attrs = {}
        self.feature_names = None
        self.feature_types = None
        self.n_features = None
        self.best_iteration = None
        self.best_score = None
        tm = self.params.get("tree_method", "hist")
        if tm not in ("hist", "gpu_hist", "auto", "approx"):
            raise XGBoostError("tree_method=%r is not supported (hist / gpu_hist only)" % (tm,))
        if (self.params.get("booster") or "gbtree") not in ("gbtree", "dart"):
            raise XGBoostError("booster=%r is not supported (supported: gbtree, dart)" % (self.params.get("booster"),))
        for d in cache:
            if isinstance(d, DMatrix) and self._train is None:
                self._attach(d)
        if model_file is not None:
            self.load_model(model_file)

    # -- engine object management
    def _param_text(self, extra=None):
        """The text B2_BoosterCreate parses, which applies the engine's parameter rules itself."""
        _check_python_forms(self.params)
        return _engine_text(self.params, extra)

    def _interaction_sets(self, n_features=None, feature_names=None):
        return interaction_sets(self.params.get("interaction_constraints"),
                                self.n_features if n_features is None else n_features,
                                self.feature_names if feature_names is None else feature_names)

    def _attach(self, dtrain):
        """Create the device booster bound to `dtrain` (quantising it if needed)."""
        old_trees = self.get_trees() if (self.handle or self._trees) else []
        old_weights = self.get_tree_weights() if old_trees else None
        self._free()
        dtrain._ensure_quantized(int(self.params.get("max_bin", 256)), cuts=self._cuts if old_trees else None)
        self._cuts = dtrain.get_cuts()
        sets = self._interaction_sets(dtrain.num_col(),
                                      self.feature_names if self.feature_names is not None else dtrain.feature_names)
        # one param line: sets separated by ';', features by ','
        extra = {"interaction_constraints": ";".join(",".join(map(str, s)) for s in sets)} if sets else None
        if old_trees:   # the trees were grown for the model's targets: the engine checks the matrix's label against them
            extra = dict(extra or {}, num_target=self._num_target())
        h = _H(0)
        _check(lib().B2_BoosterCreate(self._param_text(extra), dtrain.handle, _coll.handle, C.byref(h)))
        self.handle = h.value
        self._trained = False   # set_param takes effect through the engine once a round has run
        # the engine takes the targets from the train matrix's label; the model keeps them for its file and predictions
        nt = C.c_int32(1)
        _check(lib().B2_BoosterNumTargets(self.handle, C.byref(nt)))
        if nt.value > 1:
            self.params["num_target"] = nt.value
        else:
            self.params.pop("num_target", None)
        self._train = dtrain
        self.n_features = dtrain.num_col()
        if self.feature_names is None:
            self.feature_names = dtrain.feature_names
        if getattr(self, "feature_types", None) is None:
            self.feature_types = dtrain.feature_types
        if old_trees:
            dtrain._ensure_raw()
            self._push_trees(old_trees, old_weights)
            if is_update_mode(self.params):
                # the engine takes these as the trees to update; the model starts empty and grows by refreshed rounds
                self._trees = []
                self.__dict__.pop("_tree_json_cache", None)
            else:
                _check(lib().B2_BoosterResetTrainMargin(self.handle))

    def _ensure_predictor(self, device=None):
        if self.handle:
            return
        if self.n_features is None:
            raise XGBoostError("booster has no model")
        h = _H(0)
        extra = {"num_feature": self.n_features, "device": _default_device() if device is None else device}
        _check(lib().B2_BoosterCreate(self._param_text(extra), 0, 0, C.byref(h)))
        self.handle = h.value
        try:
            self._push_trees(self._trees, self._weights)
        except XGBoostError:   # a refused tree: no predictor of part of the model
            self._free()
            raise

    def _push_trees(self, trees, weights=None):
        for t in trees:
            rec, _arrays = B2Tree.of(t)
            _check(lib().B2_BoosterAddTree(self.handle, C.byref(rec)))
        if self.is_dart and trees and weights is not None:
            w = _f32c(weights)
            if w.size != len(trees):
                raise XGBoostError("DART model has %d tree weights for %d trees" % (w.size, len(trees)))
            _check(lib().B2_BoosterSetTreeWeights(self.handle, _fp(w), w.size))

    def _free(self):
        if self.handle:
            try:
                lib().B2_BoosterFree(self.handle)
            except Exception:
                pass
            self.handle = 0
            self._train = None

    def __del__(self):
        self._free()

    # -- model access
    def num_trees(self):
        if self.handle:
            n = C.c_int32(0)
            _check(lib().B2_BoosterNumTrees(self.handle, C.byref(n)))
            return n.value
        return len(self._trees)

    def _num_target(self):
        """Label columns of the model: T > 1 for multi-target regression / multi-label classification, else 1."""
        return int(self.params.get("num_target", 1) or 1)

    @property
    def num_class(self):
        """Outputs per row: the classes of multi:*, the alphas of reg:quantileerror, the label columns of a multi-target
        model, else 1."""
        obj = self.params.get("objective", "reg:squarederror")
        if obj == "reg:quantileerror":
            return int(quantile_alphas(self.params.get("quantile_alpha")).size)
        if self._num_target() > 1:
            return self._num_target()
        return int(self.params.get("num_class", 1)) if obj.startswith("multi:") else 1

    @property
    def is_dart(self):
        return (self.params.get("booster") or "gbtree") == "dart"

    @property
    def is_vector_leaf(self):
        """One vector-leaf tree per round for all targets (multi_strategy='multi_output_tree' with T > 1)."""
        return self.params.get("multi_strategy") == "multi_output_tree" and self._num_target() > 1

    @property
    def _trees_per_round(self):
        return 1 if self.is_vector_leaf else self.num_class * self.num_parallel_tree

    def get_tree_weights(self):
        """Per-tree weights (float32, model order): DART's weight_drop; 1 for every gbtree tree."""
        if self.handle:
            w = np.zeros(self.num_trees(), np.float32)
            _check(lib().B2_BoosterGetTreeWeights(self.handle, _fp(w), w.size))
            self._weights = w if self.is_dart else None
            return w.copy()
        if self._weights is not None:
            return np.array(self._weights, np.float32)
        return np.ones(len(self._trees), np.float32)

    @property
    def num_parallel_tree(self):
        return max(1, int(self.params.get("num_parallel_tree", 1) or 1))

    def num_boosted_rounds(self):
        return self.num_trees() // max(1, self._trees_per_round)

    def num_features(self):
        return self.n_features

    def get_tree(self, i):
        nn = C.c_int32(0)
        _check(lib().B2_BoosterTreeNumNodes(self.handle, i, C.byref(nn)))
        n = nn.value
        t = dict(left=np.zeros(n, np.int32), right=np.zeros(n, np.int32), parent=np.zeros(n, np.int32),
                 split_feature=np.zeros(n, np.int32), split_bin=np.zeros(n, np.int32),
                 split_cond=np.zeros(n, np.float32), default_left=np.zeros(n, np.uint8),
                 value=np.zeros(n, np.float32), base_weight=np.zeros(n, np.float32),
                 loss_chg=np.zeros(n, np.float32), sum_hess=np.zeros(n, np.float64),
                 split_type=np.zeros(n, np.uint8), cat_bits=np.zeros((n, 8), np.uint32))
        if self.is_vector_leaf:
            t["leaf_vector"] = np.zeros((n, self._num_target()), np.float32)
        rec, _arrays = B2Tree.of(t)
        _check(lib().B2_BoosterGetTree(self.handle, i, C.byref(rec)))
        return t

    def get_trees(self):
        if self.handle:
            have = len(self._trees)
            for i in range(have, self.num_trees()):
                self._trees.append(self.get_tree(i))
        return list(self._trees)

    # -- training
    def update(self, dtrain, iteration, fobj=None):
        if self._train is not dtrain:
            self._attach(dtrain)
        if fobj is not None:
            pred = self.predict(dtrain, output_margin=True, training=True)
            grad, hess = fobj(pred, dtrain)
            self.boost(dtrain, grad, hess)
            return
        if is_update_mode(self.params):   # refresh round `iteration` of the model's trees (DESIGN.md 2 item 20)
            _check(lib().B2_BoosterRefreshOneIter(self.handle, None, None, 0))
            self._trained = True
            return
        _check(lib().B2_BoosterUpdateOneIter(self.handle, int(iteration)))
        self._trained = True
        self._sync_base_score()

    def _sync_base_score(self):
        """Without a user base_score the engine estimates it from the labels before the first tree (xgboost >= 2.0,
        SURVEY.md A.3); keep the value with the model so that saved / pickled / predict-only boosters use it."""
        if self.handle and self.params.get("base_score") is None:
            v, fin = C.c_float(0), C.c_int32(0)
            _check(lib().B2_BoosterGetBaseScore(self.handle, C.byref(v), C.byref(fin)))
            if fin.value:
                self.params["base_score"] = float(v.value)

    def boost(self, dtrain, grad, hess):
        if self._train is not dtrain:
            self._attach(dtrain)
        g = _f32c(np.asarray(grad).reshape(-1))
        h = _f32c(np.asarray(hess).reshape(-1))
        if g.size != h.size:
            raise XGBoostError("grad / hess size mismatch")
        if is_update_mode(self.params):
            _check(lib().B2_BoosterRefreshOneIter(self.handle, _fp(g), _fp(h), g.size))
            self._trained = True
            return
        _check(lib().B2_BoosterBoostOneIter(self.handle, _fp(g), _fp(h), g.size))
        self._trained = True
        self._sync_base_score()

    def _metric_names(self):
        m = self.params.get("eval_metric")
        if m is None:
            return [_objective(self.params.get("objective", "reg:squarederror")).default_metric(self.params)]
        return list(m) if isinstance(m, (list, tuple)) else [m]

    def eval_set(self, evals, iteration=0, feval=None, output_margin=True):
        """Returns xgboost's '[it]\\tname-metric:value...' string."""
        parts = ["[%d]" % iteration]
        for dm, name in evals:
            if dm is not self._train:
                dm._ensure_raw()
            for metric in self._metric_names():
                v = C.c_double(0)
                _check(lib().B2_BoosterEvalSet(self.handle, dm.handle, metric.encode(), C.byref(v)))
                parts.append("%s-%s:%.6f" % (name, metric, v.value))
            if feval is not None:
                # the train matrix: the engine's full-model margin (for DART, not the next round's drop margin)
                pred = self.predict(dm, output_margin=output_margin, training=(dm is self._train), _full_margin=True)
                res = feval(pred, dm)
                res = res if isinstance(res, list) else [res]
                if _coll.world > 1:   # xgboost averages custom metric values over the workers (_allreduce_metric)
                    vals = collective.allreduce([float(v) for _, v in res]) / _coll.world
                    res = [(mname, float(v)) for (mname, _), v in zip(res, vals)]
                for mname, val in res:
                    parts.append("%s-%s:%.6f" % (name, mname, float(val)))
        return "\t".join(parts)

    def eval(self, data, name="eval", iteration=0):
        return self.eval_set([(data, name)], iteration)

    # -- prediction
    def _tree_range(self, iteration_range, ntree_limit):
        """(first tree, end tree) of an iteration_range / ntree_limit; end 0 = all trees."""
        per_round = self._trees_per_round
        tb, te = iteration_range if iteration_range else (0, 0)
        if ntree_limit:
            return 0, int(ntree_limit)
        return int(tb) * per_round, int(te) * per_round

    def predict(self, data, output_margin=False, ntree_limit=0, validate_features=True, training=False,
                iteration_range=(0, 0), strict_shape=False, pred_leaf=False, pred_contribs=False, approx_contribs=False,
                pred_interactions=False, _full_margin=False, **kwargs):
        """xgboost's Booster.predict.  Precedence as in xgboost: pred_leaf, then pred_interactions, then pred_contribs
        (exact TreeSHAP in margin space; output_margin does not apply)."""
        if not isinstance(data, DMatrix):
            raise TypeError("Expecting data to be a DMatrix object, got: %s" % type(data))
        self._ensure_predictor(data.device)
        if validate_features and self.n_features is not None and data.num_col() != self.n_features:
            raise XGBoostError("feature count mismatch: data has %d, model has %d" % (data.num_col(), self.n_features))
        if pred_leaf:
            return self._predict_leaf(data, iteration_range, ntree_limit, strict_shape)
        if pred_interactions or pred_contribs:
            if approx_contribs:
                raise XGBoostError("approx_contribs=True is not supported by the H100 engine: it computes exact TreeSHAP "
                                   "(leave approx_contribs=False)")
            return self._predict_contribs(data, iteration_range, ntree_limit, strict_shape, bool(pred_interactions))
        K = self.num_class
        n = data.num_row()
        out = np.zeros(n * K, np.float32)
        if training and data is self._train:
            _check(lib().B2_BoosterGetTrainMargin(self.handle, 1 if _full_margin else 0, _fp(out), out.size))
            if not output_margin:
                out = _transform(self.params.get("objective", "reg:squarederror"), out.reshape(n, K)).reshape(-1)
        else:
            data._ensure_raw()
            tb, te = self._tree_range(iteration_range, ntree_limit)
            _check(lib().B2_BoosterPredict(self.handle, data.handle, 1 if output_margin else 0, tb, te, _fp(out), out.size))
        if K == 1:
            return out
        out = out.reshape(n, K)
        if self.params.get("objective") == "multi:softmax" and not output_margin:
            return np.argmax(out, axis=1).astype(np.float32)
        return out

    def _predict_contribs(self, data, iteration_range, ntree_limit, strict_shape, interactions):
        data._ensure_raw()
        K, n, F = self.num_class, data.num_row(), data.num_col()
        tb, te = self._tree_range(iteration_range, ntree_limit)
        shape = (n, K, F + 1, F + 1) if interactions else (n, K, F + 1)
        out = np.zeros(shape, np.float32)
        _check(lib().B2_BoosterPredictContribs(self.handle, data.handle, tb, te, 1 if interactions else 0, _fp(out), out.size))
        if K == 1 and not strict_shape:
            return out.reshape(shape[:1] + shape[2:])
        return out

    def _predict_leaf(self, data, iteration_range, ntree_limit, strict_shape):
        data._ensure_raw()
        n, nt = data.num_row(), self.num_trees()
        tb, te = self._tree_range(iteration_range, ntree_limit)
        te = nt if te <= 0 or te > nt else te
        out = np.zeros((n, max(te - tb, 0)), np.float32)
        _check(lib().B2_BoosterPredictLeaf(self.handle, data.handle, tb, te, _fp(out), out.size))
        if strict_shape:
            if self.is_vector_leaf:   # one tree per round for all outputs
                return out.reshape(n, -1, 1, 1)
            return out.reshape(n, -1, self.num_class, self.num_parallel_tree)
        return out

    def inplace_predict(self, data, **kw):
        return self.predict(DMatrix(data), **kw)

    # -- attributes
    def attr(self, key):
        return self._attrs.get(key)

    def set_attr(self, **kwargs):
        for k, v in kwargs.items():
            if v is None:
                self._attrs.pop(k, None)
            else:
                self._attrs[k] = str(v)

    def attributes(self):
        return dict(self._attrs)

    def set_param(self, params, value=None):
        """Booster.set_param.  Once the device booster has trained a round, the engine's keys of the change go to the
        engine (B2_BoosterSetParam): the keys a round may change apply from the next round, any other engine key may
        only repeat its value, and a refused change raises XGBoostError and changes nothing.  Before the first round the
        next update() creates the device booster from the new parameters.  Other keys only update the dict."""
        if isinstance(params, str):
            params = {params: value}
        params = _params_dict(params)
        engine = {k: v for k, v in params.items() if k in _ENGINE_KEYS or k == "interaction_constraints"}
        if engine and self.handle and self._train is not None:
            if getattr(self, "_trained", False):
                sets = engine.pop("interaction_constraints", None)
                extra = None
                if sets is not None:
                    sets = interaction_sets(sets, self.n_features, self.feature_names)
                    extra = {"interaction_constraints": ";".join(",".join(map(str, s)) for s in sets)}
                _check(lib().B2_BoosterSetParam(self.handle, _engine_text(engine, extra)))
                # the model's params now say what the next rounds are grown with: an alias given earlier would
                # otherwise win over the new value when the booster is created again (_attach, checkpoints)
                for k in engine:
                    for alias in _ALIASES.get(k, ()):
                        self.params.pop(alias, None)
            else:
                self.get_trees()
                self.get_tree_weights()
                self._free()
        self.params.update(params)

    # -- (de)serialisation: XGBoost's JSON model format (doc/model.schema of dmlc/xgboost 2.x; SURVEY.md 8f-1).  Everything
    # a stock xgboost needs is where it expects it (objective parameter block, learner_model_param, gbtree_model_param,
    # string-valued parameters, strict JSON numbers); what only this engine uses (split bins, its own parameter set)
    # is carried under `attributes` with a "b2." prefix, which xgboost preserves and ignores.
    @staticmethod
    def _tree_json(i, t, n_features):
        n = len(t["left"])
        leaf = t["split_feature"] < 0
        st = np.asarray(t.get("split_type", np.zeros(n, np.uint8)))
        cats, cat_nodes, cat_segs, cat_sizes = [], [], [], []
        for nid in np.nonzero((st != 0) & ~leaf)[0]:
            c = _cat_list(t["cat_bits"][nid])
            cat_nodes.append(int(nid)); cat_segs.append(len(cats)); cat_sizes.append(len(c)); cats.extend(c)
        # split_conditions: leaf value for a leaf, threshold for a numeric split; a categorical split keeps its categories
        # in the arrays above and xgboost does not read the number (RegTree::ExpandCategorical stores NaN, which is not
        # JSON): 0 is written instead
        cond = np.where(leaf, t["value"], np.where(st != 0, np.float32(0.0), t["split_cond"])).astype(np.float32)
        # a numeric split on +inf (the last cut of a feature whose maximum is +inf or above FLT_MAX / 2) sends every
        # finite value left.  Strict JSON gets the nearest finite float32 (FLT_MAX), which a stock reader routes alike
        # except at x = FLT_MAX; the exact condition is returned as [node, "inf"] for the "b2.split_conds" attribute
        numeric = ~leaf & (st == 0)
        exact = [[int(nid), str(float(cond[nid]))] for nid in np.nonzero(numeric & ~np.isfinite(cond))[0]]
        cond = np.where(numeric & ~np.isnan(cond), np.clip(cond, -_FLT_MAX, _FLT_MAX), cond)
        cond = np.where(np.isfinite(cond), cond, np.float32(0.0))
        vec = t.get("leaf_vector")
        if vec is not None:   # vector-leaf tree: node-major [n][T] base weights, a leaf's condition is 0
            vec = np.asarray(vec, np.float32)
            cond = np.where(leaf, np.float32(0.0), cond)
        return exact, {
            "base_weights": [float(x) for x in (t["base_weight"] if vec is None else vec.reshape(-1))],
            "categories": cats, "categories_nodes": cat_nodes, "categories_segments": cat_segs,
            "categories_sizes": cat_sizes,
            "default_left": [int(x) for x in t["default_left"]],
            "id": i,
            "left_children": [int(x) for x in t["left"]],
            "loss_changes": [float(x) for x in t["loss_chg"]],
            "parents": [int(x) if x >= 0 else 2147483647 for x in t["parent"]],
            "right_children": [int(x) for x in t["right"]],
            "split_conditions": [float(x) for x in cond],
            "split_indices": [int(x) if x >= 0 else 0 for x in t["split_feature"]],
            "split_type": [int(x) for x in st],
            "sum_hessian": [float(x) for x in t["sum_hess"]],
            "tree_param": {"num_deleted": "0", "num_feature": str(n_features), "num_nodes": str(n),
                           "size_leaf_vector": "1" if vec is None else str(vec.shape[1])},
        }

    def _model_dict(self):
        K = self.num_class
        src = self.get_trees()
        cache = self.__dict__.setdefault("_tree_json_cache", [])     # finished trees never change: convert each once
        if len(cache) > len(src):
            del cache[:]
        for i in range(len(cache), len(src)):
            exact, tj = self._tree_json(i, src[i], self.n_features)
            cache.append((tj, [int(x) for x in src[i]["split_bin"]], exact))
        trees = [c[0] for c in cache]
        obj = self.params.get("objective", "reg:squarederror")
        quantile = obj == "reg:quantileerror" or self._num_target() > 1   # alphas and label columns are targets, not classes
        spec = _OBJECTIVES.get(obj, _OBJECTIVES["reg:squarederror"])
        obj_block = {"name": obj}
        if spec.block:
            obj_block[spec.block] = {k: str(K) if k == "num_class" else
                                     quantile_alpha_text(self.params.get(k)) if k == "quantile_alpha" else
                                     _str_param(self.params.get(k, d)) if isinstance(d, str) else _num_str(self.params.get(k, d))
                                     for k, d in spec.block_params.items()}
        attrs = {k: str(v) for k, v in self._attrs.items() if not k.startswith("b2.")}
        b2p = {k: self.params[k] for k in self.params if _json_ok(self.params[k]) and
               k not in ("objective", "num_class", "num_target", "base_score", "scale_pos_weight", "num_parallel_tree")}   # those have their own fields
        sets = self._interaction_sets() if self.n_features is not None else []
        if sets:   # in its resolved string form, which also keeps list / feature-name / numpy inputs
            b2p["interaction_constraints"] = str(sets)
        attrs["b2.params"] = json.dumps({k: b2p[k] for k in sorted(b2p)})
        attrs["b2.split_bins"] = json.dumps([c[1] for c in cache], separators=(",", ":"))
        exact = [[ti, nid, v] for ti, c in enumerate(cache) for nid, v in c[2]]
        if exact:   # [tree, node, "inf"]: the non-finite numeric conditions, which split_conditions cannot hold
            attrs["b2.split_conds"] = json.dumps(exact, separators=(",", ":"))
        gbtree = {"model": {
            "gbtree_model_param": {"num_parallel_tree": str(self.num_parallel_tree), "num_trees": str(len(trees))},
            "iteration_indptr": list(range(0, len(trees) + 1, self._trees_per_round)),
            "tree_info": [0 if self.is_vector_leaf else (i // self.num_parallel_tree) % K for i in range(len(trees))],
            "trees": trees}, "name": "gbtree"}
        if self.is_dart:   # xgboost's Dart::SaveModel: the gbtree block plus one weight per tree
            gbtree = {"name": "dart", "gbtree": gbtree,
                      "weight_drop": [float(x) for x in self.get_tree_weights()[:len(trees)]]}
        return {
            "learner": {
                "attributes": attrs,
                "feature_names": [str(x) for x in (self.feature_names or [])],
                "feature_types": [_xgb_feature_type(x) for x in (self.feature_types or [])],
                "gradient_booster": gbtree,
                "learner_model_param": {"base_score": _num_str(self.params.get("base_score", 0.5) if self.params.get("base_score") is not None else 0.5),
                                        "boost_from_average": "1", "num_class": str(K if K > 1 and not quantile else 0),
                                        "num_feature": str(self.n_features), "num_target": str(K if quantile else 1)},
                "objective": obj_block,
            },
            "version": [2, 0, 3],
        }

    def save_raw(self, raw_format="json"):
        """The model file as bytes: raw_format "json" (the default) or "ubj", xgboost's UBJSON encoding of the same
        document (DESIGN.md 2 item 25)."""
        if raw_format == "json":
            return bytearray(json.dumps(self._model_dict(), allow_nan=False).encode())
        if raw_format == "ubj":
            from xgboost_ray_b200 import ubjson
            return bytearray(ubjson.dumps(self._ubj_dict()))
        if raw_format == "deprecated":
            raise XGBoostError("raw_format='deprecated', xgboost's old binary model format, is not supported "
                               "(supported: json, ubj)")
        raise XGBoostError("raw_format=%r is not supported (supported: json, ubj)" % (raw_format,))

    def _ubj_dict(self):
        """_model_dict() as UBJSON carries it: `sum_hessian` is a float32 array in xgboost's dialect, while this engine
        keeps each node's hessian sum (the cover TreeSHAP weights paths by) in float64.  A tree whose covers float32
        cannot hold exactly gets its float32 covers in `sum_hessian` and the exact ones, little-endian float64 in
        base64, in the "b2.sum_hessian" attribute as [tree, "..."] (DESIGN.md 2 item 25)."""
        d = self._model_dict()
        gb = d["learner"]["gradient_booster"]
        trees = (gb["gbtree"] if gb["name"] == "dart" else gb)["model"]["trees"]   # a new list; its trees are cached
        exact = []
        for ti, t in enumerate(trees):
            h = np.asarray(t["sum_hessian"], np.float64)
            h32 = h.astype(np.float32)
            if not np.array_equal(h32.astype(np.float64), h):
                exact.append([ti, base64.b64encode(h.astype("<f8").tobytes()).decode()])
                trees[ti] = dict(t, sum_hessian=h32)
        if exact:
            d["learner"]["attributes"]["b2.sum_hessian"] = json.dumps(exact, separators=(",", ":"))
        return d

    def save_model(self, fname):
        """Write the model file: UBJSON when the path ends in .ubj (in any case, as xgboost compares the lowercased
        extension), JSON otherwise."""
        with open(fname, "wb") as f:
            f.write(bytes(self.save_raw("ubj" if os.fsdecode(fname).lower().endswith(".ubj") else "json")))

    def load_model(self, fname):
        """Load a model file (a path, bytes or bytearray) in JSON or UBJSON, told apart by its content."""
        if isinstance(fname, (bytes, bytearray)):
            raw = bytes(fname)
        else:
            with open(fname, "rb") as f:
                raw = f.read()
        self._load_document(_model_document(raw))

    def _load_document(self, d):
        """Fill the booster from a decoded model document, whose arrays are lists (JSON) or NumPy arrays (UBJSON)."""
        L = d["learner"]
        self._free()
        self.__dict__.pop("_tree_json_cache", None)
        attrs = dict(L.get("attributes", {}))
        params = dict(json.loads(attrs.pop("b2.params"))) if "b2.params" in attrs else dict(L.get("b2_params", {}))
        split_bins = json.loads(attrs.pop("b2.split_bins")) if "b2.split_bins" in attrs else None
        exact_conds = {}    # tree -> [(node, condition)]
        for ti, nid, v in json.loads(attrs.pop("b2.split_conds", "[]")):
            exact_conds.setdefault(int(ti), []).append((int(nid), np.float32(float(v))))
        exact_hess = _exact_covers(attrs.pop("b2.sum_hessian", None))
        params["objective"] = L["objective"]["name"]
        nc = int(L["learner_model_param"].get("num_class", "0"))
        nc = max(nc, int(L["objective"].get("softmax_multiclass_param", {}).get("num_class", "0")))
        if nc > 1:
            params["num_class"] = nc
        spw = L["objective"].get("reg_loss_param", {}).get("scale_pos_weight")
        if spw is not None and float(spw) != 1.0:
            params["scale_pos_weight"] = float(spw)
        spec = _OBJECTIVES.get(params["objective"])
        if spec is not None and spec.block not in (None, "reg_loss_param", "softmax_multiclass_param"):
            for k, v in L["objective"].get(spec.block, {}).items():
                if k in spec.block_params:
                    params[k] = str(v) if isinstance(spec.block_params[k], str) else float(v)
        params["base_score"] = float(L["learner_model_param"]["base_score"])
        gb = L["gradient_booster"]
        weights = None
        if gb.get("name") == "dart":
            params["booster"] = "dart"
            weights = np.asarray(gb.get("weight_drop", []), np.float32)
            gb = gb["gbtree"]
            if weights.size != len(gb["model"]["trees"]):
                raise XGBoostError("DART model has %d weight_drop entries for %d trees"
                                   % (weights.size, len(gb["model"]["trees"])))
        elif params.get("booster") == "dart":
            params["booster"] = "gbtree"
        npt = int(gb["model"].get("gbtree_model_param", {}).get("num_parallel_tree", "1"))
        if npt > 1:
            params["num_parallel_tree"] = npt
        params.update({k: v for k, v in self.params.items() if k not in params})
        nt = int(L["learner_model_param"].get("num_target", "1"))
        if nt > 1 and params["objective"] != "reg:quantileerror":   # quantile's targets are its alphas
            params["num_target"] = nt
        else:
            params.pop("num_target", None)
        vsizes = {int(t.get("tree_param", {}).get("size_leaf_vector", "1")) for t in gb["model"]["trees"]}
        vsizes = {1 if v == 0 else v for v in vsizes}
        if len(vsizes) > 1:
            raise XGBoostError("model mixes leaf vector sizes %s: a model keeps one multi_strategy" % sorted(vsizes))
        if vsizes and max(vsizes) > 1:   # vector-leaf trees, one per round
            if max(vsizes) != nt:
                raise XGBoostError("model has leaf vectors of size %d for %d targets" % (max(vsizes), nt))
            params["multi_strategy"] = "multi_output_tree"
        elif params.get("multi_strategy") == "multi_output_tree" and gb["model"]["trees"] and nt > 1:
            # single-output trees for several targets: the model was grown one tree per target (with T = 1 the
            # strategy is ignored and the recorded parameter is kept)
            params["multi_strategy"] = "one_output_per_tree"
        self.params = params
        self.n_features = int(L["learner_model_param"]["num_feature"])
        self.feature_names = L.get("feature_names") or None
        self.feature_types = [_b2_feature_type(x) for x in L.get("feature_types") or []] or None
        self._attrs = attrs
        self._trees = []
        self._weights = weights
        for ti, t in enumerate(gb["model"]["trees"]):
            left = np.asarray(t["left_children"], np.int32)
            leaf = left < 0
            sc = np.asarray(t["split_conditions"], np.float32)
            parent = np.asarray(t["parents"], np.int64)
            parent = np.where(parent == 2147483647, -1, parent).astype(np.int32)
            st = np.asarray(t.get("split_type", [0] * len(left)), np.uint8)
            bits = np.zeros((len(left), 8), np.uint32)
            for nid, seg, size in zip(t.get("categories_nodes", []), t.get("categories_segments", []),
                                      t.get("categories_sizes", [])):
                for c in t["categories"][seg:seg + size]:
                    if not 0 <= int(c) < 256:
                        raise XGBoostError("model has category %r outside [0, 255]" % (c,))
                    bits[nid, int(c) >> 5] |= np.uint32(1 << (int(c) & 31))
            sb = t.get("split_bins") if split_bins is None else split_bins[ti]
            cat_split = (st != 0) & ~leaf
            # a categorical node: one-hot splits keep their category as the condition, set splits have none (NaN)
            cond = np.where(leaf, 0, sc).astype(np.float32)
            for nid in np.nonzero(cat_split)[0]:
                cl = _cat_list(bits[nid])
                b_ = int(sb[nid]) if sb is not None else (cl[0] if len(cl) == 1 else -1)
                cond[nid] = np.float32(b_) if b_ >= 0 else np.float32("nan")
            for nid, v in exact_conds.get(ti, ()):
                cond[nid] = v
            bw = np.asarray(t["base_weights"], np.float32)
            vec = None
            if self.is_vector_leaf:   # node-major [n][T]; the scalar fields carry zeros
                vec = bw.reshape(len(left), nt)
                bw = np.zeros(len(left), np.float32)
                sc = np.zeros(len(left), np.float32)
            self._trees.append(dict(
                leaf_vector=vec,
                split_type=st, cat_bits=bits,
                left=left, right=np.asarray(t["right_children"], np.int32), parent=parent,
                split_feature=np.where(leaf, -1, np.asarray(t["split_indices"], np.int32)).astype(np.int32),
                split_bin=np.asarray(sb if sb is not None else [-1] * len(left), np.int32),
                split_cond=cond,
                default_left=np.asarray(t["default_left"], np.uint8),
                value=np.where(leaf, sc, bw).astype(np.float32),
                base_weight=bw,
                loss_chg=np.asarray(t["loss_changes"], np.float32),
                sum_hess=_covers(t["sum_hessian"], exact_hess.get(ti))))

    def __getstate__(self):
        return {"raw": bytes(self.save_raw()), "best_iteration": self.best_iteration, "best_score": self.best_score,
                "cuts": self._cuts}

    def __setstate__(self, state):
        self.params = {}
        self.handle = 0
        self._train = None
        self._trees = []
        self._weights = None
        self._attrs = {}
        self.feature_names = None
        self.feature_types = None
        self.n_features = None
        self._cuts = None
        self.load_model(state["raw"])
        self._cuts = state.get("cuts")
        self.best_iteration = state.get("best_iteration")
        self.best_score = state.get("best_score")

    def copy(self):
        b = Booster.__new__(Booster)
        b.__setstate__(self.__getstate__())
        return b

    def __getitem__(self, val):
        """bst[start:stop:step] / bst[i]: a new Booster with boosting rounds start, start + step, ... < stop.

        A round is _trees_per_round consecutive trees.  An int i is i:i + 1; start None is 0, stop None or 0 is
        num_boosted_rounds(), step None is 1.  A negative index, stop < start or step < 1 raises ValueError, a tuple
        ValueError, another type TypeError, and start >= num_boosted_rounds() or stop > num_boosted_rounds() IndexError
        (recalled from xgboost 2.x's Booster.__getitem__, DESIGN.md 2 item 23).  The slice keeps the params, the
        features, the attributes and each kept tree unchanged (DART: its weight too); it drops best_iteration /
        best_score, which index this model's rounds, and the frozen restart cuts.  It is built on the host: its device
        predictor is created when it first predicts, and this booster keeps its device state and can train on."""
        if isinstance(val, numbers.Integral):
            val = slice(val, val + 1)
        if isinstance(val, tuple):
            raise ValueError("Booster slicing supports only 1 dimension, got %r" % (val,))
        if not isinstance(val, slice):
            raise TypeError("Booster indices must be an int or a slice of rounds, got %s" % type(val).__name__)
        rounds = self.num_boosted_rounds()
        start = 0 if val.start is None else operator.index(val.start)
        stop = 0 if val.stop is None else operator.index(val.stop)
        step = 1 if val.step is None else operator.index(val.step)
        if start < 0 or stop < 0:
            raise ValueError("Booster slicing takes no negative index, got %r" % (val,))
        if stop == 0:
            stop = rounds
        elif stop < start:
            raise ValueError("Booster slice %r ends before it starts" % (val,))
        if step < 1:
            raise ValueError("Booster slice step must be >= 1, got %d" % step)
        if start >= rounds or stop > rounds:
            raise IndexError("Booster slice %r is out of range: the model has %d rounds" % (val, rounds))
        per = self._trees_per_round
        keep = [r * per + j for r in range(start, stop, step) for j in range(per)]
        trees = self.get_trees()
        out = Booster(self.params)
        out._trees = [{k: v.copy() if isinstance(v, np.ndarray) else v for k, v in trees[i].items()} for i in keep]
        out._weights = self.get_tree_weights()[keep] if self.is_dart else None
        out._attrs = dict(self._attrs)
        out.n_features = self.n_features
        out.feature_names = list(self.feature_names) if self.feature_names is not None else None
        out.feature_types = list(self.feature_types) if self.feature_types is not None else None
        return out

    def __iter__(self):
        """One Booster per boosting round, in model order: self[i] for i in range(num_boosted_rounds())."""
        for i in range(self.num_boosted_rounds()):
            yield self[i]

    def save_config(self):
        gbtree = {"name": "gbtree"}
        sets = self._interaction_sets() if self.n_features is not None else []
        if sets:
            gbtree["tree_train_param"] = {"interaction_constraints": str(sets)}
        if is_update_mode(self.params):   # xgboost's GBTreeTrainParam of an update run
            gbtree["gbtree_train_param"] = {"process_type": "update", "updater": "refresh",
                                            "refresh_leaf": _str_param(self.params.get("refresh_leaf", 1) in
                                                                       (1, True, "1", "true", "True"))}
        if self.is_dart:
            gbtree = {"name": "dart", "gbtree": gbtree,
                      "dart_train_param": {k: _str_param(self.params.get(k, d)) if isinstance(d, str) else
                                           _num_str(self.params.get(k, d)) for k, d in _DART_DEFAULTS.items()}}
        objective = {"name": self.params.get("objective", "reg:squarederror")}
        if objective["name"] == "reg:quantileerror":
            objective["reg_quantileerror_param"] = {"quantile_alpha": quantile_alpha_text(self.params.get("quantile_alpha"))}
        # rank:map reports the model file's lambdarank_param block (rank:pairwise / rank:ndcg keep their name-only entry)
        if objective["name"] == "rank:map":
            objective[_LAMBDARANK[0]] = {k: _str_param(self.params.get(k, d)) for k, d in _LAMBDARANK[1].items()}
        return json.dumps({"learner": {"gradient_booster": gbtree,
                                       "learner_train_param": {
                                           "multi_strategy": self.params.get("multi_strategy") or "one_output_per_tree"},
                                       "objective": objective,
                                       "b2_params": {k: v for k, v in self.params.items() if _json_ok(v)}},
                           "version": [2, 0, 3]})

    # -- dumps (A.11)
    def get_dump(self, fmap="", with_stats=False, dump_format="text"):
        names = self.feature_names
        out = []
        for t in self.get_trees():
            if dump_format == "json":
                out.append(json.dumps(_dump_json(t, 0, 0, names, with_stats)))
            else:
                lines = []
                _dump_text(t, 0, 0, names, with_stats, lines)
                out.append("".join(lines))
        return out

    def get_fscore(self, fmap=""):
        return self.get_score(importance_type="weight")

    def get_score(self, fmap="", importance_type="weight"):
        """xgboost's Booster.get_score: weight (split count), gain / cover (averages per split), total_gain / total_cover."""
        if importance_type not in ("weight", "gain", "cover", "total_gain", "total_cover"):
            raise XGBoostError("unknown importance_type %r" % (importance_type,))
        cnt, tot = {}, {}
        for t in self.get_trees():
            for nid in range(len(t["left"])):
                f = int(t["split_feature"][nid])
                if f < 0:
                    continue
                name = self.feature_names[f] if self.feature_names else "f%d" % f
                cnt[name] = cnt.get(name, 0) + 1
                v = float(t["sum_hess"][nid]) if importance_type.endswith("cover") else float(t["loss_chg"][nid])
                tot[name] = tot.get(name, 0.0) + v
        if importance_type == "weight":
            return cnt
        if importance_type.startswith("total_"):
            return tot
        return {k: tot[k] / cnt[k] for k in tot}

    def get_timers(self, reset=False):
        if not self.handle:
            return {}
        buf = C.create_string_buffer(2048)
        _check(lib().B2_BoosterGetTimers(self.handle, 1 if reset else 0, buf, len(buf)))
        return json.loads(buf.value.decode())

    def cancel(self):
        if self.handle:
            lib().B2_BoosterCancel(self.handle)


def _num_str(v):
    """Parameter values are strings in xgboost's JSON; floats with the 9 significant digits of a binary32."""
    f = float(v)
    return str(int(f)) if f == int(f) and abs(f) < 1e15 else "%.9g" % f


def _str_param(v):
    """A string-valued parameter as xgboost writes it: booleans as "1" / "0"."""
    if isinstance(v, (bool, np.bool_)):
        return "1" if v else "0"
    return str(v)


def _maximized(metric):
    """Metrics where larger is better (early stopping): auc, aucpr, interval-regression-accuracy and every ndcg / map /
    pre form (ndcg@5, map-, pre@10, ...)."""
    if metric in ("auc", "aucpr", "interval-regression-accuracy"):
        return True
    return metric.split("@")[0].rstrip("-") in ("ndcg", "map", "pre")


def _xgb_feature_type(t):
    """'q' / 'c' of the DMatrix interface -> the names xgboost stores in a model file."""
    return {"q": "float", "c": "c", "i": "int"}.get(str(t), str(t))


def _b2_feature_type(t):
    return {"float": "q", "int": "q", "i": "q", "c": "c", "q": "q"}.get(str(t), str(t))


def _json_ok(v):
    return isinstance(v, (str, int, float, bool)) or v is None


def _fname(names, f):
    return names[f] if names else "f%d" % f


def _cat_list(words):
    """Sorted categories of a 256-bit category set (8 uint32 words, LSB first)."""
    return [b for b in range(256) if (int(words[b >> 5]) >> (b & 31)) & 1]


def _is_cat_node(t, nid):
    st = t.get("split_type")
    return st is not None and bool(st[nid])


def _dump_json(t, nid, depth, names, with_stats):
    if t["split_feature"][nid] < 0:
        vec = t.get("leaf_vector")
        d = {"nodeid": int(nid), "leaf": float(t["value"][nid]) if vec is None else [float(x) for x in vec[nid]]}
        if with_stats:
            d["cover"] = float(t["sum_hess"][nid])
        return d
    l, r = int(t["left"][nid]), int(t["right"][nid])
    if _is_cat_node(t, nid):   # xgboost's dump: the listed categories go to "yes" = the right child
        d = {"nodeid": int(nid), "depth": depth, "split": _fname(names, int(t["split_feature"][nid])),
             "split_condition": _cat_list(t["cat_bits"][nid]), "yes": r, "no": l,
             "missing": l if t["default_left"][nid] else r}
    else:
        d = {"nodeid": int(nid), "depth": depth, "split": _fname(names, int(t["split_feature"][nid])),
             "split_condition": float(t["split_cond"][nid]), "yes": l, "no": r,
             "missing": l if t["default_left"][nid] else r}
    if with_stats:
        d["gain"] = float(t["loss_chg"][nid])
        d["cover"] = float(t["sum_hess"][nid])
    d["children"] = [_dump_json(t, l, depth + 1, names, with_stats), _dump_json(t, r, depth + 1, names, with_stats)]
    return d


def _dump_text(t, nid, depth, names, with_stats, lines):
    ind = "\t" * depth
    if t["split_feature"][nid] < 0:
        vec = t.get("leaf_vector")
        if vec is None:
            s = "%s%d:leaf=%.9g" % (ind, nid, float(t["value"][nid]))
        else:   # vector-leaf tree: one value per target
            s = "%s%d:leaf=[%s]" % (ind, nid, ",".join("%.9g" % float(x) for x in vec[nid]))
        if with_stats:
            s += ",cover=%.9g" % float(t["sum_hess"][nid])
        lines.append(s + "\n")
        return
    l, r = int(t["left"][nid]), int(t["right"][nid])
    if _is_cat_node(t, nid):
        s = "%s%d:[%s:{%s}] yes=%d,no=%d,missing=%d" % (ind, nid, _fname(names, int(t["split_feature"][nid])),
                                                        ",".join(str(c) for c in _cat_list(t["cat_bits"][nid])), r, l,
                                                        l if t["default_left"][nid] else r)
    else:
        s = "%s%d:[%s<%.9g] yes=%d,no=%d,missing=%d" % (ind, nid, _fname(names, int(t["split_feature"][nid])),
                                                       float(t["split_cond"][nid]), l, r,
                                                       l if t["default_left"][nid] else r)
    if with_stats:
        s += ",gain=%.9g,cover=%.9g" % (float(t["loss_chg"][nid]), float(t["sum_hess"][nid]))
    lines.append(s + "\n")
    _dump_text(t, l, depth + 1, names, with_stats, lines)
    _dump_text(t, r, depth + 1, names, with_stats, lines)


def _transform(objective, m):
    t = _OBJECTIVES[objective].transform if objective in _OBJECTIVES else None
    if t == "sigmoid":
        return (1.0 / (1.0 + np.exp(-m.astype(np.float64)))).astype(np.float32)
    if t == "exp":
        return np.exp(m.astype(np.float64)).astype(np.float32)
    if t == "softmax":
        e = np.exp(m - m.max(axis=1, keepdims=True))
        return (e / e.sum(axis=1, keepdims=True)).astype(np.float32)
    return m


# ----------------------------------------------------------------------------- train()
def _parse_eval_str(s):
    out = []
    for tok in s.split("\t")[1:]:
        k, v = tok.rsplit(":", 1)
        data, metric = k.split("-", 1)
        out.append((data, metric, float(v)))
    return out


def train(params, dtrain, num_boost_round=10, evals=(), obj=None, feval=None, maximize=None,
          early_stopping_rounds=None, evals_result=None, verbose_eval=True, xgb_model=None, callbacks=None,
          custom_metric=None):
    """xgboost.train look-alike (the call at xgboost_ray/main.py:745-752).  Epochs restart at 0 on
    every call, also when continuing from `xgb_model` (relied on by main.py:1609-1610)."""
    callbacks = list(callbacks or [])
    feval = custom_metric if custom_metric is not None else feval
    params = _params_dict(params)
    bst = Booster(params)
    update = is_update_mode(params)
    if update:
        _check_supported(params)
        if xgb_model is None:
            raise XGBoostError("process_type='update' refreshes the trees of an existing model: pass it as xgb_model")
    if xgb_model is not None:
        if isinstance(xgb_model, Booster):
            src = xgb_model
            src.get_trees()
        else:
            src = Booster(params)
            src.load_model(xgb_model)
        bst._trees = list(src._trees)
        if src.is_dart and "booster" not in params:   # a DART model continues as DART
            bst.params["booster"] = "dart"
        elif src.is_dart and not bst.is_dart:
            raise XGBoostError("cannot continue a DART model with booster=%r: its trees carry weights that a gbtree "
                               "model would drop (continue with booster='dart')" % (bst.params.get("booster"),))
        bst._weights = src.get_tree_weights() if bst.is_dart and src.is_dart else None
        if src._num_target() > 1:   # the trees of output k were fitted to label column k
            bst.params["num_target"] = src._num_target()
        if src.params.get("objective") == "reg:quantileerror" and bst.params.get("objective") == "reg:quantileerror":
            # the trees of output k were fitted to alpha_k: a continuation keeps the alphas
            old = quantile_alphas(src.params.get("quantile_alpha"))
            if bst.params.get("quantile_alpha") is None:
                bst.params["quantile_alpha"] = [float(a) for a in old]
            elif quantile_alphas(bst.params["quantile_alpha"]).tobytes() != old.tobytes():
                raise XGBoostError("cannot continue training with quantile_alpha=%s: the model was trained with %s"
                                   % (quantile_alpha_text(bst.params["quantile_alpha"]), quantile_alpha_text(old)))
        bst.n_features, bst.feature_names, bst.feature_types = src.n_features, src.feature_names, src.feature_types
        bst._attrs = dict(src._attrs)
        # a restart after an actor failure (main.py sets _freeze_cuts on the unpickled checkpoint) continues with the
        # cuts of the first attempt; a user-level continuation re-sketches the matrix it is given, like xgboost
        bst._cuts = src._cuts if getattr(src, "_freeze_cuts", False) else None
        # The trees of the source model were fitted around ITS intercept: a continuation (checkpoint restart,
        # main.py:1211-1220) must keep it, also when the user gave no base_score and it was estimated from the labels.
        if bst.params.get("base_score") is None and bst._trees:
            if src.params.get("base_score") is None:
                raise XGBoostError("cannot continue training: the model passed as xgb_model carries no base_score")
            bst.params["base_score"] = float(src.params["base_score"])
        if update:
            # the trees keep their shape and their intercept: num_parallel_tree and base_score are the model's own
            if src.is_vector_leaf:
                raise XGBoostError("process_type='update' is not supported for a multi_strategy='multi_output_tree' "
                                   "model")
            if src.is_dart:
                raise XGBoostError("process_type='update' is not supported for a booster='dart' model")
            if src.params.get("base_score") is None:
                raise XGBoostError("process_type='update': the model passed as xgb_model carries no base_score")
            if src.params.get("objective") == "reg:quantileerror":
                raise XGBoostError("process_type='update' is not supported for a reg:quantileerror model: its leaf "
                                   "values are residual quantiles, which the refresh updater does not recompute")
            bst.params["base_score"] = float(src.params["base_score"])
            bst.params["num_parallel_tree"] = src.num_parallel_tree
            per_round = src._trees_per_round
            if bst._trees_per_round != per_round:
                # round r's trees are cut from the model by its own outputs; the engine refreshes them by the update
                # call's (its objective, num_class): the two must agree, else trees would be refreshed for other outputs
                raise XGBoostError("process_type='update': the model has %d trees per round (%d outputs x "
                                   "num_parallel_tree %d), the update parameters give %d outputs (objective=%r); pass "
                                   "the model's objective and num_class"
                                   % (per_round, src.num_class, src.num_parallel_tree, bst.num_class,
                                      bst.params.get("objective", "reg:squarederror")))
            rounds = len(bst._trees) // max(1, per_round)
            if num_boost_round > rounds:
                raise XGBoostError("process_type='update' refreshes existing rounds: num_boost_round=%d but the model has "
                                   "%d rounds" % (num_boost_round, rounds))
            bst._trees = bst._trees[:num_boost_round * per_round]
    bst._attach(dtrain)
    evals = list(evals or [])
    evals_log = {}
    for cb in callbacks:
        r = cb.before_training(bst)
        bst = r if r is not None else bst
    best_score, best_iter, best_msg = None, 0, None
    try:
        for epoch in range(num_boost_round):
            if any(cb.before_iteration(bst, epoch, evals_log) for cb in callbacks):
                break
            bst.update(dtrain, epoch, fobj=obj)
            if evals:
                msg = bst.eval_set(evals, epoch, feval, output_margin=obj is not None)
                for data, metric, v in _parse_eval_str(msg):
                    evals_log.setdefault(data, {}).setdefault(metric, []).append(v)
                if verbose_eval and (verbose_eval is True or epoch % int(verbose_eval) == 0) and _coll.rank == 0:
                    print(msg, flush=True)
                if early_stopping_rounds:
                    data, metric, v = _parse_eval_str(msg)[-1]
                    mx = maximize if maximize is not None else _maximized(metric)
                    better = best_score is None or (v > best_score if mx else v < best_score)
                    if better:
                        best_score, best_iter, best_msg = v, epoch, msg
                    elif epoch - best_iter >= early_stopping_rounds:
                        bst.best_iteration, bst.best_score = best_iter, best_score
                        raise EarlyStopException(best_iter)
            stop = False
            for cb in callbacks:
                if cb.after_iteration(bst, epoch, evals_log):
                    stop = True
            if stop:
                break
    except EarlyStopException:
        pass
    if early_stopping_rounds and best_score is not None and bst.best_iteration is None:
        bst.best_iteration, bst.best_score = best_iter, best_score
    for cb in callbacks:
        r = cb.after_training(bst)
        bst = r if r is not None else bst
    if evals_result is not None:
        evals_result.clear()
        evals_result.update(evals_log)
    return bst


# ----------------------------------------------------------------------------- cv()
def cv_folds(n_rows, nfold=3, label=None, group_sizes=None, stratified=False, folds=None, seed=0, shuffle=True):
    """The folds of cv() as xgboost 2.x's mknfold / mkgroupfold make them, recalled and not checked against its source
    (DESIGN.md 2 item 24): a list of (train rows, test rows, train group sizes, test group sizes); the group sizes are
    None unless the rows are split by query groups.  Needs no device.

    - Default: np.random.seed(seed); the rows (with `group_sizes`, the groups) are permuted if `shuffle`, else kept in
      order, and split by np.array_split into nfold test sets.  Fold k trains on the other folds' rows concatenated in
      fold order.  Groups are turned back into their rows, in the group order of each side.
    - stratified=True: scikit-learn's StratifiedKFold(nfold, shuffle=True, random_state=seed) on the label.
    - folds: a list of (train_idx, test_idx) pairs, or an object with split(X, y) (such as a KFold), called with the
      label as X and y; nfold is then the number of folds."""
    np.random.seed(seed)
    if folds is not None:
        try:
            pairs = [(f[0], f[1]) for f in folds]
        except TypeError:
            if not hasattr(folds, "split"):
                raise XGBoostError("cv: folds must be a list of (train_idx, test_idx) pairs or an object with "
                                   "split(X, y), got %s" % type(folds).__name__) from None
            pairs = [(f[0], f[1]) for f in folds.split(X=label, y=label)]
        except (IndexError, KeyError):
            raise XGBoostError("cv: every entry of folds must be a (train_idx, test_idx) pair") from None
        if not pairs:
            raise XGBoostError("cv: folds holds no fold")
        return [(np.asarray(a), np.asarray(b), None, None) for a, b in pairs]
    if isinstance(nfold, bool) or not isinstance(nfold, numbers.Integral) or nfold < 2:
        raise XGBoostError("cv: nfold must be an integer >= 2, got %r" % (nfold,))
    nfold = int(nfold)
    if stratified:
        try:
            from sklearn.model_selection import StratifiedKFold
        except ImportError:
            raise XGBoostError("cv(stratified=True) needs scikit-learn (StratifiedKFold), which is not installed") from None
        skf = StratifiedKFold(n_splits=nfold, shuffle=True, random_state=seed)
        return [(a, b, None, None) for a, b in skf.split(X=label, y=label)]
    if group_sizes is not None:
        sizes = np.asarray(group_sizes, np.int64)
        bounds = np.r_[0, np.cumsum(sizes)]
        idx = np.random.permutation(sizes.size) if shuffle else np.arange(sizes.size)
        out_g = np.array_split(idx, nfold)
        in_g = [np.concatenate([out_g[i] for i in range(nfold) if i != k]) for k in range(nfold)]

        def to_rows(groups):
            return np.concatenate([np.arange(bounds[g], bounds[g + 1]) for g in groups] or [np.zeros(0, np.int64)])

        return [(to_rows(in_g[k]), to_rows(out_g[k]), sizes[in_g[k]], sizes[out_g[k]]) for k in range(nfold)]
    idx = np.random.permutation(n_rows) if shuffle else np.arange(n_rows)
    out_idx = np.array_split(idx, nfold)
    return [(np.concatenate([out_idx[i] for i in range(nfold) if i != k]), out_idx[k], None, None) for k in range(nfold)]


def aggcv(rlist):
    """xgboost's _aggcv: the eval_set strings of the folds of one round -> [(key, mean, std)], one per 'data-metric'
    entry in the strings' order; mean and std (np.std, population) of the printed %.6f values."""
    cvmap = {}
    it = rlist[0].split()[0]
    for line in rlist:
        arr = line.split()
        if arr[0] != it:
            raise XGBoostError("cv: folds evaluated different rounds (%s, %s)" % (it, arr[0]))
        for i, tok in enumerate(arr[1:]):
            k, v = tok.rsplit(":", 1)
            cvmap.setdefault((i, k), []).append(float(v))
    return [(k, float(np.mean(v)), float(np.std(v))) for (_, k), v in sorted(cvmap.items(), key=lambda x: x[0][0])]


class _PackedBooster:
    """The fold boosters of cv() as one model for the callbacks (xgboost's _PackedBooster): set_param, attributes and
    best_iteration / best_score reach every fold; the rest is read from fold 0."""

    def __init__(self, boosters):
        self.boosters = boosters

    def num_boosted_rounds(self):
        return self.boosters[0].num_boosted_rounds()

    def set_param(self, params, value=None):
        for b in self.boosters:
            b.set_param(params, value)

    def set_attr(self, **kwargs):
        for b in self.boosters:
            b.set_attr(**kwargs)

    def attr(self, key):
        return self.boosters[0].attr(key)

    @property
    def best_iteration(self):
        return self.boosters[0].best_iteration

    @best_iteration.setter
    def best_iteration(self, v):
        for b in self.boosters:
            b.best_iteration = v

    @property
    def best_score(self):
        return self.boosters[0].best_score

    @best_score.setter
    def best_score(self, v):
        for b in self.boosters:
            b.best_score = v


class _CVMonitor(TrainingCallback):
    """xgboost's EvaluationMonitor under cv(): '[i]\\tdata-metric:mean+std...' (%.5f; without '+std' if not
    show_stdv) every `period` rounds, and the last round at the end if it was not printed."""

    def __init__(self, period, show_stdv):
        self.period, self.show_stdv, self.latest = int(period), bool(show_stdv), None

    def after_iteration(self, model, epoch, evals_log):
        msg = "[%d]" % epoch
        for data, log in evals_log.items():
            for metric, vals in log.items():
                mean, std = vals[-1]
                msg += ("\t%s-%s:%.5f+%.5f" % (data, metric, mean, std) if self.show_stdv
                        else "\t%s-%s:%.5f" % (data, metric, mean))
        if epoch % self.period == 0 or self.period == 1:
            if _coll.rank == 0:
                print(msg, flush=True)
            self.latest = None
        else:
            self.latest = msg
        return False

    def after_training(self, model):
        if self.latest is not None and _coll.rank == 0:
            print(self.latest, flush=True)
        return model


def cv(params, dtrain, num_boost_round=10, nfold=3, stratified=False, folds=None, metrics=(), obj=None, feval=None,
       maximize=None, early_stopping_rounds=None, fpreproc=None, as_pandas=True, verbose_eval=None, show_stdv=True,
       seed=0, callbacks=None, shuffle=True, custom_metric=None):
    """xgboost.cv: k-fold cross-validation.  Returns, per round, the mean and std over the folds of every metric on the
    train and test side of each fold: keys 'train-<m>-mean', 'train-<m>-std', 'test-<m>-mean', 'test-<m>-std'; a pandas
    DataFrame when as_pandas and pandas is importable, else a dict of lists.

    The folds are cv_folds(...); each side is dtrain.slice(rows) (gathered on the device), with set_group for a matrix
    split by query groups.  fpreproc(dtrain_k, dtest_k, params.copy()) may replace both and the params.  A non-empty
    `metrics` replaces eval_metric.  Each fold trains one Booster on [(train, 'train'), (test, 'test')]; in every round
    all folds' rounds are enqueued before any metric is read back, and each fold computes what train() computes on its
    slices.  obj and custom_metric / feval take the paths of train().

    The callbacks see one model for all folds and a history of (mean, std) pairs.  early_stopping_rounds (with
    maximize) adds EarlyStopping on the last metric of 'test'; verbose_eval (True or a period) with show_stdv prints
    the rounds.  When a callback stops training, every list is cut to best_iteration + 1 rounds.  LearningRateScheduler
    sets the rate of every fold.  EarlyStopping(save_best=True) is refused: there is no single model to cut.  These
    rules are recalled from xgboost 2.x, not checked against its source (DESIGN.md 2 item 24)."""
    callbacks = list(callbacks or [])
    for cb in callbacks:
        if isinstance(cb, EarlyStopping) and cb.save_best:
            raise XGBoostError("cv: EarlyStopping(save_best=True) is not supported: cv returns the evaluation history "
                               "of several fold models, not one model to keep the best rounds of")
    feval = custom_metric if custom_metric is not None else feval
    if isinstance(params, (list, tuple)):
        listed = [v for k, v in params if k == "eval_metric"]
        params = dict(params)
        if listed:
            params["eval_metric"] = listed
    else:
        params = _params_dict(params)
    metrics = [metrics] if isinstance(metrics, str) else list(metrics)
    if not metrics and "eval_metric" in params:
        m = params["eval_metric"]
        metrics = list(m) if isinstance(m, (list, tuple)) else [m]
    params.pop("eval_metric", None)

    spec = cv_folds(dtrain.num_row(), nfold, label=dtrain.get_label(), group_sizes=dtrain._group_sizes,
                    stratified=stratified, folds=folds, seed=seed, shuffle=shuffle)
    packs = []
    for in_idx, out_idx, in_groups, out_groups in spec:
        grouped = in_groups is not None
        d_in, d_out = dtrain.slice(in_idx, allow_groups=grouped), dtrain.slice(out_idx, allow_groups=grouped)
        if grouped:
            d_in.set_group(in_groups)
            d_out.set_group(out_groups)
        tparams = dict(params)
        if fpreproc is not None:
            d_in, d_out, tparams = fpreproc(d_in, d_out, dict(params))
        if metrics:
            tparams = dict(tparams, eval_metric=list(metrics))
        bst = Booster(tparams)
        bst._attach(d_in)
        packs.append((bst, d_in, d_out))
    model = _PackedBooster([p[0] for p in packs])
    if verbose_eval:
        callbacks.append(_CVMonitor(1 if verbose_eval is True else verbose_eval, show_stdv))
    if early_stopping_rounds:
        callbacks.append(EarlyStopping(early_stopping_rounds, maximize=maximize))
    for cb in callbacks:
        cb.before_training(model)
    results, history = {}, {}
    for epoch in range(num_boost_round):
        if any(cb.before_iteration(model, epoch, history) for cb in callbacks):
            break
        for bst, d_in, _ in packs:   # every fold's round is enqueued before any metric is read back
            bst.update(d_in, epoch, fobj=obj)
        msgs = [bst.eval_set([(d_in, "train"), (d_out, "test")], epoch, feval, output_margin=obj is not None)
                for bst, d_in, d_out in packs]
        for key, mean, std in aggcv(msgs):
            data, metric = key.split("-", 1)
            history.setdefault(data, {}).setdefault(metric, []).append((mean, std))
            results.setdefault(key + "-mean", []).append(mean)
            results.setdefault(key + "-std", []).append(std)
        stop = False
        for cb in callbacks:
            if cb.after_iteration(model, epoch, history):
                stop = True
        if stop:
            if model.best_iteration is not None:
                results = {k: v[: model.best_iteration + 1] for k, v in results.items()}
            break
    for cb in callbacks:
        cb.after_training(model)
    if as_pandas:
        try:
            import pandas as pd
        except ImportError:
            return results
        return pd.DataFrame.from_dict(results)
    return results


def hist_build_raw(bins, qg, qh, ridx=None, window_rows=8192, chunk_rows=2048, device=None):
    """Kernel-level entry (tests / roofline probe): returns (hist [F,256,2] int64, kernel_ms)."""
    bins = np.ascontiguousarray(bins, np.uint8)
    n, f = bins.shape
    qg = np.ascontiguousarray(qg, np.int32)
    qh = np.ascontiguousarray(qh, np.int32)
    ri = None if ridx is None else np.ascontiguousarray(ridx, np.int32)
    nsel = n if ri is None else ri.size
    out = np.zeros((f, 256, 2), np.int64)
    ms = C.c_float(0)
    _check(lib().B2_HistBuildRaw(_bp(bins), n, f, _ip(qg), _ip(qh), _ip(ri), nsel, window_rows, chunk_rows,
                                 _default_device() if device is None else device,
                                 out.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(ms)))
    return out, ms.value


def hist_build_raw_csr(indptr, indices, bins, n_cols, qg, qh, ridx=None, chunk_rows=2048, device=None):
    """Kernel-level entry (tests): hist_build_raw's histogram from the CSR bin layout, one bin per stored entry
    (absent entries have bin 255).  Returns (hist [F,256,2] int64, kernel_ms)."""
    indptr = np.ascontiguousarray(indptr, np.int64)
    indices = np.ascontiguousarray(indices, np.int32)
    bins = np.ascontiguousarray(bins, np.uint8)
    n = indptr.size - 1
    if indices.size != indptr[-1] or bins.size != indptr[-1]:
        raise ValueError("indices and bins must hold indptr[-1] entries")
    qg = np.ascontiguousarray(qg, np.int32)
    qh = np.ascontiguousarray(qh, np.int32)
    ri = None if ridx is None else np.ascontiguousarray(ridx, np.int32)
    nsel = n if ri is None else ri.size
    out = np.zeros((n_cols, 256, 2), np.int64)
    ms = C.c_float(0)
    _check(lib().B2_HistBuildRawCSR(indptr.ctypes.data_as(_LP), _ip(indices), _bp(bins), n, n_cols, _ip(qg), _ip(qh), _ip(ri),
                                    nsel, chunk_rows, _default_device() if device is None else device,
                                    out.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(ms)))
    return out, ms.value


def quantize_raw(g, h, qbits, device=None):
    """Kernel-level entry (tests): the training path's fixed-point quantisation of gradient pairs.  Returns
    (qg, qh, (eg, eh)): q = rint(v * 2^(qbits - e)), e the frexp exponent of max |v| (0 when every v is 0)."""
    g = np.ascontiguousarray(g, np.float32)
    h = np.ascontiguousarray(h, np.float32)
    if g.shape != h.shape or g.ndim != 1:
        raise ValueError("g and h must be 1-d arrays of the same length")
    q = np.zeros((g.size, 2), np.int32)
    e = np.zeros(2, np.int32)
    _check(lib().B2_QuantizeRaw(_fp(g), _fp(h), g.size, int(qbits), _default_device() if device is None else device,
                                _ip(q), _ip(e)))
    return q[:, 0].copy(), q[:, 1].copy(), (int(e[0]), int(e[1]))
