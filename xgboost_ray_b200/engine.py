"""ctypes binding of libb2hist.so + the `xgboost`-shaped objects the actor code uses.

This module is the import seam the reference keeps in ``xgboost_ray/xgb.py:1-11``: the names
``DMatrix``, ``QuantileDMatrix``, ``DeviceQuantileDMatrix``, ``Booster``, ``train``,
``collective.CommunicatorContext`` and ``callback.TrainingCallback`` are what
``xgboost_ray/main.py`` uses from the ``xgboost`` package (sites main.py:386, 418, 437, 724,
745-752, 804; session.py:73), re-implemented on top of the sm_90a engine (include/b2hist.h).

There is NO CPU fallback: if the CUDA extension is not built or no H100 is visible, the first
compute call raises ``XGBoostError``.
"""
import ctypes as C
import json
import os
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
_H = C.c_uint64

# name -> (restype, argtypes); every symbol declared in include/b2hist.h
ABI = {
    "B2_GetLastError": (C.c_char_p, []),
    "B2_GetVersion": (C.c_int, []),
    "B2_SetOption": (C.c_int, [C.c_char_p, C.c_char_p]),
    "B2_DeviceCount": (C.c_int, [C.POINTER(C.c_int)]),
    "B2_GetUniqueId": (C.c_int, [_BP]),
    "B2_CommCreate": (C.c_int, [_BP, C.c_int, C.c_int, C.c_int, C.POINTER(_H)]),
    "B2_CommRank": (C.c_int, [_H, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "B2_CommAllReduce": (C.c_int, [_H, _DP, C.c_int32, C.c_int32]),
    "B2_CommAbort": (C.c_int, [_H]),
    "B2_CommFree": (C.c_int, [_H]),
    "B2_MatrixCreateFromDense": (C.c_int, [_FP, C.c_int64, C.c_int32, C.c_float, C.c_int, C.POINTER(_H)]),
    "B2_MatrixCreate": (C.c_int, [C.c_int64, C.c_int32, C.c_float, C.c_int, C.POINTER(_H)]),
    "B2_MatrixCreateFromProcessInterleaved": (C.c_int, [C.c_int64, C.c_uint64, C.c_int64, C.c_int32, C.c_int32, _H,
                                                        C.c_float, C.c_int, C.POINTER(_H)]),
    "B2_MatrixCreateFromProcess": (C.c_int, [C.c_int64, C.c_uint64, C.c_int64, C.c_int64, C.c_int32, C.c_float, C.c_int,
                                             C.POINTER(_H)]),
    "B2_MatrixSetRows": (C.c_int, [_H, C.c_int64, _FP, C.c_int64]),
    "B2_MatrixSetFloatInfo": (C.c_int, [_H, C.c_char_p, _FP, C.c_int64]),
    "B2_MatrixSetGroups": (C.c_int, [_H, _IP, C.c_int64]),
    "B2_MatrixSetFeatureTypes": (C.c_int, [_H, _BP, C.c_int32]),
    "B2_MatrixGetFeatureTypes": (C.c_int, [_H, _BP]),
    "B2_MatrixNumRow": (C.c_int, [_H, C.POINTER(C.c_int64)]),
    "B2_MatrixNumCol": (C.c_int, [_H, C.POINTER(C.c_int32)]),
    "B2_MatrixQuantize": (C.c_int, [_H, _H, C.c_int32, _H, C.c_int32]),
    "B2_MatrixQuantizeWithCuts": (C.c_int, [_H, _IP, _FP, _FP, _BP, C.c_int32, C.c_int32]),
    "B2_MatrixEnsureRaw": (C.c_int, [_H, _FP]),
    "B2_MatrixCutsSize": (C.c_int, [_H, _IP]),
    "B2_MatrixGetCuts": (C.c_int, [_H, _IP, _FP, _FP, _BP]),
    "B2_MatrixGetBins": (C.c_int, [_H, _BP]),
    "B2_MatrixFree": (C.c_int, [_H]),
    "B2_BoosterCreate": (C.c_int, [C.c_char_p, _H, _H, C.POINTER(_H)]),
    "B2_BoosterUpdateOneIter": (C.c_int, [_H, C.c_int32]),
    "B2_BoosterBoostOneIter": (C.c_int, [_H, _FP, _FP, C.c_int64]),
    "B2_BoosterGetGradients": (C.c_int, [_H, _FP, _FP, C.c_int64]),
    "B2_BoosterEvalSet": (C.c_int, [_H, _H, C.c_char_p, _DP]),
    "B2_BoosterPredict": (C.c_int, [_H, _H, C.c_int32, C.c_int32, C.c_int32, _FP, C.c_int64]),
    "B2_BoosterPredictContribs": (C.c_int, [_H, _H, C.c_int32, C.c_int32, C.c_int32, _FP, C.c_int64]),
    "B2_BoosterPredictLeaf": (C.c_int, [_H, _H, C.c_int32, C.c_int32, _FP, C.c_int64]),
    "B2_BoosterGetTrainMargin": (C.c_int, [_H, _FP, C.c_int64]),
    "B2_BoosterResetTrainMargin": (C.c_int, [_H]),
    "B2_BoosterGetBaseScore": (C.c_int, [_H, _FP, _IP]),
    "B2_BoosterNumTrees": (C.c_int, [_H, _IP]),
    "B2_BoosterTreeNumNodes": (C.c_int, [_H, C.c_int32, _IP]),
    "B2_BoosterGetTree": (C.c_int, [_H, C.c_int32, _IP, _IP, _IP, _IP, _IP, _FP, _BP, _FP, _FP, _FP, _DP]),
    "B2_BoosterAddTree": (C.c_int, [_H, C.c_int32, _IP, _IP, _IP, _IP, _IP, _FP, _BP, _FP, _FP, _FP, _DP]),
    "B2_BoosterGetTreeCategories": (C.c_int, [_H, C.c_int32, _BP, C.POINTER(C.c_uint32)]),
    "B2_BoosterSetTreeCategories": (C.c_int, [_H, C.c_int32, _BP, C.POINTER(C.c_uint32)]),
    "B2_BoosterGetTimers": (C.c_int, [_H, C.c_int32, C.c_char_p, C.c_int64]),
    "B2_BoosterCancel": (C.c_int, [_H]),
    "B2_BoosterFree": (C.c_int, [_H]),
    "B2_HistBuildRaw": (C.c_int, [_BP, C.c_int64, C.c_int32, _IP, _IP, _IP, C.c_int64, C.c_int32, C.c_int32, C.c_int,
                                  C.POINTER(C.c_int64), _FP]),
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


# ----------------------------------------------------------------------------- DMatrix
class DMatrix:
    """Device matrix.  Float data is uploaded at construction; quantisation (GPU sketch + binning)
    happens when a Booster first trains on it, because cuts are global over the communicator."""

    def __init__(self, data, label=None, weight=None, base_margin=None, missing=None, feature_names=None,
                 feature_types=None, nthread=None, enable_categorical=False, max_bin=None, ref=None,
                 device=None, label_lower_bound=None, label_upper_bound=None, qid=None, group=None, **kwargs):
        if hasattr(data, "values") and not isinstance(data, np.ndarray):  # pandas
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
        if remote is not None:                                     # rows of another process (matrix.RemoteBlock)
            data = remote
        elif hasattr(data, "next") and hasattr(data, "reset"):       # xgboost.DataIter protocol (matrix.py:127-196)
            blocks, label, weight, base_margin = _drain_data_iter(data, label, weight, base_margin)
        elif isinstance(data, (list, tuple)) and data and all(hasattr(b, "shape") for b in data):
            blocks = [np.asarray(b.values if hasattr(b, "values") and not isinstance(b, np.ndarray) else b) for b in data]
        if remote is not None:
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
        self._host = data
        self.missing = float("nan") if missing is None else float(missing)
        self.device = _default_device() if device is None else int(device)
        self.feature_names = list(feature_names) if feature_names is not None else None
        self.feature_types = list(feature_types) if feature_types is not None else None
        self.enable_categorical = bool(enable_categorical)
        self.max_bin = max_bin
        self.ref = ref
        self._quantized = False
        self._has_raw = True
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
        elif isinstance(self._host, _BlockList):
            # several row blocks (multi-file shard / DataIter): one device allocation, each block uploaded at its row
            # offset -- the host never concatenates them
            _check(lib().B2_MatrixCreate(n, f, self.missing, self.device, C.byref(h)))
            self.handle = h.value
            self._upload_blocks()
        else:
            _check(lib().B2_MatrixCreateFromDense(_fp(self._host), n, f, self.missing, self.device, C.byref(h)))
            self.handle = h.value
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
            a = _f32c(np.asarray(v).reshape(-1))
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
            _check(lib().B2_MatrixQuantizeWithCuts(self.handle, _ip(ptrs), _fp(vals), _fp(mins), _bp(hm), mb, 1 if keep_raw else 0))
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
            if isinstance(self._host, _BlockList):   # rare (predicting on a block-built training matrix): one host copy
                self._host = np.concatenate(self._host.blocks, axis=0)
            elif not isinstance(self._host, np.ndarray):   # rows of another process: fetch them once
                self._host = _f32c(np.asarray(self._host))
            _check(lib().B2_MatrixEnsureRaw(self.handle, _fp(self._host)))
            self._has_raw = True

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


def _drain_data_iter(it, label, weight, base_margin):
    """Pull every batch out of an xgboost.DataIter-style object: `it.next(input_data)` calls `input_data(data=...,
    label=..., weight=..., base_margin=...)` once per batch and returns 0 at the end (matrix.py:166-196)."""
    got = {"data": [], "label": [], "weight": [], "base_margin": []}

    def input_data(data=None, label=None, weight=None, base_margin=None, **kw):
        got["data"].append(np.asarray(data.values if hasattr(data, "values") and not isinstance(data, np.ndarray) else data))
        for k, v in (("label", label), ("weight", weight), ("base_margin", base_margin)):
            if v is not None:
                got[k].append(np.asarray(v.values if hasattr(v, "values") and not isinstance(v, np.ndarray) else v).reshape(-1))

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


class callback:  # namespace shim: xgb.callback.TrainingCallback
    TrainingCallback = TrainingCallback


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
        if self.metric == "ndcg":              # ranking: ndcg at the objective's pair cut-off
            return "ndcg@%d" % int(params.get("lambdarank_num_pair_per_sample", 32))
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
    "multi:softprob": _Objective("mlogloss", "softmax", *_SOFTMAX),
    "multi:softmax": _Objective("mlogloss", "softmax", *_SOFTMAX),
}


def _objective(name):
    o = _OBJECTIVES.get(name)
    if o is None:
        raise XGBoostError("unsupported objective '%s' (supported: %s)" % (name, ", ".join(sorted(_OBJECTIVES))))
    return o


_TREE_FIELDS = ("left", "right", "parent", "split_feature", "split_bin", "split_cond", "default_left", "value",
                "base_weight", "loss_chg", "sum_hess")
_ENGINE_KEYS = ("objective", "num_class", "max_depth", "eta", "learning_rate", "gamma", "min_split_loss",
                "min_child_weight", "lambda", "reg_lambda", "alpha", "reg_alpha", "base_score", "hist_qbits",
                "hist_chunk_rows", "profile", "max_cat_to_onehot", "max_cat_threshold", "scale_pos_weight",
                "max_delta_step", "subsample", "colsample_bytree", "colsample_bylevel", "colsample_bynode", "seed",
                "random_state", "num_parallel_tree", "huber_slope", "tweedie_variance_power", "aft_loss_distribution",
                "aft_loss_distribution_scale", "lambdarank_pair_method", "lambdarank_num_pair_per_sample",
                "lambdarank_unbiased", "ndcg_exp_gain")

# xgboost parameters that change the trained model and that this engine does not implement: a value different
# from the neutral one is an error, never silently ignored (a drop-in must not train a different model quietly)
_UNSUPPORTED_NEUTRAL = {
    "sampling_method": ("uniform",), "max_leaves": (0,), "grow_policy": ("depthwise",),
    "monotone_constraints": (None, "", "()", (), []), "interaction_constraints": (None, "", "[]", (), []),
    "multi_strategy": ("one_output_per_tree",), "refresh_leaf": (1, True), "process_type": ("default",),
    "updater": (None, "grow_quantile_histmaker", "grow_gpu_hist"),
}


def _check_supported(params):
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


def _params_dict(params):
    if params is None:
        return {}
    if isinstance(params, (list, tuple)):
        return dict(params)
    return dict(params)


class Booster:
    def __init__(self, params=None, cache=(), model_file=None):
        self.params = _params_dict(params)
        self.handle = 0
        self._train = None
        self._trees = []          # list of dict of numpy arrays (host copy for pickling / dumps)
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
        if self.params.get("booster", "gbtree") != "gbtree":
            raise XGBoostError("only booster=gbtree is supported")
        for d in cache:
            if isinstance(d, DMatrix) and self._train is None:
                self._attach(d)
        if model_file is not None:
            self.load_model(model_file)

    # -- engine object management
    def _param_text(self, extra=None):
        _check_supported(self.params)
        p = {k: self.params[k] for k in _ENGINE_KEYS if k in self.params and self.params[k] is not None}
        if extra:
            p.update(extra)
        return "\n".join("%s=%s" % (k, v) for k, v in p.items()).encode()

    def _attach(self, dtrain):
        """Create the device booster bound to `dtrain` (quantising it if needed)."""
        old_trees = self.get_trees() if (self.handle or self._trees) else []
        self._free()
        dtrain._ensure_quantized(int(self.params.get("max_bin", 256)), cuts=self._cuts if old_trees else None)
        self._cuts = dtrain.get_cuts()
        h = _H(0)
        _check(lib().B2_BoosterCreate(self._param_text(), dtrain.handle, _coll.handle, C.byref(h)))
        self.handle = h.value
        self._train = dtrain
        self.n_features = dtrain.num_col()
        if self.feature_names is None:
            self.feature_names = dtrain.feature_names
        if getattr(self, "feature_types", None) is None:
            self.feature_types = dtrain.feature_types
        if old_trees:
            dtrain._ensure_raw()
            self._push_trees(old_trees)
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
        self._push_trees(self._trees)

    def _push_trees(self, trees):
        for t in trees:
            n = len(t["left"])
            _check(lib().B2_BoosterAddTree(
                self.handle, n, _ip(np.ascontiguousarray(t["left"], np.int32)),
                _ip(np.ascontiguousarray(t["right"], np.int32)), _ip(np.ascontiguousarray(t["parent"], np.int32)),
                _ip(np.ascontiguousarray(t["split_feature"], np.int32)),
                _ip(np.ascontiguousarray(t["split_bin"], np.int32)), _fp(_f32c(t["split_cond"])),
                _bp(np.ascontiguousarray(t["default_left"], np.uint8)), _fp(_f32c(t["value"])),
                _fp(_f32c(t["base_weight"])), _fp(_f32c(t["loss_chg"])),
                np.ascontiguousarray(t["sum_hess"], np.float64).ctypes.data_as(_DP)))
            st = t.get("split_type")
            if st is not None and np.any(st):
                nt = C.c_int32(0)
                _check(lib().B2_BoosterNumTrees(self.handle, C.byref(nt)))
                _check(lib().B2_BoosterSetTreeCategories(
                    self.handle, nt.value - 1, _bp(np.ascontiguousarray(st, np.uint8)),
                    np.ascontiguousarray(t["cat_bits"], np.uint32).ctypes.data_as(C.POINTER(C.c_uint32))))

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

    @property
    def num_class(self):
        obj = self.params.get("objective", "reg:squarederror")
        return int(self.params.get("num_class", 1)) if obj.startswith("multi:") else 1

    @property
    def num_parallel_tree(self):
        return max(1, int(self.params.get("num_parallel_tree", 1) or 1))

    def num_boosted_rounds(self):
        return self.num_trees() // max(1, self.num_class * self.num_parallel_tree)

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
        _check(lib().B2_BoosterGetTreeCategories(self.handle, i, _bp(t["split_type"]),
                                                 t["cat_bits"].ctypes.data_as(C.POINTER(C.c_uint32))))
        _check(lib().B2_BoosterGetTree(self.handle, i, _ip(t["left"]), _ip(t["right"]), _ip(t["parent"]),
                                       _ip(t["split_feature"]), _ip(t["split_bin"]), _fp(t["split_cond"]),
                                       _bp(t["default_left"]), _fp(t["value"]), _fp(t["base_weight"]),
                                       _fp(t["loss_chg"]), t["sum_hess"].ctypes.data_as(_DP)))
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
        _check(lib().B2_BoosterUpdateOneIter(self.handle, int(iteration)))
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
        _check(lib().B2_BoosterBoostOneIter(self.handle, _fp(g), _fp(h), g.size))
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
                pred = self.predict(dm, output_margin=output_margin, training=(dm is self._train))
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
        per_round = self.num_class * self.num_parallel_tree
        tb, te = iteration_range if iteration_range else (0, 0)
        if ntree_limit:
            return 0, int(ntree_limit)
        return int(tb) * per_round, int(te) * per_round

    def predict(self, data, output_margin=False, ntree_limit=0, validate_features=True, training=False,
                iteration_range=(0, 0), strict_shape=False, pred_leaf=False, pred_contribs=False, approx_contribs=False,
                pred_interactions=False, **kwargs):
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
            _check(lib().B2_BoosterGetTrainMargin(self.handle, _fp(out), out.size))
            if not output_margin:
                out = _transform(self.params.get("objective", "reg:squarederror"), out.reshape(n, K)).reshape(-1)
        else:
            data._ensure_raw()
            tb, te = iteration_range if iteration_range else (0, 0)
            tb_t, te_trees = tb * K * self.num_parallel_tree, te * K * self.num_parallel_tree
            if ntree_limit:
                tb_t, te_trees = 0, ntree_limit
            _check(lib().B2_BoosterPredict(self.handle, data.handle, 1 if output_margin else 0, tb_t, te_trees,
                                           _fp(out), out.size))
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
        if isinstance(params, str):
            params = {params: value}
        self.params.update(_params_dict(params))

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
        cond = np.where(np.isfinite(cond), cond, np.float32(0.0))
        return {
            "base_weights": [float(x) for x in t["base_weight"]],
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
                           "size_leaf_vector": "1"},
        }

    def _model_dict(self):
        K = self.num_class
        src = self.get_trees()
        cache = self.__dict__.setdefault("_tree_json_cache", [])     # finished trees never change: convert each once
        if len(cache) > len(src):
            del cache[:]
        for i in range(len(cache), len(src)):
            cache.append((self._tree_json(i, src[i], self.n_features), [int(x) for x in src[i]["split_bin"]]))
        trees = [c[0] for c in cache]
        obj = self.params.get("objective", "reg:squarederror")
        spec = _OBJECTIVES.get(obj, _OBJECTIVES["reg:squarederror"])
        obj_block = {"name": obj}
        if spec.block:
            obj_block[spec.block] = {k: str(K) if k == "num_class" else
                                     _str_param(self.params.get(k, d)) if isinstance(d, str) else _num_str(self.params.get(k, d))
                                     for k, d in spec.block_params.items()}
        attrs = {k: str(v) for k, v in self._attrs.items() if not k.startswith("b2.")}
        attrs["b2.params"] = json.dumps({k: self.params[k] for k in sorted(self.params) if _json_ok(self.params[k]) and
                                         k not in ("objective", "num_class", "base_score", "scale_pos_weight", "num_parallel_tree")})   # those have their own fields
        attrs["b2.split_bins"] = json.dumps([c[1] for c in cache], separators=(",", ":"))
        return {
            "learner": {
                "attributes": attrs,
                "feature_names": [str(x) for x in (self.feature_names or [])],
                "feature_types": [_xgb_feature_type(x) for x in (self.feature_types or [])],
                "gradient_booster": {"model": {
                    "gbtree_model_param": {"num_parallel_tree": str(self.num_parallel_tree), "num_trees": str(len(trees))},
                    "iteration_indptr": list(range(0, len(trees) + 1, K * self.num_parallel_tree)),
                    "tree_info": [(i // self.num_parallel_tree) % K for i in range(len(trees))],
                    "trees": trees}, "name": "gbtree"},
                "learner_model_param": {"base_score": _num_str(self.params.get("base_score", 0.5) if self.params.get("base_score") is not None else 0.5),
                                        "boost_from_average": "1", "num_class": str(K if K > 1 else 0),
                                        "num_feature": str(self.n_features), "num_target": "1"},
                "objective": obj_block,
            },
            "version": [2, 0, 3],
        }

    def save_raw(self, raw_format="json"):
        return bytearray(json.dumps(self._model_dict(), allow_nan=False).encode())

    def save_model(self, fname):
        with open(fname, "wb") as f:
            f.write(bytes(self.save_raw()))

    def load_model(self, fname):
        if isinstance(fname, (bytes, bytearray)):
            raw = bytes(fname)
        else:
            with open(fname, "rb") as f:
                raw = f.read()
        d = json.loads(raw.decode())
        L = d["learner"]
        self._free()
        self.__dict__.pop("_tree_json_cache", None)
        attrs = dict(L.get("attributes", {}))
        params = dict(json.loads(attrs.pop("b2.params"))) if "b2.params" in attrs else dict(L.get("b2_params", {}))
        split_bins = json.loads(attrs.pop("b2.split_bins")) if "b2.split_bins" in attrs else None
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
        npt = int(L["gradient_booster"]["model"].get("gbtree_model_param", {}).get("num_parallel_tree", "1"))
        if npt > 1:
            params["num_parallel_tree"] = npt
        params.update({k: v for k, v in self.params.items() if k not in params})
        self.params = params
        self.n_features = int(L["learner_model_param"]["num_feature"])
        self.feature_names = L.get("feature_names") or None
        self.feature_types = [_b2_feature_type(x) for x in L.get("feature_types") or []] or None
        self._attrs = attrs
        self._trees = []
        for ti, t in enumerate(L["gradient_booster"]["model"]["trees"]):
            left = np.asarray(t["left_children"], np.int32)
            leaf = left < 0
            sc = np.asarray(t["split_conditions"], np.float32)
            parent = np.asarray([p if p != 2147483647 else -1 for p in t["parents"]], np.int32)
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
            ncat = np.array([bin(int(w)).count("1") for w in bits.reshape(len(left), -1).astype(np.uint64).sum(axis=1)]) if False else None
            cond = np.where(leaf, 0, sc).astype(np.float32)
            for nid in np.nonzero(cat_split)[0]:
                cl = _cat_list(bits[nid])
                b_ = int(sb[nid]) if sb is not None else (cl[0] if len(cl) == 1 else -1)
                cond[nid] = np.float32(b_) if b_ >= 0 else np.float32("nan")
            self._trees.append(dict(
                split_type=st, cat_bits=bits,
                left=left, right=np.asarray(t["right_children"], np.int32), parent=parent,
                split_feature=np.where(leaf, -1, np.asarray(t["split_indices"], np.int32)).astype(np.int32),
                split_bin=np.asarray(sb if sb is not None else [-1] * len(left), np.int32),
                split_cond=cond,
                default_left=np.asarray(t["default_left"], np.uint8),
                value=np.where(leaf, sc, np.asarray(t["base_weights"], np.float32)).astype(np.float32),
                base_weight=np.asarray(t["base_weights"], np.float32),
                loss_chg=np.asarray(t["loss_changes"], np.float32),
                sum_hess=np.asarray(t["sum_hessian"], np.float64)))

    def __getstate__(self):
        return {"raw": bytes(self.save_raw()), "best_iteration": self.best_iteration, "best_score": self.best_score,
                "cuts": self._cuts}

    def __setstate__(self, state):
        self.params = {}
        self.handle = 0
        self._train = None
        self._trees = []
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

    def save_config(self):
        return json.dumps({"learner": {"gradient_booster": {"name": "gbtree"},
                                       "objective": {"name": self.params.get("objective", "reg:squarederror")},
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
    """Metrics where larger is better (early stopping): auc, interval-regression-accuracy and every ndcg / map / pre
    form (ndcg@5, map-, pre@10, ...)."""
    if metric in ("auc", "interval-regression-accuracy"):
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
        d = {"nodeid": int(nid), "leaf": float(t["value"][nid])}
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
        s = "%s%d:leaf=%.9g" % (ind, nid, float(t["value"][nid]))
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
    if xgb_model is not None:
        if isinstance(xgb_model, Booster):
            src = xgb_model
            src.get_trees()
        else:
            src = Booster(params)
            src.load_model(xgb_model)
        bst._trees = list(src._trees)
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
    bst._attach(dtrain)
    evals = list(evals or [])
    for dm, _ in evals:
        if dm is not dtrain and dm.ref is None and not dm._quantized:
            pass  # evaluation matrices are traversed on raw floats; no quantisation needed
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


def set_option(key, value):
    """Process-wide engine option (B2_SetOption)."""
    _check(lib().B2_SetOption(str(key).encode(), str(value).encode()))


def hist_build_raw(bins, qg, qh, ridx=None, window_rows=8192, chunk_rows=2048, device=None, narrow=None):
    """Kernel-level entry (tests / roofline probe): returns (hist [F,256,2] int64, kernel_ms).  narrow = 0 / 1 selects
    the feature-group layout for this call (None: the process default)."""
    if narrow is not None:
        try:
            set_option("hist_narrow", int(narrow))
            return hist_build_raw(bins, qg, qh, ridx, window_rows, chunk_rows, device)
        finally:
            set_option("hist_narrow", 1 if os.environ.get("B2_HIST_NARROW", "0") not in ("", "0") else 0)
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
