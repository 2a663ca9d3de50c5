"""RayDMatrix: lazily loaded, row-sharded training / prediction data.

Host-side mirror of xgboost_ray/matrix.py for the hot path (SURVEY.md 8a rows a1-a3):
  RayShardingMode            matrix.py:105-124
  _get_sharding_indices      matrix.py:1088-1110  (here: slices / strided views, not Python int lists)
  combine_data               matrix.py:1113-1157
  RayDMatrix                 matrix.py:696-968    (central loading; FIXED file sharding for file lists)
  RayQuantileDMatrix / RayDeviceQuantileDMatrix   matrix.py:971-1033

One shard maps to one GPU actor.  A shard is a dict of float32 numpy blocks (data, label, weight,
base_margin, ...), which is what the device upload consumes; the Ray object store of the reference
is replaced by plain process-local references handed to the actor processes.
"""
import atexit
import copy
import os
import threading
import uuid
from concurrent.futures import ThreadPoolExecutor
from enum import Enum
from typing import Dict, Iterable, List, Optional, Sequence

import numpy as np

from xgboost_ray_b200.data_sources import LoadedFrame, RayFileType, resolve_data_source  # noqa: F401


class RayShardingMode(Enum):
    INTERLEAVED = 1
    BATCH = 2
    FIXED = 3


def _get_sharding_indices(sharding: RayShardingMode, rank: int, num_actors: int, n: int):
    """Rows of `rank`: a slice (zero-copy selection) -- same row sets as matrix.py:1088-1110."""
    if sharding == RayShardingMode.BATCH:
        n_per_actor, extras = divmod(n, num_actors)
        start = rank * n_per_actor + min(rank, extras)
        stop = start + n_per_actor + (1 if rank < extras else 0)
        return slice(start, stop)
    if sharding == RayShardingMode.INTERLEAVED:
        return slice(rank, n, num_actors)
    raise ValueError(
        f"Invalid value for `sharding` parameter: {sharding}"
        f"\nFIX THIS by passing any item of the `RayShardingMode` enum, for instance `RayShardingMode.BATCH`.")


def group_offsets(qid: np.ndarray) -> np.ndarray:
    """Row offsets of the query groups of a non-decreasing qid: a group is a maximal run of equal ids."""
    q = np.asarray(qid).reshape(-1)
    if q.size == 0:
        return np.zeros(1, np.int64)
    starts = np.flatnonzero(np.r_[True, q[1:] != q[:-1]])
    return np.r_[starts, q.size].astype(np.int64)


def group_sharding_rows(sharding: RayShardingMode, rank: int, num_actors: int, offsets: np.ndarray) -> np.ndarray:
    """Rows of `rank` when every query group goes whole to one actor: group g to rank g mod W (INTERLEAVED), or the
    group list split like numpy.array_split (BATCH).  A LambdaMART gradient depends on the rows of its group only, so
    whole groups make the gradients independent of the number of actors."""
    n_groups = len(offsets) - 1
    if n_groups < num_actors:
        raise ValueError(f"Trying to shard {n_groups} query groups (qid) over {num_actors} actors: every group goes "
                         f"whole to one actor, so there must be at least as many groups as actors."
                         f"\nFIX THIS by using at most {n_groups} actors.")
    if sharding == RayShardingMode.INTERLEAVED:
        groups = np.arange(rank, n_groups, num_actors)
    elif sharding == RayShardingMode.BATCH:
        groups = np.array_split(np.arange(n_groups), num_actors)[rank]
    else:
        raise ValueError(f"Invalid value for `sharding` parameter: {sharding}"
                         f"\nFIX THIS by passing any item of the `RayShardingMode` enum, for instance `RayShardingMode.BATCH`.")
    if len(groups) == 0:
        return np.zeros(0, np.int64)
    sizes = offsets[groups + 1] - offsets[groups]
    starts = np.repeat(offsets[groups] - np.r_[0, np.cumsum(sizes)[:-1]], sizes)
    return (starts + np.arange(int(sizes.sum()))).astype(np.int64)


def combine_by_index(row_index: Sequence[np.ndarray], data: Iterable) -> np.ndarray:
    """Reassemble per-actor prediction arrays whose rows are `row_index[rank]` (group-aligned shards)."""
    data = [np.asarray(d) for d in data]
    n = sum(len(ix) for ix in row_index)
    shaped = [d for d in data if len(d)]
    if not shaped:
        return np.zeros(0, np.float32)
    out = np.empty((n,) + shaped[0].shape[1:], dtype=shaped[0].dtype)
    for ix, d in zip(row_index, data):
        out[ix] = d
    return out


def combine_data(sharding: RayShardingMode, data: Iterable) -> np.ndarray:
    """Reassemble per-actor prediction arrays in original row order (matrix.py:1113-1157)."""
    if sharding not in (RayShardingMode.BATCH, RayShardingMode.INTERLEAVED):
        raise ValueError(
            f"Invalid value for `sharding` parameter: {sharding}"
            f"\nFIX THIS by passing any item of the `RayShardingMode` enum, for instance `RayShardingMode.BATCH`.")
    data = [np.asarray(d) for d in data if len(d)]
    if not data:
        return np.zeros(0, np.float32)
    if sharding == RayShardingMode.BATCH:
        return np.concatenate(data) if data[0].ndim == 1 else np.vstack(data)
    n = sum(len(d) for d in data)
    out = np.empty((n,) + data[0].shape[1:], dtype=data[0].dtype)
    for r, d in enumerate(data):
        out[r::len(data)] = d
    return out


# ---- shard hand-off through /dev/shm (the role of ray.put / the plasma store, matrix.py:471-484): the driver writes
# every shard ONCE, row-sliced straight out of the source array by several threads, into a memory-mapped .npy file; the
# actor process maps the file read-only and uploads from it.  Nothing is pickled through a pipe.
_SHM_FILES = set()
_SHM_LOCK = threading.Lock()


def _shm_dir() -> Optional[str]:
    d = os.environ.get("B2_SHM_DIR", "/dev/shm")
    return d if d and os.path.isdir(d) and os.access(d, os.W_OK) else None


def _cleanup_shm():
    with _SHM_LOCK:
        files = list(_SHM_FILES)
        _SHM_FILES.clear()
    for f in files:
        try:
            os.unlink(f)
        except OSError:
            pass


atexit.register(_cleanup_shm)
_COPY_POOL = None


def _copy_pool():
    global _COPY_POOL
    if _COPY_POOL is None:
        _COPY_POOL = ThreadPoolExecutor(max_workers=max(1, min(32, (os.cpu_count() or 1))))
    return _COPY_POOL


def _parallel_copy(dst: np.ndarray, src: np.ndarray):
    """dst[:] = src with the rows split over threads (numpy releases the GIL inside the copy loops)."""
    n = len(dst)
    if n == 0:
        return
    if dst.nbytes < (8 << 20):
        np.copyto(dst, src, casting="unsafe")
        return
    pool = _copy_pool()
    parts = pool._max_workers * 2
    step = (n + parts - 1) // parts
    list(pool.map(lambda i: np.copyto(dst[i:i + step], src[i:i + step], casting="unsafe"), range(0, n, step)))


def _shared_copy(src: Optional[np.ndarray], tag: str):
    """Copy `src` (any strided view) into a float32 .npy file under /dev/shm; returns (array view, ('shm', path)).
    Without a usable /dev/shm the copy stays in process memory and travels by pickle."""
    if src is None:
        return None, None
    d = _shm_dir()
    if d is not None:
        try:
            st = os.statvfs(d)
            if st.f_bavail * st.f_frsize < src.size * 4 + (64 << 20):
                d = None
        except OSError:
            d = None
    if d is None:
        a = np.empty(src.shape, np.float32)
        _parallel_copy(a, src)
        return a, a
    path = os.path.join(d, "b2x_%d_%s_%s.npy" % (os.getpid(), tag, uuid.uuid4().hex[:12]))
    a = np.lib.format.open_memmap(path, mode="w+", dtype=np.float32, shape=tuple(src.shape))
    with _SHM_LOCK:
        _SHM_FILES.add(path)
    _parallel_copy(a, src)
    return a, ("shm", path)


# ---- zero-copy hand-off: the actor reads its rows straight out of the DRIVER's memory (process_vm_readv) into the pinned
# upload buffers of the engine (B2_MatrixCreateFromProcess).  The shard is then never copied on the host at all; the
# /dev/shm files above remain the fallback when the kernel refuses the read (ptrace restrictions).
_PTRACE_ALLOWED = [False]


def allow_actors_to_read_this_process():
    """prctl(PR_SET_PTRACER, PR_SET_PTRACER_ANY): lets the actor processes (children) read this process' memory where the
    Yama LSM restricts ptrace to descendants.  A no-op error (EINVAL) where Yama is not in use."""
    if _PTRACE_ALLOWED[0]:
        return
    _PTRACE_ALLOWED[0] = True
    try:
        import ctypes
        libc = ctypes.CDLL("libc.so.6", use_errno=True)
        libc.prctl(0x59616D61, ctypes.c_ulong(0xFFFFFFFFFFFFFFFF), 0, 0, 0)
    except Exception:
        pass


class RemoteBlock:
    """n_rows x n_cols float32 rows living in process `pid` at `addr`, `row_stride` bytes apart."""

    def __init__(self, pid, addr, row_stride, n_rows, n_cols, interleave=None):
        self.pid, self.addr, self.row_stride = int(pid), int(addr), int(row_stride)
        # (address of the full C-contiguous matrix, its row count, shard rank, number of shards) when these rows are the
        # INTERLEAVED shard `rank` of that matrix: lets W ranks read 1/W each and redistribute on the device
        self.interleave = tuple(int(v) for v in interleave) if interleave else None
        self.shape = (int(n_rows), int(n_cols))
        self.ndim = 2
        self.dtype = np.dtype(np.float32)

    def __len__(self):
        return self.shape[0]

    def __array__(self, dtype=None, copy=None):
        """Materialise on the host (the CPU stand-in engine and rare re-uploads use this; the GPU path does not)."""
        import ctypes

        class _IoVec(ctypes.Structure):
            _fields_ = [("base", ctypes.c_void_p), ("len", ctypes.c_size_t)]

        libc = ctypes.CDLL("libc.so.6", use_errno=True)
        n, f = self.shape
        out = np.empty((n, f), np.float32)
        row_bytes = f * 4
        if n == 0:
            return out
        if self.row_stride == row_bytes:
            done, total = 0, n * row_bytes
            while done < total:
                lo = _IoVec(out.ctypes.data + done, total - done)
                ro = _IoVec(self.addr + done, total - done)
                got = libc.process_vm_readv(self.pid, ctypes.byref(lo), 1, ctypes.byref(ro), 1, 0)
                if got <= 0:
                    raise OSError(ctypes.get_errno(), "process_vm_readv failed: %s" % os.strerror(ctypes.get_errno()))
                done += got
        else:
            step = 512
            riov = (_IoVec * step)()
            for r0 in range(0, n, step):
                k = min(step, n - r0)
                for i in range(k):
                    riov[i].base = self.addr + (r0 + i) * self.row_stride
                    riov[i].len = row_bytes
                lo = _IoVec(out.ctypes.data + r0 * row_bytes, k * row_bytes)
                got = libc.process_vm_readv(self.pid, ctypes.byref(lo), 1, riov, k, 0)
                if got != k * row_bytes:
                    raise OSError(ctypes.get_errno(), "process_vm_readv failed: %s" % os.strerror(ctypes.get_errno()))
        return out if dtype is None else out.astype(dtype, copy=False)


def _column_or_array(frame: LoadedFrame, spec, exclude: set):
    """`spec` is None, a column name of the loaded frame, or an array-like of row values."""
    if spec is None:
        return None
    if isinstance(spec, str):
        exclude.add(spec)
        return np.ascontiguousarray(frame.column(spec), dtype=np.float32)
    if hasattr(spec, "values") and not isinstance(spec, np.ndarray):
        spec = spec.values
    return np.ascontiguousarray(np.asarray(spec), dtype=np.float32)


class RayDMatrix:
    """See xgboost_ray/matrix.py:696-786 for the argument contract."""

    def __init__(self, data, label=None, weight=None, feature_weights=None, base_margin=None, missing=None,
                 label_lower_bound=None, label_upper_bound=None, feature_names=None, feature_types=None, qid=None,
                 enable_categorical=None, num_actors: Optional[int] = None, filetype: Optional[RayFileType] = None,
                 ignore: Optional[List[str]] = None, distributed: Optional[bool] = None,
                 sharding: RayShardingMode = RayShardingMode.INTERLEAVED, lazy: bool = False, **kwargs):
        if kwargs.get("group", None) is not None:
            raise ValueError("`group` parameter is not supported. If you are using XGBoost-Ray, use `qid` parameter instead.")
        if qid is not None and weight is not None:
            raise NotImplementedError("per-group weight is not implemented.")
        self._uid = uuid.uuid4().int
        self.data, self.label, self.weight, self.base_margin = data, label, weight, base_margin
        self.feature_weights = feature_weights
        self.label_lower_bound, self.label_upper_bound = label_lower_bound, label_upper_bound
        self.feature_names, self.feature_types = feature_names, feature_types
        self.qid = qid
        self.enable_categorical = enable_categorical
        self.missing = missing
        self.num_actors = num_actors
        self.sharding = sharding
        self.filetype = filetype
        self.ignore = ignore
        self.kwargs = kwargs
        self.data_source = resolve_data_source(data, filetype)
        if distributed is None:
            distributed = _detect_distributed(self.data_source, data)
        elif distributed and not self.data_source.supports_distributed_loading:
            raise ValueError(f"Distributed data loading is not supported for input data of type {type(data)}. "
                             f"\nFIX THIS by passing file names or setting `distributed=False`.")
        self.distributed = bool(distributed)
        if self.distributed and qid is not None:
            raise ValueError("ranking (qid) with distributed loading (a list of files read by the actors) is not "
                             "supported: a query group may span files.\nFIX THIS by loading the data centrally "
                             "(`distributed=False`).")
        self._row_index: Optional[List[np.ndarray]] = None   # qid: rows of every rank in the qid-sorted order
        if self.distributed:
            self.sharding = RayShardingMode.FIXED if sharding == RayShardingMode.FIXED else sharding
        self.refs: Dict[int, Dict[str, Optional[np.ndarray]]] = {}
        self._shared: Dict[int, Dict] = {}      # rank -> {field: ('shm', path) | ndarray | None}: what an actor is sent
        self.n = None
        self.loaded = False
        self._columns = None
        self._inferred_types = None             # feature types of pandas `category` columns ('c' / 'q')
        if num_actors is not None and not lazy:
            self.load_data(num_actors)

    # -- reference API
    @property
    def has_label(self):
        return self.label is not None

    def assert_enough_shards_for_actors(self, num_actors: int):
        n = self.data_source.get_n(self.data)
        if self.distributed and num_actors > n:
            raise RuntimeError(f"Trying to shard data for {num_actors} actors, but the maximum number of shards "
                               f"(i.e. the number of data files) is {n}. Consider using fewer actors.")

    def assign_shards_to_actors(self, actors: Sequence) -> bool:
        return False  # locality-aware assignment only exists for distributed frames (out of scope)

    def _split(self, frame: LoadedFrame):
        exclude = set()
        y = _column_or_array(frame, self.label, exclude)
        w = _column_or_array(frame, self.weight, exclude)
        b = _column_or_array(frame, self.base_margin, exclude)
        ll = _column_or_array(frame, self.label_lower_bound, exclude)
        lu = _column_or_array(frame, self.label_upper_bound, exclude)
        fw = None if self.feature_weights is None else np.asarray(self.feature_weights, np.float32)
        q = None
        if self.qid is not None:                # the ids keep their dtype (float32 would merge large ids)
            if isinstance(self.qid, str):
                exclude.add(self.qid)
                q = np.asarray(frame.column(self.qid)).reshape(-1)
            else:
                q = np.asarray(self.qid.values if hasattr(self.qid, "values") and not isinstance(self.qid, np.ndarray)
                               else self.qid).reshape(-1)
        self._qid_rows = q
        x = frame.drop(exclude) if exclude else frame
        if x.feature_types is not None:
            if not self.enable_categorical:
                raise ValueError("The data has `category` columns. Pass `enable_categorical=True` to the RayDMatrix "
                                 "(they are trained on as categorical features) or convert them to numbers first.")
            if self.feature_types is None:
                self._inferred_types = list(x.feature_types)
        return x, y, w, fw, b, ll, lu

    def load_data(self, num_actors: Optional[int] = None, rank: Optional[int] = None, transport: Optional[str] = None):
        """Central loading (matrix.py:431-487): read once, shard per rank.  Distributed (file lists,
        matrix.py:614-693): rank r reads files r, r+W, ... itself.  transport = "remote": the feature matrix is NOT
        copied per shard -- every shard is a description of its rows inside this process that the actor reads directly
        (RemoteBlock); "shm" (default): shards are written to /dev/shm files."""
        if transport is not None:
            self._transport = transport
        if num_actors is not None:
            if self.num_actors is not None and num_actors != self.num_actors:
                raise ValueError(f"The `RayDMatrix` was initialized or `load_data()`has been called with a different "
                                 f"numbers of `actors`. Existing value: {self.num_actors}. Current value: {num_actors}."
                                 f"\nFIX THIS by not instantiating the matrix with `num_actors` and making sure "
                                 f"calls to `load_data()` or `get_data()` use the same numbers.")
            self.num_actors = num_actors
        if self.loaded and rank is None:
            return
        if self.num_actors is None:
            raise ValueError("Trying to load data for `RayDMatrix` object, but `num_actors` is not set."
                             "\nFIX THIS by passing `num_actors` on instantiation or when calling `load_data()`.")
        W = self.num_actors
        if self.distributed:
            self.assert_enough_shards_for_actors(W)
            ranks = [rank] if rank is not None else list(range(W))
            n_files = self.data_source.get_n(self.data)
            total = 0
            cat = lambda parts: None if parts[0] is None else np.concatenate(parts)  # noqa: E731
            for r in ranks:
                idx = list(range(n_files))[_get_sharding_indices(
                    RayShardingMode.INTERLEAVED if self.sharding != RayShardingMode.BATCH else RayShardingMode.BATCH,
                    r, W, n_files)]
                # one row block per file (matrix.py:127-196: the shards of an actor stay separate and go to the device
                # matrix one by one); only the small side columns are concatenated
                parts = [self._split(self.data_source.load_data(self.data, ignore=self.ignore, indices=[i], **self.kwargs))
                         for i in idx]
                self._columns = parts[0][0].columns
                blocks = [p[0].values for p in parts]
                self.refs[r] = {"data": blocks if len(blocks) > 1 else blocks[0], "label": cat([p[1] for p in parts]),
                                "weight": cat([p[2] for p in parts]), "feature_weights": parts[0][3],
                                "base_margin": cat([p[4] for p in parts]), "label_lower_bound": cat([p[5] for p in parts]),
                                "label_upper_bound": cat([p[6] for p in parts]), "qid": None}
                self._shared[r] = dict(self.refs[r])
                total += sum(len(b) for b in blocks)
            self.n = total if rank is None else self.n
            self.sharding = RayShardingMode.FIXED
        else:
            n_src = self.data_source.get_n(self.data)
            if W > n_src and self.data_source.needs_partitions:
                raise RuntimeError(f"Trying to shard data for {W} actors, but the maximum number of shards "
                                   f"(i.e. the number of data rows) is {n_src}. Consider using fewer actors.")
            frame = self.data_source.load_data(self.data, ignore=self.ignore, indices=None, **self.kwargs)
            x, y, w, fw, b, ll, lu = self._split(frame)
            n = len(x)
            for v, name in ((y, "label"), (w, "weight"), (ll, "label_lower_bound"), (lu, "label_upper_bound")):
                if v is not None and len(v) != n:
                    raise ValueError(f"`{name}` has {len(v)} rows but the data has {n}")
            self._columns = x.columns
            if self._qid_rows is not None:
                self._load_groups(x.values, {"label": y, "weight": w, "base_margin": b, "label_lower_bound": ll,
                                             "label_upper_bound": lu}, fw, self._qid_rows, W)
                self.loaded = True
                return
            remote = getattr(self, "_transport", "shm") == "remote" and x.values.flags.c_contiguous and n > 0
            if remote:
                allow_actors_to_read_this_process()
                self._keep_alive = x.values            # the actors read these bytes until their upload is done
            for r in range(W):
                sl = _get_sharding_indices(self.sharding, r, W, n)
                ref, shared = {"feature_weights": fw, "qid": None}, {"feature_weights": fw, "qid": None}
                for name, a in (("data", x.values), ("label", y), ("weight", w), ("base_margin", b),
                                ("label_lower_bound", ll), ("label_upper_bound", lu)):
                    if name == "data" and remote:
                        view = a[sl]                  # no copy: a strided / contiguous view of the caller's matrix
                        ref[name] = view
                        inter = None
                        if self.sharding == RayShardingMode.INTERLEAVED and W > 1 and n >= W:
                            inter = (int(a.ctypes.data), n, r, W)
                        shared[name] = ("remote", os.getpid(), int(view.ctypes.data) if len(view) else 0,
                                        int(view.strides[0]) if len(view) else a.shape[1] * 4, len(view), a.shape[1], inter)
                        continue
                    ref[name], shared[name] = _shared_copy(None if a is None else a[sl], "%x_%d_%s" % (self._uid & 0xffffffff, r, name))
                self.refs[r], self._shared[r] = ref, shared
            self.n = n
        self.loaded = True

    def _load_groups(self, xv: np.ndarray, side: Dict[str, Optional[np.ndarray]], fw, q: np.ndarray, W: int):
        """Shards of a ranking matrix: rows sorted stably by qid (merge sort; the reference's pandas sort is not
        stable), then whole query groups per actor.  Every shard is a gathered copy, so it always travels as a /dev/shm
        file; its qid is the shard-local group number (exact in float32)."""
        n = len(xv)
        if len(q) != n:
            raise ValueError(f"`qid` has {len(q)} rows but the data has {n}")
        order = None if n < 2 or not np.any(q[1:] < q[:-1]) else np.argsort(q, kind="mergesort")
        qs = q if order is None else q[order]
        offsets = group_offsets(qs)
        self._row_index = []
        for r in range(W):
            rows = group_sharding_rows(self.sharding, r, W, offsets)     # positions in the qid-sorted order
            src = rows if order is None else order[rows]                 # rows of the caller's arrays
            ref, shared = {"feature_weights": fw}, {"feature_weights": fw}
            tag = "%x_%d_" % (self._uid & 0xffffffff, r)
            ref["data"], shared["data"] = _shared_copy(xv[src], tag + "data")
            for name, a in side.items():
                ref[name], shared[name] = _shared_copy(None if a is None else a[src], tag + name)
            local = group_offsets(qs[rows])
            gid = np.repeat(np.arange(len(local) - 1), np.diff(local)).astype(np.float32)
            ref["qid"], shared["qid"] = _shared_copy(gid, tag + "qid")
            self.refs[r], self._shared[r] = ref, shared
            self._row_index.append(rows)
        self.n = n

    def get_data(self, rank: int, num_actors: Optional[int] = None) -> Dict[str, Optional[np.ndarray]]:
        self.load_data(num_actors=num_actors, rank=rank if (self.distributed and rank not in self.refs) else None)
        if rank not in self.refs:
            self.load_data(num_actors=num_actors, rank=rank)
        return dict(self.refs[rank])

    def get_shared(self, rank: int, num_actors: Optional[int] = None) -> Dict:
        """What the actor of `rank` is sent: /dev/shm descriptors of its shard (arrays when /dev/shm is unusable)."""
        self.get_data(rank, num_actors)
        return dict(self._shared[rank])

    def without_data(self) -> "RayDMatrix":
        """Copy that carries the data SPEC only (file names, column names): what an actor needs to read its own files
        (distributed loading, matrix.py:614-693)."""
        m = copy.copy(self)
        m.refs, m._shared, m.loaded = {}, {}, False
        return m

    def unload_data(self):
        for sh in self._shared.values():
            for v in sh.values():
                if isinstance(v, tuple) and len(v) == 2 and v[0] == "shm":
                    with _SHM_LOCK:
                        _SHM_FILES.discard(v[1])
                    try:
                        os.unlink(v[1])
                    except OSError:
                        pass
        self.refs, self._shared = {}, {}
        self._keep_alive = None
        self.loaded = False

    def __del__(self):
        try:
            self.unload_data()
        except Exception:
            pass

    def update_matrix_properties(self, matrix):
        """numpy sources reset names to f0..fN (data_sources/numpy.py:21-23); frames keep theirs."""
        names = self.feature_names if self.feature_names is not None else self._columns
        try:
            matrix.feature_names = list(names) if names is not None else None
        except Exception:
            pass

    def __hash__(self):
        return self._uid

    def __eq__(self, other):
        return isinstance(other, RayDMatrix) and self.__hash__() == other.__hash__()


class RayQuantileDMatrix(RayDMatrix):
    """Quantised on the device at construction time on the actor (main.py:380-386)."""


class RayDeviceQuantileDMatrix(RayDMatrix):
    """Kept for API compatibility (matrix.py:977-1033); every matrix of this engine is a device
    quantile matrix, so no cupy iterator is involved."""

    def __init__(self, *args, max_bin: int = 256, **kwargs):
        if kwargs.get("qid") is not None:
            raise ValueError("RayDeviceQuantileDMatrix does not support ranking (qid)")
        self.max_bin = max_bin
        super().__init__(*args, **kwargs)


def _detect_distributed(source, data) -> bool:
    """File lists with more than one file are loaded per actor (matrix.py:1063-1085)."""
    if not source.supports_distributed_loading:
        return False
    return isinstance(data, (list, tuple)) and len(data) > 1


def concat_dataframes(dfs: List[Optional[np.ndarray]]):
    filtered = [d for d in dfs if d is not None]
    return np.concatenate(filtered) if filtered else None
