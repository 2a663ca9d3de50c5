"""ctypes wrapper around oracle/liboracle.so (hist_oracle.c).

TEST INFRASTRUCTURE ONLY -- see the header of hist_oracle.c.  Only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
The product package (xgboost_ray_b200/) never does.

PARITY UNPINNED: restatement of XGBoost 2.x `tree_method="hist"` (SURVEY.md Appendix A);
the reference (xgboost_ray/main.py:745-752) delegates this arithmetic to the absent
`xgboost` wheel and holds no golden vectors for it.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")

OBJECTIVES = {"reg:squarederror": 0, "reg:linear": 0, "binary:logistic": 1,
              "multi:softprob": 2, "multi:softmax": 2}
METRICS = {"rmse": 0, "logloss": 1, "error": 2, "mlogloss": 3, "merror": 4, "mae": 5}


class OrParams(C.Structure):
    _fields_ = [("objective", C.c_int32), ("num_class", C.c_int32), ("max_depth", C.c_int32),
                ("max_bin", C.c_int32), ("eta", C.c_float), ("gamma", C.c_float),
                ("min_child_weight", C.c_float), ("lambda_", C.c_float), ("alpha", C.c_float),
                ("base_score", C.c_float), ("qbits", C.c_int32), ("nthread", C.c_int32),
                ("max_cat_to_onehot", C.c_int32), ("max_cat_threshold", C.c_int32),
                ("scale_pos_weight", C.c_float), ("max_delta_step", C.c_float), ("subsample", C.c_float),
                ("colsample_bytree", C.c_float), ("colsample_bylevel", C.c_float), ("colsample_bynode", C.c_float),
                ("seed", C.c_int32), ("rank", C.c_int32)]


def build(force=False):
    """Compile liboracle.so with the committed Makefile (gcc)."""
    src = os.path.join(_HERE, "hist_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        fp, ip, bp, dp = (C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint8),
                          C.POINTER(C.c_double))
        L.or_cuts_create.restype = C.c_void_p
        L.or_cuts_create.argtypes = [fp, C.c_int64, C.c_int32, C.c_float, C.c_int32]
        L.or_cuts_create_cat.restype = C.c_void_p
        L.or_cuts_create_cat.argtypes = [fp, C.c_int64, C.c_int32, C.c_float, C.c_int32, bp]
        L.or_cuts_create_w.restype = C.c_void_p
        L.or_cuts_create_w.argtypes = [fp, C.c_int64, C.c_int32, C.c_float, C.c_int32, bp, fp]
        L.or_cuts_set_cat.argtypes = [C.c_void_p, bp]
        L.or_cuts_get_cat.argtypes = [C.c_void_p, bp]
        L.or_tree_get_cat.argtypes = [C.c_void_p, C.c_int32, bp, C.POINTER(C.c_uint32)]
        L.or_cuts_from_arrays.restype = C.c_void_p
        L.or_cuts_from_arrays.argtypes = [C.c_int32, C.c_int32, ip, fp, fp, bp]
        L.or_cuts_free.argtypes = [C.c_void_p]
        L.or_cuts_total.restype = C.c_int32
        L.or_cuts_total.argtypes = [C.c_void_p]
        L.or_cuts_get.argtypes = [C.c_void_p, ip, fp, fp, bp]
        L.or_bin_matrix.argtypes = [C.c_void_p, fp, C.c_int64, C.c_float, bp]
        L.or_gradients.argtypes = [C.c_int32, C.c_int32, fp, fp, fp, C.c_int64, fp, fp]
        L.or_quantize.argtypes = [fp, C.c_int64, C.c_int64, C.c_int32, ip, ip]
        L.or_hist_int.argtypes = [bp, C.c_int32, ip, ip, ip, C.c_int64, C.POINTER(C.c_int64)]
        L.or_model_new.restype = C.c_void_p
        L.or_model_new.argtypes = [C.POINTER(OrParams), C.c_int32]
        L.or_model_free.argtypes = [C.c_void_p]
        L.or_estimate_base_score.restype = C.c_float
        L.or_estimate_base_score.argtypes = [C.c_void_p, fp, fp, C.c_int64]
        L.or_model_set_feature_weights.restype = C.c_int
        L.or_model_set_feature_weights.argtypes = [C.c_void_p, fp, C.c_int32]
        L.or_base_margin.restype = C.c_float
        L.or_base_margin.argtypes = [C.POINTER(OrParams)]
        L.or_boost_one_round.restype = C.c_int
        L.or_boost_one_round.argtypes = [C.c_void_p, C.c_void_p, bp, C.c_int64, fp, fp, fp, fp, fp]
        L.or_num_trees.restype = C.c_int32
        L.or_num_trees.argtypes = [C.c_void_p]
        L.or_tree_num_nodes.restype = C.c_int32
        L.or_tree_num_nodes.argtypes = [C.c_void_p, C.c_int32]
        L.or_tree_get.argtypes = [C.c_void_p, C.c_int32, ip, ip, ip, ip, ip, fp, bp, fp, fp, fp, dp]
        L.or_predict_margin.argtypes = [C.c_void_p, fp, C.c_int64, C.c_float, C.c_int32, C.c_int32, fp, fp]
        L.or_transform.argtypes = [C.c_int32, C.c_int32, fp, C.c_int64]
        L.or_metric_sums.argtypes = [C.c_int32, C.c_int32, fp, fp, fp, C.c_int64, dp, dp]
        L.or_metric_sums_obj.argtypes = [C.c_int32, C.c_int32, C.c_int32, fp, fp, fp, C.c_int64, dp, dp]
        L.or_expf.restype = C.c_float
        L.or_expf.argtypes = [C.c_float]
        L.or_num_threads.restype = C.c_int32
        L.or_set_num_threads.argtypes = [C.c_int32]
        _lib = L
    return _lib


def use_all_cores(calibrate=True):
    """Pick the OpenMP thread count for the CPU baseline legs.  torchrun exports OMP_NUM_THREADS=1, and on
    shared hosts asking for every logical CPU can be far slower than a smaller team (oversubscribed
    cores and memory bandwidth), so the candidates
    {all, 64, 32, 16} are timed on a small synthetic round and the fastest is used.  Returns the count."""
    n_all = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    L = lib()
    cands = sorted({c for c in (n_all, 64, 32, 16) if 1 <= c <= n_all} | {min(n_all, 8)}, reverse=True)
    if not calibrate or len(cands) == 1:
        L.or_set_num_threads(n_all)
        return L.or_num_threads()
    rng = np.random.RandomState(0)
    n, f = 400_000, 32
    X = rng.uniform(0, 10, size=(n, f)).astype(np.float32)
    y = (X[:, 0] + X[:, 1]).astype(np.float32)
    L.or_set_num_threads(min(n_all, 16))
    cuts = Cuts.from_data(X, 256)
    bins = cuts.bin(X)
    best, best_t = cands[-1], float("inf")
    import time
    for c in cands:
        L.or_set_num_threads(c)
        b = Booster({"objective": "reg:squarederror", "max_depth": 6, "hist_qbits": 0}, cuts)
        b.init_margin(n)
        b.boost(bins, y)
        t0 = time.perf_counter()
        b.boost(bins, y)
        dt = time.perf_counter() - t0
        if dt < best_t * 0.95:      # prefer the larger team unless a smaller one is clearly faster
            best, best_t = c, min(dt, best_t)
    L.or_set_num_threads(best)
    return L.or_num_threads()


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float)) if a is not None else None


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32)) if a is not None else None


def _bp(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint8)) if a is not None else None


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


class Cuts:
    """Per-feature cut points (A.2).  ptrs[F+1], vals[total], mins[F], has_missing[F]."""

    def __init__(self, handle, n_features, max_bin):
        self.h = handle
        self.n_features = n_features
        self.max_bin = max_bin
        L = lib()
        tot = L.or_cuts_total(handle)
        self.ptrs = np.zeros(n_features + 1, np.int32)
        self.vals = np.zeros(max(tot, 1), np.float32)
        self.mins = np.zeros(n_features, np.float32)
        self.has_missing = np.zeros(n_features, np.uint8)
        L.or_cuts_get(handle, _ip(self.ptrs), _fp(self.vals), _fp(self.mins), _bp(self.has_missing))
        self.vals = self.vals[:tot]
        self.is_cat = np.zeros(n_features, np.uint8)
        L.or_cuts_get_cat(handle, _bp(self.is_cat))

    @classmethod
    def from_data(cls, X, max_bin=256, missing=np.nan, is_cat=None, weight=None):
        """is_cat: optional bool/uint8 [F]; categorical features get the cuts 0..max code (bin = code).
        weight: optional sample weights [n] -> weighted quantile sketch."""
        X = _f32(X)
        n, f = X.shape
        ic = None if is_cat is None else np.ascontiguousarray(is_cat, np.uint8)
        w = _f32(weight)
        h = lib().or_cuts_create_w(_fp(X), n, f, float(missing), max_bin, _bp(ic), _fp(w))
        if not h:
            raise ValueError("or_cuts_create failed (max_bin must be in [2,256]; category codes must be integers "
                             "in [0,255], [0,254] for a feature with missing values)")
        return cls(h, f, max_bin)

    @classmethod
    def from_arrays(cls, ptrs, vals, mins, has_missing, max_bin=256, is_cat=None):
        ptrs = np.ascontiguousarray(ptrs, np.int32)
        vals = _f32(vals)
        mins = _f32(mins)
        hm = np.ascontiguousarray(has_missing, np.uint8)
        f = len(ptrs) - 1
        h = lib().or_cuts_from_arrays(f, max_bin, _ip(ptrs), _fp(vals), _fp(mins), _bp(hm))
        if is_cat is not None:
            lib().or_cuts_set_cat(h, _bp(np.ascontiguousarray(is_cat, np.uint8)))
        return cls(h, f, max_bin)

    def borrowed_by(self, X, missing=np.nan):
        """The cuts a matrix X trains with when it borrows these ones (DESIGN.md §2 item 6): a categorical feature
        that has missing values in X is marked has_missing, so that its bin 255 is routed by the default direction
        (as prediction routes a missing value) rather than as an unknown category.  Numeric features keep theirs."""
        X = _f32(X)
        miss = np.isnan(X) if np.isnan(missing) else (np.isnan(X) | (X == np.float32(missing)))
        hm = self.has_missing | (self.is_cat.astype(bool) & miss.any(axis=0)).astype(np.uint8)
        if np.array_equal(hm, self.has_missing):
            return self
        return Cuts.from_arrays(self.ptrs, self.vals, self.mins, hm, self.max_bin, is_cat=self.is_cat)

    def bin(self, X, missing=np.nan):
        X = _f32(X)
        n, f = X.shape
        assert f == self.n_features
        out = np.zeros((n, f), np.uint8)
        lib().or_bin_matrix(self.h, _fp(X), n, float(missing), _bp(out))
        return out

    def __del__(self):
        try:
            lib().or_cuts_free(self.h)
        except Exception:
            pass


def make_params(params):
    """dict of xgboost-style params -> OrParams (A.1 defaults)."""
    p = OrParams()
    obj = params.get("objective", "reg:squarederror")
    p.objective = OBJECTIVES[obj]
    p.num_class = int(params.get("num_class", 1)) if p.objective == 2 else 1
    p.max_depth = int(params.get("max_depth", 6))
    p.max_bin = int(params.get("max_bin", 256))
    p.eta = float(params.get("eta", params.get("learning_rate", 0.3)))
    p.gamma = float(params.get("gamma", params.get("min_split_loss", 0.0)))
    p.min_child_weight = float(params.get("min_child_weight", 1.0))
    p.lambda_ = float(params.get("lambda", params.get("reg_lambda", 1.0)))
    p.alpha = float(params.get("alpha", params.get("reg_alpha", 0.0)))
    p.base_score = float(params.get("base_score", 0.5))
    p.qbits = int(params.get("hist_qbits", 18))
    p.nthread = int(params.get("nthread", 0))
    p.max_cat_to_onehot = int(params.get("max_cat_to_onehot", 4))
    p.max_cat_threshold = int(params.get("max_cat_threshold", 64))
    p.scale_pos_weight = float(params.get("scale_pos_weight", 1.0))
    p.max_delta_step = float(params.get("max_delta_step", 0.0))
    p.subsample = float(params.get("subsample", 1.0))
    p.colsample_bytree = float(params.get("colsample_bytree", 1.0))
    p.colsample_bylevel = float(params.get("colsample_bylevel", 1.0))
    p.colsample_bynode = float(params.get("colsample_bynode", 1.0))
    p.seed = int(params.get("seed", params.get("random_state", 0)) or 0)
    p.rank = int(params.get("_rank", 0))
    return p


class Tree:
    FIELDS = ("left", "right", "parent", "split_feature", "split_bin", "split_cond", "default_left",
              "value", "base_weight", "loss_chg", "sum_hess", "split_type", "cat_bits")

    def categories(self, nid):
        """Sorted category codes that go RIGHT at categorical node nid."""
        w = self.cat_bits[nid]
        return [b for b in range(256) if (int(w[b >> 5]) >> (b & 31)) & 1]

    def __init__(self, **kw):
        for k in self.FIELDS:
            setattr(self, k, kw[k])

    @property
    def n_nodes(self):
        return len(self.left)


class Booster:
    """Oracle booster: grows trees on a binned matrix, keeps the margin cache of the train set."""

    def __init__(self, params, cuts):
        self.params = dict(params)
        self.p = make_params(params)
        self.cuts = cuts
        self.h = lib().or_model_new(C.byref(self.p), cuts.n_features)
        self.K = self.p.num_class
        self.margin = None

    def estimate_base_score(self, label, weight=None):
        """xgboost >= 2.0 default when no base_score is given (A.3); updates the model and self.p."""
        label = _f32(label)
        v = float(lib().or_estimate_base_score(self.h, _fp(label), _fp(_f32(weight)), len(label)))
        self.p.base_score = v
        self.params["base_score"] = v
        return v

    def set_feature_weights(self, fw):
        fw = _f32(fw)
        if lib().or_model_set_feature_weights(self.h, _fp(fw), len(fw)) != 0:
            raise ValueError("feature_weights must have one finite non-negative value per feature")

    def base_margin_value(self):
        return float(lib().or_base_margin(C.byref(self.p)))

    def init_margin(self, n, base_margin=None):
        if base_margin is not None:
            self.margin = _f32(np.asarray(base_margin).reshape(n, -1)).copy()
            if self.margin.shape[1] != self.K:
                self.margin = np.repeat(self.margin, self.K, axis=1)
        else:
            self.margin = np.full((n, self.K), self.base_margin_value(), np.float32)
        return self.margin

    def boost(self, bins, label, weight=None, custom_g=None, custom_h=None):
        bins = np.ascontiguousarray(bins, np.uint8)
        n = bins.shape[0]
        if self.margin is None:
            self.init_margin(n)
        label = _f32(label)
        weight = _f32(weight)
        cg, ch = _f32(custom_g), _f32(custom_h)
        rc = lib().or_boost_one_round(self.h, self.cuts.h, _bp(bins), n, _fp(label), _fp(weight),
                                      _fp(self.margin), _fp(cg), _fp(ch))
        assert rc == 0

    @property
    def num_trees(self):
        return lib().or_num_trees(self.h)

    def tree(self, i):
        L = lib()
        nn = L.or_tree_num_nodes(self.h, i)
        a = dict(left=np.zeros(nn, np.int32), right=np.zeros(nn, np.int32), parent=np.zeros(nn, np.int32),
                 split_feature=np.zeros(nn, np.int32), split_bin=np.zeros(nn, np.int32),
                 split_cond=np.zeros(nn, np.float32), default_left=np.zeros(nn, np.uint8),
                 value=np.zeros(nn, np.float32), base_weight=np.zeros(nn, np.float32),
                 loss_chg=np.zeros(nn, np.float32), sum_hess=np.zeros(nn, np.float64),
                 split_type=np.zeros(nn, np.uint8), cat_bits=np.zeros((nn, 8), np.uint32))
        L.or_tree_get(self.h, i, _ip(a["left"]), _ip(a["right"]), _ip(a["parent"]), _ip(a["split_feature"]),
                      _ip(a["split_bin"]), _fp(a["split_cond"]), _bp(a["default_left"]), _fp(a["value"]),
                      _fp(a["base_weight"]), _fp(a["loss_chg"]),
                      a["sum_hess"].ctypes.data_as(C.POINTER(C.c_double)))
        L.or_tree_get_cat(self.h, i, _bp(a["split_type"]), a["cat_bits"].ctypes.data_as(C.POINTER(C.c_uint32)))
        return Tree(**a)

    def trees(self):
        return [self.tree(i) for i in range(self.num_trees)]

    def predict_margin(self, X, missing=np.nan, tree_begin=0, tree_end=0, base_margin=None):
        X = _f32(X)
        n = X.shape[0]
        out = np.zeros((n, self.K), np.float32)
        bm = None
        if base_margin is not None:
            bm = _f32(np.asarray(base_margin).reshape(n, -1))
            if bm.shape[1] != self.K:
                bm = np.ascontiguousarray(np.repeat(bm, self.K, axis=1))
        lib().or_predict_margin(self.h, _fp(X), n, float(missing), tree_begin, tree_end, _fp(bm), _fp(out))
        return out

    def predict(self, X, missing=np.nan, output_margin=False, base_margin=None):
        m = self.predict_margin(X, missing, base_margin=base_margin)
        if not output_margin:
            lib().or_transform(self.p.objective, self.K, _fp(m), m.shape[0])
        if self.K == 1:
            return m[:, 0]
        if self.params.get("objective") == "multi:softmax" and not output_margin:
            return np.argmax(m, axis=1).astype(np.float32)
        return m

    def metric(self, name, margin, label, weight=None):
        margin = _f32(margin)
        s, ws = C.c_double(), C.c_double()
        lib().or_metric_sums_obj(self.p.objective, METRICS[name], self.K, _fp(margin), _fp(_f32(label)),
                                 _fp(_f32(weight)), margin.shape[0], C.byref(s), C.byref(ws))
        v = s.value / ws.value if ws.value > 0 else 0.0
        return float(np.sqrt(v)) if name == "rmse" else v

    def __del__(self):
        try:
            lib().or_model_free(self.h)
        except Exception:
            pass


def train(params, X, y, num_boost_round, weight=None, missing=np.nan, cuts=None, base_margin=None, is_cat=None,
          feature_weights=None):
    """Convenience: cuts -> bins -> rounds.  Returns (Booster, bins).  `cuts` are borrowed (Cuts.borrowed_by)."""
    X = _f32(X)
    if cuts is not None:
        cuts = cuts.borrowed_by(X, missing)
    else:
        cuts = Cuts.from_data(X, int(params.get("max_bin", 256)), missing, is_cat=is_cat, weight=weight)
    bins = cuts.bin(X, missing)
    bst = Booster(params, cuts)
    if feature_weights is not None:
        bst.set_feature_weights(feature_weights)
    if params.get("base_score") is None:
        bst.estimate_base_score(y, weight)
    bst.init_margin(X.shape[0], base_margin)
    for _ in range(num_boost_round):
        bst.boost(bins, y, weight)
    return bst, bins


def hist_int(bins, qg, qh, ridx=None):
    bins = np.ascontiguousarray(bins, np.uint8)
    n, f = bins.shape
    out = np.zeros((f, 256, 2), np.int64)
    ri = None if ridx is None else np.ascontiguousarray(ridx, np.int32)
    nrows = n if ri is None else len(ri)
    lib().or_hist_int(_bp(bins), f, _ip(np.ascontiguousarray(qg, np.int32)),
                      _ip(np.ascontiguousarray(qh, np.int32)), _ip(ri), nrows,
                      out.ctypes.data_as(C.POINTER(C.c_int64)))
    return out


def quantize(v, qbits):
    v = _f32(v)
    q = np.zeros(len(v), np.int32)
    e = C.c_int32()
    lib().or_quantize(_fp(v), len(v), 1, qbits, _ip(q), C.byref(e))
    return q, e.value


def gradients(objective, margin, label, weight=None, num_class=1):
    margin = _f32(margin)
    n = margin.shape[0]
    g = np.zeros(margin.size, np.float32)
    h = np.zeros(margin.size, np.float32)
    lib().or_gradients(OBJECTIVES[objective], num_class, _fp(margin), _fp(_f32(label)), _fp(_f32(weight)),
                       n, _fp(g), _fp(h))
    return g, h
