"""scikit-learn estimators on top of train()/predict() -- the surface of xgboost_ray/sklearn.py
(RayXGBRegressor.fit :455-560, RayXGBClassifier.fit :648-791 / predict :798-835 / predict_proba
:839-865), SURVEY.md 8f-4.

The reference subclasses xgboost.sklearn.XGB* (absent here), so these derive from
sklearn.base.BaseEstimator directly and cover the parameters the engine supports.
"""
from typing import Optional

import numpy as np
from sklearn.base import BaseEstimator, ClassifierMixin, RegressorMixin

from xgboost_ray_b200.main import RayParams, predict, train
from xgboost_ray_b200.matrix import RayDMatrix

# estimator attributes forwarded to the engine as training parameters (None = leave the engine default)
_PARAM_NAMES = ("max_depth", "learning_rate", "gamma", "min_child_weight", "reg_lambda", "reg_alpha", "max_bin",
                "base_score", "tree_method", "subsample", "colsample_bytree", "colsample_bylevel", "colsample_bynode",
                "scale_pos_weight", "max_delta_step", "max_cat_to_onehot", "max_cat_threshold", "eval_metric",
                "tweedie_variance_power", "huber_slope", "interaction_constraints", "booster", "rate_drop", "skip_drop",
                "sample_type", "normalize_type", "one_drop", "quantile_alpha", "multi_strategy", "process_type", "updater",
                "refresh_leaf")


def _check_if_params_are_ray_dmatrix(X, sample_weight, base_margin, eval_set):
    """sklearn.py:280-334: X may already be a RayDMatrix, then y & co must be None."""
    train_dmatrix, evals = None, ()
    if isinstance(X, RayDMatrix):
        if sample_weight is not None or base_margin is not None:
            raise ValueError("Cannot pass sample_weight / base_margin together with a RayDMatrix: set them on the matrix.")
        train_dmatrix = X
        if eval_set:
            mats = [e[0] if isinstance(e, tuple) else e for e in eval_set]
            if any(not isinstance(e, RayDMatrix) for e in mats):
                raise ValueError("If X is a RayDMatrix, all elements of `eval_set` must be RayDMatrix as well.")
            evals = tuple((e, "validation_%d" % i) for i, e in enumerate(mats))
    return train_dmatrix, evals


class RayXGBMixin(BaseEstimator):
    def __init__(self, n_estimators: int = 100, max_depth: int = 6, learning_rate: float = 0.3, gamma: float = 0.0,
                 min_child_weight: float = 1.0, reg_lambda: float = 1.0, reg_alpha: float = 0.0, max_bin: int = 256,
                 base_score: Optional[float] = None, tree_method: str = "hist", objective: Optional[str] = None,
                 n_jobs: Optional[int] = None, random_state: Optional[int] = None, subsample: Optional[float] = None,
                 colsample_bytree: Optional[float] = None, colsample_bylevel: Optional[float] = None,
                 colsample_bynode: Optional[float] = None, scale_pos_weight: Optional[float] = None,
                 max_delta_step: Optional[float] = None, max_cat_to_onehot: Optional[int] = None,
                 max_cat_threshold: Optional[int] = None, enable_categorical: bool = False, missing: float = np.nan,
                 eval_metric=None, early_stopping_rounds: Optional[int] = None, callbacks=None,
                 tweedie_variance_power: Optional[float] = None, huber_slope: Optional[float] = None,
                 interaction_constraints=None, booster: Optional[str] = None, rate_drop: Optional[float] = None,
                 skip_drop: Optional[float] = None, sample_type: Optional[str] = None,
                 normalize_type: Optional[str] = None, one_drop: Optional[int] = None, quantile_alpha=None,
                 multi_strategy: Optional[str] = None, process_type: Optional[str] = None,
                 updater: Optional[str] = None, refresh_leaf: Optional[int] = None):
        self.n_estimators = n_estimators
        self.max_depth = max_depth
        self.learning_rate = learning_rate
        self.gamma = gamma
        self.min_child_weight = min_child_weight
        self.reg_lambda = reg_lambda
        self.reg_alpha = reg_alpha
        self.max_bin = max_bin
        self.base_score = base_score          # None: estimated from the labels like xgboost >= 2.0
        self.tree_method = tree_method
        self.objective = objective
        self.n_jobs = n_jobs
        self.random_state = random_state
        self.subsample = subsample
        self.colsample_bytree = colsample_bytree
        self.colsample_bylevel = colsample_bylevel
        self.colsample_bynode = colsample_bynode
        self.scale_pos_weight = scale_pos_weight
        self.max_delta_step = max_delta_step
        self.max_cat_to_onehot = max_cat_to_onehot
        self.max_cat_threshold = max_cat_threshold
        self.enable_categorical = enable_categorical
        self.missing = missing
        self.eval_metric = eval_metric
        self.early_stopping_rounds = early_stopping_rounds
        self.callbacks = callbacks
        self.tweedie_variance_power = tweedie_variance_power   # reg:tweedie rho in [1, 2); None = 1.5
        self.huber_slope = huber_slope                         # reg:pseudohubererror delta > 0; None = 1
        self.interaction_constraints = interaction_constraints   # feature sets, e.g. "[[0, 1], [2, 3, 4]]"; None = off
        self.booster = booster                 # "gbtree" (None) or "dart"; the next five are DART's, ignored by gbtree
        self.rate_drop = rate_drop
        self.skip_drop = skip_drop
        self.sample_type = sample_type
        self.normalize_type = normalize_type
        self.one_drop = one_drop
        self.quantile_alpha = quantile_alpha   # reg:quantileerror alphas, e.g. [0.05, 0.5, 0.95]; None = 0.5
        self.multi_strategy = multi_strategy   # 2-D y: "one_output_per_tree" (None) or "multi_output_tree" (vector leaves)
        # "update" with updater="refresh": fit(xgb_model=...) refreshes that model's trees on X (refresh_leaf: new leaves)
        self.process_type = process_type
        self.updater = updater
        self.refresh_leaf = refresh_leaf

    def get_xgb_params(self):
        p = {k: getattr(self, k) for k in _PARAM_NAMES if getattr(self, k) is not None}
        p["objective"] = self.objective
        if self.random_state is not None:
            p["seed"] = int(self.random_state)
        return p

    def get_num_boosting_rounds(self):
        return self.n_estimators

    def _ray_params(self, ray_params):
        if ray_params is None:
            return RayParams(num_actors=self.n_jobs if self.n_jobs and self.n_jobs > 0 else 1)
        return ray_params

    def get_booster(self):
        if not hasattr(self, "_Booster"):
            raise RuntimeError("need to call fit or load_model beforehand")
        return self._Booster

    def _fit(self, params, X, y, sample_weight, base_margin, eval_set, ray_params, ray_dmatrix_params, **kw):
        ray_dmatrix_params = dict(ray_dmatrix_params or {})
        if self.enable_categorical:
            ray_dmatrix_params.setdefault("enable_categorical", True)
        if not (isinstance(self.missing, float) and np.isnan(self.missing)):
            ray_dmatrix_params.setdefault("missing", self.missing)
        if self.early_stopping_rounds is not None:
            kw.setdefault("early_stopping_rounds", self.early_stopping_rounds)
        if self.callbacks is not None:
            kw.setdefault("callbacks", self.callbacks)
        train_dmatrix, evals = _check_if_params_are_ray_dmatrix(X, sample_weight, base_margin, eval_set)
        if train_dmatrix is None:
            train_dmatrix = RayDMatrix(X, y, weight=sample_weight, base_margin=base_margin, **ray_dmatrix_params)
            evals = tuple((RayDMatrix(ex, ey, **ray_dmatrix_params), "validation_%d" % i)
                          for i, (ex, ey) in enumerate(eval_set or ()))
        self.evals_result_ = {}
        self.additional_results_ = {}
        self._Booster = train(params, train_dmatrix, self.get_num_boosting_rounds(), evals=evals, evals_result=self.evals_result_,
                              additional_results=self.additional_results_, ray_params=self._ray_params(ray_params), **kw)
        self.n_features_in_ = self._Booster.n_features
        self.best_iteration = getattr(self._Booster, "best_iteration", None)
        self.best_score = getattr(self._Booster, "best_score", None)
        return self

    def evals_result(self):
        return self.evals_result_

    @property
    def feature_importances_(self):
        """Normalised average gain per feature (importance_type "gain", xgboost's default for tree boosters)."""
        b = self.get_booster()
        score = b.get_score(importance_type="gain")
        out = np.zeros(self.n_features_in_, np.float32)
        names = getattr(b, "feature_names", None)
        for k, v in score.items():
            idx = names.index(k) if names and k in names else int(k[1:])
            out[idx] = v
        tot = out.sum()
        return out / tot if tot > 0 else out

    def save_model(self, fname):
        self.get_booster().save_model(fname)

    def load_model(self, fname):
        from xgboost_ray_b200.xgb import xgboost as _x
        self._Booster = _x.Booster(model_file=fname)
        self.n_features_in_ = self._Booster.n_features
        return self

    def _predict(self, X, ray_params, ray_dmatrix_params, **kw):
        ray_dmatrix_params = dict(ray_dmatrix_params or {})
        if not (isinstance(self.missing, float) and np.isnan(self.missing)):   # the sentinel the model was fitted with
            ray_dmatrix_params.setdefault("missing", self.missing)
        data = X if isinstance(X, RayDMatrix) else RayDMatrix(X, **ray_dmatrix_params)
        return predict(self.get_booster(), data, ray_params=self._ray_params(ray_params), **kw)

    def apply(self, X, iteration_range=None, ray_params=None, ray_dmatrix_params=None):
        """Leaf index of every row in every tree, float32 (n, trees) -- xgboost's XGBModel.apply (pred_leaf=True)."""
        return self._predict(X, ray_params, ray_dmatrix_params, pred_leaf=True, iteration_range=iteration_range or (0, 0))


class RayXGBRegressor(RayXGBMixin, RegressorMixin):
    def fit(self, X, y=None, *, sample_weight=None, base_margin=None, eval_set=None, ray_params=None,
            ray_dmatrix_params=None, **kw):
        params = self.get_xgb_params()
        params["objective"] = params["objective"] or "reg:squarederror"
        return self._fit(params, X, y, sample_weight, base_margin, eval_set, ray_params, ray_dmatrix_params, **kw)

    def predict(self, X, output_margin=False, ray_params=None, ray_dmatrix_params=None, **kw):
        return self._predict(X, ray_params, ray_dmatrix_params, output_margin=output_margin, **kw)


class RayXGBClassifier(RayXGBMixin, ClassifierMixin):
    def fit(self, X, y=None, *, sample_weight=None, base_margin=None, eval_set=None, ray_params=None,
            ray_dmatrix_params=None, **kw):
        params = self.get_xgb_params()
        if isinstance(X, RayDMatrix):
            n_classes = getattr(self, "n_classes_", None) or kw.pop("num_class", None)
            if n_classes is None:
                raise ValueError("When X is a RayDMatrix, set `n_classes_` (or pass num_class=) before fit().")
            self.classes_ = np.arange(n_classes)
            yy = None
        elif np.ndim(y) == 2 and np.shape(y)[1] > 1:
            # multi-label classification (xgboost 2.x): a 0/1 label matrix, binary:logistic with one target per column
            yy = np.asarray(y.values if hasattr(y, "values") and not isinstance(y, np.ndarray) else y, np.float32)
            if not np.all((yy == 0) | (yy == 1)):
                raise ValueError("a 2-D label is multi-label classification: every label must be 0 or 1")
            self.classes_ = np.array([0, 1])
            self.n_classes_ = 2
            self._multi_label = True
            params["objective"] = params["objective"] or "binary:logistic"
            return self._fit(params, X, yy, sample_weight, base_margin, eval_set, ray_params, ray_dmatrix_params, **kw)
        else:
            self.classes_ = np.unique(np.asarray(y))
            lookup = {c: i for i, c in enumerate(self.classes_)}
            yy = np.asarray([lookup[v] for v in np.asarray(y)], np.float32)
        self.n_classes_ = len(self.classes_)
        self._multi_label = False
        if self.n_classes_ > 2:
            params["objective"] = "multi:softprob"
            params["num_class"] = self.n_classes_
        else:
            params["objective"] = params["objective"] or "binary:logistic"
        return self._fit(params, X, yy, sample_weight, base_margin, eval_set, ray_params, ray_dmatrix_params, **kw)

    def predict_proba(self, X, ray_params=None, ray_dmatrix_params=None, **kw):
        p = self._predict(X, ray_params, ray_dmatrix_params, **kw)
        if getattr(self, "_multi_label", False):   # (n, T): the probability of label 1 in each column
            return p
        if p.ndim == 1:
            return np.vstack((1.0 - p, p)).T
        return p

    def predict(self, X, output_margin=False, ray_params=None, ray_dmatrix_params=None, **kw):
        if output_margin:
            return self._predict(X, ray_params, ray_dmatrix_params, output_margin=True, **kw)
        proba = self.predict_proba(X, ray_params, ray_dmatrix_params, **kw)
        if getattr(self, "_multi_label", False):
            return (proba > 0.5).astype(np.int64)
        return self.classes_[np.argmax(proba, axis=1)]


class _Unsupported:
    _why = ""

    def __init__(self, *a, **k):
        raise NotImplementedError(self._why)


_RF_DEFAULTS = {"learning_rate": 1.0, "subsample": 0.8, "colsample_bynode": 0.8, "reg_lambda": 1e-5}


def _rf_init(base):
    """__init__ with the explicit parameter list of `base` (scikit-learn reads it for get_params / clone) and the
    defaults of xgboost's XGBRF* estimators (xgboost_ray/sklearn.py:611-628)."""
    import inspect
    sig = inspect.signature(base.__init__)
    new_sig = sig.replace(parameters=[p.replace(default=_RF_DEFAULTS.get(n, p.default)) for n, p in sig.parameters.items()])

    def __init__(self, *args, **kwargs):
        bound = new_sig.bind(self, *args, **kwargs)
        bound.apply_defaults()
        base.__init__(*bound.args, **bound.kwargs)

    __init__.__signature__ = new_sig
    return __init__


class _RandomForestMixin:
    """xgboost_ray/sklearn.py:602-637, 880-914: ONE boosting round that grows n_estimators trees in parallel
    (num_parallel_tree) on row / column samples of the same gradients, leaf values averaged."""

    def get_xgb_params(self):
        params = super().get_xgb_params()
        params["num_parallel_tree"] = self.n_estimators
        return params

    def get_num_boosting_rounds(self):
        return 1


class RayXGBRFRegressor(_RandomForestMixin, RayXGBRegressor):
    __init__ = _rf_init(RayXGBRegressor)


class RayXGBRFClassifier(_RandomForestMixin, RayXGBClassifier):
    __init__ = _rf_init(RayXGBClassifier)


class RayXGBRanker(_Unsupported):
    """xgboost_ray/sklearn.py:868-1083: ranking objectives (qid groups) are outside the hot path (DESIGN.md 7)."""
    _why = "ranking objectives (rank:pairwise / rank:ndcg, qid groups) are not implemented by the H100 hist engine"
