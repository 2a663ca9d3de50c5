"""Multi-target regression and multi-label classification (a label of T > 1 columns) on top of the oracle.

What the engine implements (csrc/objective_kernel.cu gradient_multi_target_kernel / metric_multi_target_kernel,
csrc/round.cu estimate_base_score; DESIGN.md 2 item 18), written out per column so that the GPU tests can replay a
trained model round by round:
  * the gradients of column k are the single-target binary32 sequence of tests/objective_reference.py on margin[:, k] and
    label[:, k], with the row's weight (scale_pos_weight applies per element where y == 1);
  * round r grows T trees, tree k from column k's gradients, laid out like multi-class trees (tree r*T + k);
  * the intercept (base_score=None) is transform(sum_k fp32(stump_k / T)), the sum in binary32 in k order, stump_k the
    fixed-point Newton stump of column k at margin 0;
  * the elementwise metrics count every (row, column) element with its row's weight: sum w_i v_ik / (T sum w_i).
The oracle grows the trees through its custom-gradient path with num_class = T; nothing of it changes."""
import numpy as np

from tests import objective_reference as O

F32 = np.float32
# objectives that take a label of several columns (xgboost's RegLossObj family and pseudo-Huber)
MULTI_TARGET_OBJECTIVES = ("reg:squarederror", "reg:squaredlogerror", "reg:logistic", "binary:logistic",
                           "binary:logitraw", "reg:pseudohubererror")


def column_gradients(params, margin, label, weight=None):
    """(g, h, non-finite count) [n][T] in binary32: the single-target sequence of every column."""
    g, h, bad = O.gradients_multi_target(params, margin, label, weight)
    return g.T.copy(), h.T.copy(), bad


def intercept(params, label, weight=None):
    """base_score when none is given: transform(sum_k fp32(stump_k / T)) in binary32, k in order."""
    from tests.fixed_sums_reference import node_sums, quant_exponent
    y = np.asarray(label, F32)
    T = y.shape[1]
    g, h, _ = column_gradients(params, np.zeros_like(y), y, weight)
    s = None
    for k in range(T):
        G, H = node_sums(g[:, k], h[:, k], quant_exponent(g[:, k]), quant_exponent(h[:, k]))
        stump = F32(0.0) if H <= 1e-6 else F32(-G / H)
        term = F32(stump / F32(T))
        s = term if s is None else F32(s + term)
    obj = params["objective"]
    if obj in ("binary:logistic", "reg:logistic"):
        return float(O.sigmoid_(np.array([s], F32))[0])
    return float(s)


def metric(name, obj, margin, label, weight=None, params=None):
    """Elementwise metric over the n x T elements in float64, each with its row's weight."""
    y = np.asarray(label, F32)
    n, T = y.shape
    w = None if weight is None else np.repeat(np.asarray(weight, F32), T)
    o = "binary:logistic" if obj == "binary:logistic" else obj
    if name == "error":
        p = O.sigmoid_(np.asarray(margin, F32).reshape(-1)) if obj in ("binary:logistic", "reg:logistic") \
            else np.asarray(margin, F32).reshape(-1)
        v = ((p > F32(0.5)) != (y.reshape(-1) > F32(0.5))).astype(np.float64)
        ww = np.ones(n * T) if w is None else w.astype(np.float64)
        return float(np.sum(v * ww) / np.sum(ww))
    if name == "logloss" and obj == "binary:logistic":
        o = "reg:logistic"   # the same sigmoid; objective_reference keys its transform by reg:logistic
    return O.metric(name, o, np.asarray(margin, F32).reshape(-1), y.reshape(-1), w, params)


def base_margin_of(obj, b):
    return O.base_margin("reg:logistic" if obj == "binary:logistic" else obj, b)


class Model:
    """Trees in the engine's order (tree r*T + k), the margins [n][T] they give on the train rows, the intercept."""

    def __init__(self, bst, margin, base_score):
        self.bst, self.margin, self.base_score = bst, margin, base_score

    @property
    def num_trees(self):
        return self.bst.num_trees

    def tree(self, i):
        return self.bst.tree(i)

    def predict_margin(self, X):
        return self.bst.predict_margin(X)


def train(oracle, params, X, Y, rounds, weight=None, is_cat=None, base_margin=None):
    """`rounds` rounds of T trees grown by the oracle from the per-column gradients (custom-gradient path)."""
    obj = params["objective"]
    X = np.ascontiguousarray(X, F32)
    Y = np.ascontiguousarray(Y, F32)
    n, T = Y.shape
    for k in range(T):
        O.check_labels(obj, Y[:, k])
    b = params.get("base_score")
    b = intercept(params, Y, weight) if b is None else float(F32(b))
    m0 = base_margin_of(obj, b)
    op = {k: v for k, v in params.items() if k not in ("objective", "base_score", "eval_metric", "scale_pos_weight",
                                                       "huber_slope")}
    op.update(objective="multi:softprob", num_class=T, base_score=float(m0))
    cuts = oracle.Cuts.from_data(X, int(params.get("max_bin", 256)), np.nan, is_cat=is_cat, weight=weight)
    bins = cuts.bin(X)
    bst = oracle.Booster(op, cuts)
    if base_margin is not None:
        margin = np.array(np.asarray(base_margin, F32).reshape(n, T), F32)
    else:
        margin = np.full((n, T), m0, F32)
    bst.init_margin(n, margin)
    for _ in range(rounds):
        g, h, bad = column_gradients(params, bst.margin, Y, weight)
        if bad:
            raise FloatingPointError("%s: a gradient or hessian is not finite" % obj)
        bst.boost(bins, Y[:, 0], weight, custom_g=g.reshape(-1), custom_h=h.reshape(-1))
    return Model(bst, bst.margin, b)
