"""float64 NumPy restatement of the `auc` / `aucpr` rules (DESIGN.md §2 item 17), binary and one-vs-rest, with the
combination over the workers.  Written from the rules, not from the engine's code.

    value(metric, pred, label, weight=None, shards=None)

pred is (n,) for a single-output model or (n, K) probabilities of a K-class model; shards is a list of row selections,
one per worker (default: one worker with every row).  The value is what B2_BoosterEvalSet returns."""
import numpy as np


def tie_group_ends(pred, y, w):
    """Cumulative (tp, fp) at the end of each tie group, rows in descending prediction order, with (0, 0) in front."""
    pred = np.asarray(pred, np.float64)
    y = np.asarray(y, np.float64)
    w = np.ones_like(y) if w is None else np.asarray(w, np.float64)
    order = np.argsort(-pred, kind="stable")
    p, y, w = pred[order], y[order], w[order]
    tp, fp = np.cumsum(y * w), np.cumsum((1.0 - y) * w)
    ends = np.nonzero(np.append(p[1:] != p[:-1], True))[0] if len(p) else np.zeros(0, np.int64)
    return np.concatenate([[0.0], tp[ends]]), np.concatenate([[0.0], fp[ends]])


def pr_segment(tp0, fp0, tp1, fp1, P):
    """Area under the Davis & Goadrich interpolation of precision over recall between (tp0, fp0) and (tp1, fp1),
    elementwise over arrays of segments."""
    tp0, fp0, tp1, fp1 = (np.asarray(v, np.float64) for v in (tp0, fp0, tp1, fp1))
    dtp = tp1 - tp0
    h = np.divide(fp1 - fp0, dtp, out=np.zeros_like(dtp), where=dtp != 0)   # h = 0 when tp1 = tp0
    a = 1.0 + h
    b = (fp0 - h * tp0) / P
    t0, t1 = tp0 / P, tp1 / P
    with np.errstate(divide="ignore", invalid="ignore"):
        log_term = np.where(b == 0.0, 0.0, (b / a ** 2) * (np.log(a * t1 + b) - np.log(a * t0 + b)))
    return (t1 - t0) / a - log_term


def roc_triple(pred, y, w=None):
    """A worker's ROC contribution for one class: (area, fp * tp, tp)."""
    tp, fp = tie_group_ends(pred, y, w)
    area = float(np.sum(np.abs(fp[1:] - fp[:-1]) * (tp[1:] + tp[:-1]) * 0.5))
    return area, float(fp[-1] * tp[-1]), float(tp[-1])


def pr_local(pred, y, w=None):
    """A worker's aucpr for one class; NaN without positive or without negative weight."""
    tp, fp = tie_group_ends(pred, y, w)
    P, N = tp[-1], fp[-1]
    if not (P > 0 and N > 0):
        return float("nan")
    return float(np.sum(pr_segment(tp[:-1], fp[:-1], tp[1:], fp[1:], P)))


def pr_triple(pred, y, w=None):
    return pr_local(pred, y, w), 1.0, 1.0


def worker_triples(metric, pred, label, w=None):
    """(K, 3) contributions of one worker; raises ValueError on a multi-class label outside [0, K)."""
    pred = np.asarray(pred)
    label = np.asarray(label, np.float32)
    local = roc_triple if metric == "auc" else pr_triple
    if pred.ndim == 1:
        return np.array([local(pred, label, w)])
    K = pred.shape[1]
    if np.any(~((label >= 0) & (label < K))):
        raise ValueError("label must be in [0, num_class)")
    return np.array([local(pred[:, c], (label == c).astype(np.float64), w) for c in range(K)])


def combine(metric, triples, multiclass):
    """The value from the (K, 3) triples summed over the workers."""
    A, L, T = triples[:, 0], triples[:, 1], triples[:, 2]
    if not multiclass:
        if metric == "auc":
            return A[0] / L[0] if L[0] > 0 else 0.5
        return A[0] / L[0]
    if np.any(~(L > 0)) or not np.sum(T) > 0:
        return float("nan")
    return float(np.sum(A / L * T) / np.sum(T))


def value(metric, pred, label, weight=None, shards=None):
    pred = np.asarray(pred)
    label = np.asarray(label)
    shards = [slice(None)] if shards is None else shards
    total = sum(worker_triples(metric, pred[s], label[s], None if weight is None else np.asarray(weight)[s])
                for s in shards)
    return combine(metric, total, pred.ndim == 2)
