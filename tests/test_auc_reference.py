"""tests/auc_reference.py (the `auc` / `aucpr` rules of DESIGN.md §2 item 17) against scikit-learn, scipy quadrature
and hand-computed answers.  CPU only."""
import math

import numpy as np
import pytest
from scipy import integrate
from sklearn.metrics import roc_auc_score

from tests import auc_reference as R


def tied_binary(n=3000, seed=0, weighted=True):
    rng = np.random.RandomState(seed)
    pred = np.round(rng.uniform(size=n), 1).astype(np.float32)           # 11 distinct values: heavy ties
    y = (rng.uniform(size=n) < 0.2 + 0.6 * pred).astype(np.float32)
    w = rng.gamma(2.0, 1.0, size=n).astype(np.float32) if weighted else None
    return pred, y, w


def softmax_probs(n, K, seed, pool=300):
    """float64 probabilities drawn from `pool` distinct rows (heavy ties within every class) and noisy labels."""
    rng = np.random.RandomState(seed)
    m = rng.normal(size=(pool, K))[rng.randint(0, pool, size=n)]
    y = np.argmax(m + rng.normal(scale=1.5, size=(n, K)), axis=1).astype(np.float32)
    e = np.exp(m)
    return e / e.sum(axis=1, keepdims=True), y


@pytest.mark.parametrize("weighted", [False, True])
def test_binary_roc_is_sklearn(weighted):
    pred, y, w = tied_binary(seed=1, weighted=weighted)
    assert abs(R.value("auc", pred, y, w) - roc_auc_score(y, pred, sample_weight=w)) < 1e-12


@pytest.mark.parametrize("K", [3, 20])
def test_multiclass_roc_is_sklearn_ovr_weighted(K):
    P, y = softmax_probs(4000, K, seed=K)
    w = np.random.RandomState(K).uniform(0.2, 3.0, size=len(y)).astype(np.float32)
    # float64 weights: scikit-learn sums the class weights in the weights' own dtype
    want = roc_auc_score(y, P, multi_class="ovr", average="weighted", sample_weight=w.astype(np.float64),
                         labels=np.arange(K))
    assert abs(R.value("auc", P, y, w) - want) < 1e-12
    want = roc_auc_score(y, P, multi_class="ovr", average="weighted", labels=np.arange(K))
    assert abs(R.value("auc", P, y) - want) < 1e-12


def test_pr_segments_are_the_integral_of_the_interpolated_precision():
    rng = np.random.RandomState(3)
    P = 37.5
    for _ in range(200):
        tp0, fp0 = rng.uniform(0, 20) * rng.randint(0, 2), rng.uniform(0, 20) * rng.randint(0, 2)
        tp1, fp1 = tp0 + rng.uniform(0, 15), fp0 + rng.uniform(0, 15) * rng.randint(0, 2)
        h = (fp1 - fp0) / (tp1 - tp0)

        def precision(t):
            tp = t * P
            fp = fp0 + h * (tp - tp0)
            return tp / (tp + fp)
        want, err = integrate.quad(precision, tp0 / P, tp1 / P, epsabs=1e-13, epsrel=1e-12)
        assert abs(R.pr_segment(tp0, fp0, tp1, fp1, P) - want) < 1e-10 + 10 * err
    assert R.pr_segment(3.0, 2.0, 3.0, 7.0, P) == 0.0                   # a step with negatives only adds nothing


def test_hand_computed_answers():
    # perfect ranking: both metrics 1
    assert R.value("aucpr", [0.9, 0.8, 0.3, 0.2], [1, 1, 0, 0]) == 1.0
    assert R.value("auc", [0.9, 0.8, 0.3, 0.2], [1, 1, 0, 0]) == 1.0
    # everything tied: aucpr = P / (P + N), auc = 1/2
    w = np.array([1.0, 2.0, 0.5, 1.5, 3.0])
    y = np.array([1, 0, 1, 0, 0])
    assert math.isclose(R.value("aucpr", np.full(5, 0.4), y, w), 1.5 / 8.0, rel_tol=1e-15)
    assert R.value("auc", np.full(5, 0.4), y, w) == 0.5
    # 4 rows, positives at ranks 1 and 3: the segment (1, 1) -> (2, 1) has h = 0, b = 1/2, a = 1:
    # 1/2 + 1/2 - 1/2 ln(3/2) for recall 1/2 -> 1, plus 1/2 from (0, 0) -> (1, 0)
    got = R.value("aucpr", [0.9, 0.7, 0.5, 0.1], [1, 0, 1, 0])
    assert math.isclose(got, 0.5 + 0.5 - 0.5 * math.log(1.5), rel_tol=1e-15)
    assert R.value("auc", [0.9, 0.7, 0.5, 0.1], [1, 0, 1, 0]) == 0.75
    # a tie group mixing both classes: (0, 0) -> (1, 1) -> (2, 2): h = 1, a = 2, b = 0 both times
    assert math.isclose(R.value("aucpr", [0.8, 0.8, 0.2, 0.2], [1, 0, 1, 0]), 0.5, rel_tol=1e-15)
    # six rows, three classes, perfect one-vs-rest separation
    P = np.array([[.7, .2, .1], [.6, .3, .1], [.1, .8, .1], [.2, .7, .1], [.1, .1, .8], [.2, .2, .6]])
    lab = np.array([0, 0, 1, 1, 2, 2])
    assert R.value("auc", P, lab) == 1.0 and R.value("aucpr", P, lab) == 1.0


def test_nan_rules():
    y1 = np.ones(4)
    p = [0.9, 0.5, 0.4, 0.1]
    assert R.value("auc", p, y1) == 0.5                                  # binary ROC, one class: 0.5
    assert math.isnan(R.value("aucpr", p, y1))                           # no negatives
    assert math.isnan(R.value("aucpr", p, np.zeros(4)))                  # no positives
    P, y = softmax_probs(300, 4, seed=5)
    y[y == 2] = 0                                                       # class 2 absent
    assert math.isnan(R.value("auc", P, y)) and math.isnan(R.value("aucpr", P, y))
    with pytest.raises(ValueError, match="num_class"):
        R.value("auc", P, np.append(y[:-1], 4.0))
    with pytest.raises(ValueError, match="num_class"):
        R.value("aucpr", P, np.append(y[:-1], -1.0))


def test_multi_worker_rules():
    pred, y, w = tied_binary(n=2000, seed=7)
    shards = [slice(0, None, 2), slice(1, None, 2)]
    # ROC: areas and fp*tp summed separately
    t0, t1 = (R.roc_triple(pred[s], y[s], w[s]) for s in shards)
    assert R.value("auc", pred, y, w, shards) == (t0[0] + t1[0]) / (t0[1] + t1[1])
    # PR: the mean of the workers' values, which differs from the one-worker value
    a0, a1 = (R.pr_local(pred[s], y[s], w[s]) for s in shards)
    assert R.value("aucpr", pred, y, w, shards) == (a0 + a1) / 2
    assert R.value("aucpr", pred, y, w, shards) != R.value("aucpr", pred, y, w)
    # one worker without negatives makes the whole aucpr NaN
    y2 = y.copy()
    y2[0::2] = 1
    assert math.isnan(R.value("aucpr", pred, y2, w, shards))
    # multi-class aucpr: unweighted mean over classes and workers
    P, lab = softmax_probs(1200, 3, seed=8)
    per = [R.pr_local(P[s][:, c], (lab[s] == c).astype(float)) for s in shards for c in range(3)]
    assert math.isclose(R.value("aucpr", P, lab, None, shards), np.mean(per), rel_tol=1e-14)
    # multi-class ROC: per class sum(area) / sum(fp*tp), weighted by the summed positives
    tri = [R.worker_triples("auc", P[s], lab[s]) for s in shards]
    tot = tri[0] + tri[1]
    want = np.sum(tot[:, 0] / tot[:, 1] * tot[:, 2]) / np.sum(tot[:, 2])
    assert R.value("auc", P, lab, None, shards) == want


def test_aucpr_is_maximized_for_early_stopping():
    from xgboost_ray_b200.engine import _maximized
    assert _maximized("aucpr") and _maximized("auc")
    assert not _maximized("logloss")
