"""CPU checks of tests/ranking_reference.py (the restatement the GPU ranking tests compare against) and of the
group-aligned sharding of xgboost_ray_b200/matrix.py: Delta NDCG against a brute-force swap, lambda against the
RankNet loss's derivative, the metrics on hand-computed groups, the sharding rules and the golden fixtures."""
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import ranking_reference as R
from tests.golden.make_golden_ranking import CASES, run_case
from xgboost_ray_b200.matrix import (RayDMatrix, RayDeviceQuantileDMatrix, RayShardingMode, combine_by_index,
                                     group_offsets, group_sharding_rows)

F = np.float32


def dcg(y_in_order, exp_gain, k):
    """Plain DCG@k of labels in model order (float64, NumPy log2): the brute-force side."""
    y = np.asarray(y_in_order, np.float64)[:k]
    g = 2.0 ** y - 1.0 if exp_gain else y
    return float(np.sum(g / np.log2(np.arange(len(y)) + 2.0)))


@pytest.mark.parametrize("exp_gain", [True, False])
def test_delta_ndcg_equals_swap(exp_gain):
    """|Delta NDCG| of a pair equals the change of DCG * invIDCG when the two rows swap places (whole group, k = n)."""
    rng = np.random.RandomState(0)
    for _ in range(20):
        n = rng.randint(2, 12)
        y = rng.randint(0, 5, n).astype(F)
        inv = R.inv_idcg(y, n, exp_gain)
        dsc = R.disc(n)
        for i in range(n):
            for j in range(i + 1, n):
                if y[i] == y[j]:
                    continue
                swapped = y.copy()
                swapped[[i, j]] = swapped[[j, i]]
                want = abs(dcg(swapped, exp_gain, n) - dcg(y, exp_gain, n)) * inv
                _, _, ah = R.pair_values("rank:ndcg", F(0), y[i], i, F(0), y[j], j, exp_gain, dsc, inv, False)
                gh, gl = R.gain(max(y[i], y[j]), exp_gain), R.gain(min(y[i], y[j]), exp_gain)
                dh, dl = (dsc[i], dsc[j]) if ah else (dsc[j], dsc[i])
                got = abs(((gh * dh + gl * dl) - (gl * dh + gh * dl)) * inv)
                assert abs(got - want) <= 1e-12 * max(1.0, want)


def test_pairwise_lambda_is_ranknet_derivative():
    """rank:pairwise, one pair, before both normalisations: lambda = d/ds_high log(1 + e^-(s_high - s_low)) and
    H = 2 * its second derivative (central differences)."""
    for sh, sl in ((0.3, -0.2), (2.0, 1.5), (-1.0, 0.7), (4.0, -3.0)):
        lam, H, ah = R.pair_values("rank:pairwise", F(sh), F(1), 0, F(sl), F(0), 1, True, R.disc(2), 0.0, False)
        assert ah
        loss = lambda s: np.log1p(np.exp(-(s - sl)))  # noqa: E731
        e = 1e-5
        d1 = (loss(sh + e) - loss(sh - e)) / (2 * e)
        d2 = (loss(sh + e) - 2 * loss(sh) + loss(sh - e)) / (e * e)
        assert abs(float(np.asarray(lam).reshape(-1)[0]) - d1) <= 1e-5
        assert abs(float(np.asarray(H).reshape(-1)[0]) - 2 * d2) <= 1e-3


def test_group_gradients_hand_computed():
    """Tied margins (round 0), labels 0 1 2 0 1, k = 2: every formed pair has lambda = -0.5, H = 0.5; S = 5 and every
    row is scaled by log2(6) / 5."""
    g, h = R.group_gradients("rank:pairwise", np.zeros(5, F), np.array([0, 1, 2, 0, 1], F), 2, True)
    norm = np.log2(6.0) / 5.0
    np.testing.assert_allclose(g, np.array([1.5, -0.5, -1.0, 0.5, -0.5]) * norm, rtol=1e-6)
    np.testing.assert_allclose(h, np.array([1.5, 1.5, 1.0, 0.5, 0.5]) * norm, rtol=1e-6)
    g1, h1 = R.group_gradients("rank:ndcg", np.zeros(1, F), np.ones(1, F), 32, True)
    assert g1[0] == 0 and h1[0] == 0                     # a group of one row
    ge, he = R.group_gradients("rank:ndcg", np.zeros(4, F), np.full(4, 2, F), 32, True)
    assert np.all(ge == 0) and np.all(he == 0)           # all labels equal: no pair


def test_model_order_ties_and_signed_zero():
    assert R.model_order(np.array([0.0, -0.0, 1.0, 0.0], F)).tolist() == [2, 0, 1, 3]
    assert R.model_order(np.full(5, 0.5, F)).tolist() == [0, 1, 2, 3, 4]


def test_metrics_hand_computed():
    ptr = np.array([0, 4])
    pred = np.array([0.9, 0.8, 0.7, 0.1], F)
    y = np.array([0, 1, 0, 1], F)
    # map: hits at positions 2 and 4 -> (1/2 + 2/4) / 2
    assert R.metric("map", pred, y, ptr) == pytest.approx(0.5)
    assert R.metric("map@2", pred, y, ptr) == pytest.approx(0.25)
    assert R.metric("pre@2", pred, y, ptr) == pytest.approx(0.5)
    assert R.metric("pre@10", pred, y, ptr) == pytest.approx(0.2)             # @k beyond the group: hits / k
    d = 1 / np.log2(3) + 1 / np.log2(5)
    assert R.metric("ndcg", pred, y, ptr) == pytest.approx(d / (1 + 1 / np.log2(3)))
    assert R.metric("ndcg@10", pred, y, ptr) == pytest.approx(d / (1 + 1 / np.log2(3)))
    # all-zero labels: 1, or 0 with the trailing '-'
    z = np.zeros(4, F)
    assert R.metric("ndcg", pred, z, ptr) == 1.0 and R.metric("ndcg-", pred, z, ptr) == 0.0
    assert R.metric("map", pred, z, ptr) == 1.0 and R.metric("map@2-", pred, z, ptr) == 0.0
    # ties in the prediction keep the row order
    assert R.metric("pre@1", np.zeros(4, F), np.array([0, 1, 1, 1], F), ptr) == 0.0
    assert R.metric("pre@1", np.zeros(4, F), np.array([1, 0, 0, 0], F), ptr) == 1.0
    # averaged over groups
    assert R.metric("pre@1", np.zeros(4, F), np.array([1, 0, 0, 1], F), np.array([0, 2, 4])) == 0.5
    assert R.parse_metric("ndcg@5-") == ("ndcg", 5, True)


def test_groups_and_sharding_rules():
    qid = np.array([3, 3, 5, 7, 7, 7, 9, 9, 11])
    off = group_offsets(qid)
    assert off.tolist() == R.group_ptr(qid).tolist() == [0, 2, 3, 6, 8, 9]
    for mode, name in ((RayShardingMode.INTERLEAVED, "interleaved"), (RayShardingMode.BATCH, "batch")):
        for W in (1, 2, 3, 5):
            shards = [group_sharding_rows(mode, r, W, off) for r in range(W)]
            assert all(s.tolist() == R.shard_rows(off, name, r, W).tolist() for r, s in enumerate(shards))
            assert sorted(np.concatenate(shards).tolist()) == list(range(len(qid)))      # the union is all rows
            for s in shards:                                                           # every group whole
                for b, e in zip(off[:-1], off[1:]):
                    inside = np.isin(np.arange(b, e), s)
                    assert inside.all() or not inside.any()
            pred = [np.asarray(s, F) * 10 for s in shards]                           # reassembly
            assert combine_by_index(shards, pred).tolist() == (np.arange(len(qid)) * 10).tolist()
    assert [g.tolist() for g in [group_sharding_rows(RayShardingMode.INTERLEAVED, r, 2, off) for r in range(2)]] == \
        [[0, 1, 3, 4, 5, 8], [2, 6, 7]]
    with pytest.raises(ValueError, match="5 query groups .* 6 actors"):
        group_sharding_rows(RayShardingMode.BATCH, 0, 6, off)


def test_raydmatrix_sorts_by_qid_stably_and_shards_whole_groups():
    rng = np.random.RandomState(1)
    n = 300
    X = rng.rand(n, 3).astype(F)
    qid = rng.randint(0, 20, n)
    y = rng.randint(0, 4, n).astype(F)
    d = RayDMatrix(X, y, qid=qid, num_actors=3)
    order = np.argsort(qid, kind="mergesort")
    rows = np.concatenate(d._row_index)
    assert sorted(rows.tolist()) == list(range(n))
    for r in range(3):
        shard = d.get_data(r)
        assert np.array_equal(np.asarray(shard["data"]), X[order][d._row_index[r]])
        assert np.array_equal(np.asarray(shard["label"]), y[order][d._row_index[r]])
        local = np.asarray(shard["qid"])
        assert np.all(np.diff(local) >= 0)                                 # shard-local group numbers, sorted
        assert len(np.unique(local)) == len(np.unique(qid[order][d._row_index[r]]))
    # a qid column of a frame is not a feature
    import pandas as pd
    df = pd.DataFrame(X, columns=["a", "b", "c"])
    df["q"], df["y"] = qid, y
    d2 = RayDMatrix(df, label="y", qid="q", num_actors=2)
    assert np.asarray(d2.get_data(0)["data"]).shape[1] == 3


def test_raydmatrix_errors():
    X = np.zeros((10, 2), F)
    y = np.zeros(10, F)
    with pytest.raises(NotImplementedError, match="per-group weight"):
        RayDMatrix(X, y, qid=np.zeros(10), weight=np.ones(10))
    with pytest.raises(ValueError, match="does not support ranking"):
        RayDeviceQuantileDMatrix(X, y, qid=np.zeros(10))
    with pytest.raises(ValueError, match="2 query groups .* 3 actors"):
        RayDMatrix(X, y, qid=np.repeat([0, 1], 5), num_actors=3)


@pytest.mark.parametrize("name", CASES)
def test_golden_ranking_fixtures_reproduced(name):
    want = json.load(open(os.path.join(os.path.dirname(__file__), "golden", name + ".json")))
    got = run_case(name)
    assert got == want
