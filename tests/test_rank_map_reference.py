"""CPU checks of tests/rank_map_reference.py (the restatement the GPU rank:map tests compare against): Delta AP against a brute-force swap in exact arithmetic, the hit prefixes' summation order against exact
sums and a scalar replay of the kernel's loop, groups without a formed pair, the binary-label rule and the golden
fixture."""
import json
import math
import os
from fractions import Fraction

import numpy as np
import pytest

from tests import rank_map_reference as R
from tests.golden.make_golden_rank_map import CASES, run_case

F = np.float32


def exact_ap_scaled(hits, weights):
    """N * L * AP of a 0/1 list as a Python integer: sum over the hits p of R_p * L / (p + 1), L = lcm(1..n)."""
    total, r = 0, 0
    for p, h in enumerate(hits):
        if h:
            r += 1
            total += r * weights[p]
    return total


def check_group(hits):
    """Every pair i < j with different labels: the reference's Delta equals |AP(swapped) - AP| within 1e-12 relative."""
    hits = [int(v) for v in hits]
    n = len(hits)
    L = math.lcm(*range(1, n + 1))
    weights = [L // (p + 1) for p in range(n)]
    Rr, A = R.hit_prefixes(np.array(hits, bool))
    N = int(Rr[-1])
    base = exact_ap_scaled(hits, weights)
    checked = 0
    for i in range(n):
        for j in range(i + 1, n):
            if hits[i] == hits[j]:
                continue
            sw = list(hits)
            sw[i], sw[j] = sw[j], sw[i]
            want = float(Fraction(abs(exact_ap_scaled(sw, weights) - base), N * L))
            got = float(R.map_delta(Rr, A, N, i, j, hits[i] > hits[j]))
            assert abs(got - want) <= 1e-12 * want, (n, i, j, got, want)
            checked += 1
    return checked


def patterns(n, rng):
    out = [rng.rand(n) < 0.5, rng.rand(n) < 0.1]
    one = np.zeros(n, bool)
    one[rng.randint(n)] = True                                   # a single hit
    out.append(one)
    most = np.ones(n, bool)
    most[rng.randint(n)] = False                                 # all hits but one
    out.append(most)
    ends = np.zeros(n, bool)
    ends[[0, n - 1]] = True                                      # hits only at the ends
    out.append(ends)
    return [p for p in out if 0 < p.sum() < n]


@pytest.mark.parametrize("n", [2, 3, 7, 50, 300])
def test_delta_map_equals_brute_force_swap(n):
    rng = np.random.RandomState(n)
    assert sum(check_group(p) for p in patterns(n, rng)) > 0
    if n == 3:
        for bits in range(1, 7):                                 # every mixed 3-row group
            check_group([(bits >> b) & 1 for b in range(3)])


def test_delta_map_hand_computed():
    """r = [1, 0, 1, 0]: AP = (1/1 + 2/3) / 2 = 5/6.  Swap (0, 1): [0, 1, 1, 0], AP = (1/2 + 2/3) / 2 = 7/12, -1/4.
    Swap (1, 2): [1, 1, 0, 0], AP = 1, +1/6.  Swap (0, 3): [0, 0, 1, 1], AP = (1/3 + 2/4) / 2 = 5/12, -5/12."""
    hits = np.array([1, 0, 1, 0], bool)
    Rr, A = R.hit_prefixes(hits)
    assert Rr.tolist() == [1, 1, 2, 2] and A.tolist() == [1.0, 1.0, 1.0 + 1.0 / 3.0, 1.0 + 1.0 / 3.0]
    for (i, j), want in (((0, 1), 1 / 4), ((1, 2), 1 / 6), ((0, 3), 5 / 12), ((2, 3), 1 / 12)):
        got = float(R.map_delta(Rr, A, 2, i, j, hits[i] > hits[j]))
        assert got == pytest.approx(want, rel=1e-15), (i, j)
    check_group(hits)


def kernel_replay(hits):
    """rank_kernel.cu's prefix loops, one scalar operation at a time (128 threads, chunks of ceil(n / 128))."""
    n = len(hits)
    c = (n + 127) // 128
    A, Rr = [0.0] * n, [0] * n
    tot_a, tot_r = [0.0] * 128, [0] * 128
    for t in range(128):
        a, r = 0.0, 0
        for p in range(min(t * c, n), min(t * c + c, n)):
            if hits[p]:
                r += 1
                a = a + 1.0 / float(p + 1)
            A[p], Rr[p] = a, r
        tot_a[t], tot_r[t] = a, r
    ca, cr = 0.0, 0
    for t in range(128):
        tot_a[t], tot_r[t], ca, cr = ca, cr, ca + tot_a[t], cr + tot_r[t]
    for t in range(128):
        for p in range(min(t * c, n), min(t * c + c, n)):
            A[p], Rr[p] = tot_a[t] + A[p], Rr[p] + tot_r[t]
    return np.array(Rr), np.array(A)


@pytest.mark.parametrize("n", [1, 2, 127, 128, 129, 300, 4097])
def test_hit_prefixes_order(n):
    """The vectorised prefixes are the kernel's loop bit for bit, and close to the exact sums: the longest addition
    chain of A_p is ceil(n / 128) local additions plus 128 carries, so its error is at most that many units of
    2^-53 of A_p (positive terms).  The sequential carries cost a few ulps (6 at n = 4097, all hits), not 1."""
    rng = np.random.RandomState(n)
    for hits in (np.ones(n, bool), rng.rand(n) < 0.3, np.zeros(n, bool)):
        Rr, A = R.hit_prefixes(hits)
        kr, ka = kernel_replay(hits)
        assert np.array_equal(Rr, kr) and np.array_equal(A.view(np.uint64), ka.view(np.uint64))
        assert np.array_equal(Rr, np.cumsum(hits))
        chain = (n + 127) // 128 + 128
        s = Fraction(0)
        for p in range(n):
            if hits[p]:
                s += Fraction(1, p + 1)
            e = float(s)
            assert abs(Fraction(float(A[p])) - s) <= chain * Fraction(1, 2 ** 53) * s, (p, A[p], e)


@pytest.mark.parametrize("n", [1, 2, 5, 40, 300])
def test_no_pair_gives_zero_gradients(n):
    for y in (np.zeros(n, F), np.ones(n, F)):
        for m in (np.zeros(n, F), np.linspace(-1, 1, n).astype(F)):
            g, h = R.group_gradients(m, y, 32)
            assert np.all(g == 0) and np.all(h == 0)


def test_map_gradients_sanity():
    """Hits get negative g (pushed up) and misses positive; h > 0 where a pair formed; the group's g sums to ~0."""
    rng = np.random.RandomState(3)
    y = (rng.rand(60) < 0.3).astype(F)
    m = rng.normal(size=60).astype(F)
    g, h = R.group_gradients(m, y, 60)
    assert np.all(g[y == 1] < 0) and np.all(g[y == 0] > 0) and np.all(h > 0)
    assert abs(float(np.sum(g.astype(np.float64)))) <= 1e-5 * float(np.sum(np.abs(g)))


def test_label_check():
    R.check_labels(np.array([0, 1, 1, 0], F))
    for bad in (0.5, 2.0, np.nan, -1.0, np.inf):
        with pytest.raises(ValueError, match="0 or 1"):
            R.check_labels(np.array([0, 1, bad], F))


@pytest.mark.parametrize("name", CASES)
def test_golden_rank_map_fixture_reproduced(name):
    want = json.load(open(os.path.join(os.path.dirname(__file__), "golden", name + ".json")))
    assert run_case(name) == want
