"""reg:quantileerror's exact selection on the H100 at the boundaries of its radix select (quantile_kernel.cu; DESIGN.md
§2 item 16): order statistics j and j + 1 whose keys part in each of the four bytes, the sign boundary and signed zeros,
subnormals and ±FLT_MAX/2, ties straddling the target, the alphas where the unweighted rule switches to the minimum or
maximum or has frac = 0, and fixed-point masses that round half-way, round to 0 or end exactly on the target.

The intercept (base_score unset) selects over the labels as one segment, so a label set is a residual set under exact
control; it is compared bit for bit with tests/quantile_reference.py's np.sort rule at 1-257 rows and at 1.2M rows,
where every SM's CTA flushes its shared-memory counts.  Leaf refreshes run both count paths: per-CTA shared-memory
counts (unweighted max_depth 7, weighted 6) and global atomics (unweighted 8, weighted 7), with the trees, every leaf
value and the train margins compared bit for bit, and each case shows from the reference that its leaves put the
targets on the boundaries.

Measured on an H100 80 GB HBM3 (700 W power limit): the file runs in about 30 s (23 s of it the 1.2M-row intercepts),
and the test process peaks at 816 MiB of device memory, CUDA context included."""
import numpy as np
import pytest

from tests import quantile_reference as R
from tests.test_gpu_quantile import same_as_reference

pytestmark = pytest.mark.gpu
F32 = np.float32
BIG = 1_200_000


@pytest.fixture(scope="module")
def eng():
    from xgboost_ray_b200 import engine
    if engine.device_count() < 1:
        pytest.fail("no CUDA device visible: GPU tests must run on an H100")
    return engine


def bits(v):
    return np.array([v], F32).tobytes()


def intercept(eng, y, alphas, w=None):
    X = (np.arange(y.size) % 7).astype(F32).reshape(-1, 1)
    params = {"objective": "reg:quantileerror", "quantile_alpha": [float(a) for a in alphas], "max_depth": 2}
    bst = eng.train(params, eng.DMatrix(X, label=y, weight=w), num_boost_round=1, verbose_eval=False)
    return F32(bst.params["base_score"])


@pytest.mark.timeout(900)
@pytest.mark.parametrize("n", [1, 2, 3, 4, 255, 256, 257, BIG])
def test_intercept_is_the_sort_at_the_boundaries(eng, n):
    rng = np.random.RandomState(n)
    bad, runs = [], 0

    def check(name, y, alphas, w=None):
        nonlocal runs
        got, want = intercept(eng, y, alphas, w), R.intercept(y, w, alphas)
        runs += 1
        if bits(got) != bits(want):
            bad.append("%s alphas %s: got %r, want %r" % (name, [float(a) for a in alphas], got, want))

    sets = R.boundary_sets(n)
    for name, y, alphas in sets:
        for a in alphas:
            check(name, y, [a])
        for kind in ("int", "half", "pow2"):
            if n == BIG and name.startswith("tied"):
                continue
            w = R.boundary_weights(kind, n, rng)
            check("%s %s weights" % (name, kind), y, alphas[:2], w)
            if kind == "pow2":
                a = R.boundary_alpha(y, w, rng)
                if a is not None:
                    check("%s on a cumulative boundary" % name, y, [a], w)
    # nine alphas at once over moderate labels (the fp32 mean of nine quantiles of ±FLT_MAX/2 would overflow)
    y = rng.choice(R.POOL[np.abs(R.POOL) <= 4], n)
    nine = [F32(1e-7), F32(0.1), F32(0.25), F32(1.0 / (n + 1)), F32(0.5), F32(n / (n + 1)), F32(0.75), F32(0.9),
            F32(0.99999994)]
    check("nine alphas", y, nine)
    check("nine alphas, int weights", y, nine, R.boundary_weights("int", n, rng))
    assert not bad, "%d of %d intercepts differ:\n%s" % (len(bad), runs, "\n".join(bad[:20]))


# ------------------------------------------------------------------ leaf refresh on both count paths
ALPHAS = [0.25, 0.5, 0.7]        # 0.25 = 1/(n+1) at n = 3 and below 1/3 at n = 2; 0.7 above 2/3, below 3/4
LEAF_POOL = R.POOL[np.abs(R.POOL) <= 4]      # every split pair but ±FLT_MAX/2, whose later residuals could overflow

CASES = {
    # name: (max_depth, weights, extra)  -- unweighted smem <= 7 < global; weighted smem <= 6 < global
    "unweighted-smem": (7, None, None),
    "unweighted-global": (8, None, None),
    "weighted-smem": (6, "int", None),
    "weighted-global": (7, "int", None),
    "half-masses-global": (7, "half", None),
    "weighted-subsample": (7, "int", "subsample"),
    "weighted-base_margin": (7, "half", "base_margin"),
    "weighted-nan-categorical": (7, "int", "nan_cat"),
}


def leaf_coverage(ref):
    """From the reference's leaves: the passes at which the two targets split (unweighted), the passes at which the
    chosen value's key parts from the next larger residual of its leaf (weighted), whether a leaf holds both -0 and
    +0 residuals, a leaf of at most 3 rows, and a leaf with a row of mass 0"""
    splits, parts = set(), set()
    both_zeros = small = zero_mass = False
    for alpha, segs in ref.segments:
        for r, m in segs:
            q, split = R.radix_select(r, alpha, m)
            splits.add(split)
            above = np.unique(np.where(r == 0, F32(0.0), r)[r > q])
            if above.size:
                diff = int(R.q_key([q])[0] ^ R.q_key(above[:1])[0])
                parts.add(3 - (diff.bit_length() - 1) // 8)
            zeros = np.signbit(r[r == 0])
            both_zeros |= bool(zeros.any() and (~zeros).any())
            small |= r.size <= 3
            zero_mass |= m is not None and bool((m == 0).any())
    return splits, parts, both_zeros, small, zero_mass


@pytest.mark.timeout(600)
@pytest.mark.parametrize("case", list(CASES))
def test_leaf_refresh_on_both_count_paths(eng, oracle, case):
    depth, wkind, extra = CASES[case]
    n, f = 3000, 6
    rng = np.random.RandomState(len(case))
    X = rng.uniform(0, 10, size=(n, f)).astype(F32)
    y = rng.choice(LEAF_POOL, n)
    w = None if wkind is None else R.boundary_weights(wkind, n, rng)
    params = {"objective": "reg:quantileerror", "quantile_alpha": ALPHAS, "max_depth": depth, "eta": 0.5,
              "base_score": 0.0, "min_child_weight": 0.0}
    kw, is_cat, bm = {}, None, None
    if extra == "subsample":
        params.update(subsample=0.6, seed=11)
    elif extra == "base_margin":
        bm = np.where(rng.uniform(size=(n, len(ALPHAS))) < 0.25, F32(0.5), F32(0.0)).astype(F32)
        kw["base_margin"] = bm
    elif extra == "nan_cat":
        X[rng.uniform(size=X.shape) < 0.05] = np.nan
        X[:, f - 1] = rng.randint(0, 12, size=n)
        is_cat = [0] * (f - 1) + [1]
        kw.update(feature_types=["q"] * (f - 1) + ["c"], enable_categorical=True)
    d = eng.DMatrix(X, label=y, weight=w, **kw)
    bst = eng.train(params, d, num_boost_round=3, verbose_eval=False)
    ref = same_as_reference(oracle, bst, params, X, y, 3, weight=w, is_cat=is_cat, base_margin=bm)
    m = np.asarray(bst.predict(d, output_margin=True, training=True)).reshape(n, len(ALPHAS))
    assert m.tobytes() == ref.margin.tobytes()
    if extra == "nan_cat":
        assert any(t["split_type"].any() for t in bst.get_trees())
    splits, parts, both_zeros, small, zero_mass = leaf_coverage(ref)
    if wkind is None:
        assert splits >= {0, 1, 2, 3, None}, splits
    else:
        assert parts >= {0, 1, 2, 3}, parts
    assert both_zeros and small
    assert zero_mass or wkind != "half"
