"""CPU checks of tests/objective_reference.py's scalar objective gradients at the edges of binary32: the margins where
b2_expf clamps (88.7) or flushes to zero (-103), the sigmoid's 1e-16 terms and hessian floor, squared-log's clamp and
hessian floor, b2_log1pf's branches, pseudo-Huber's overflowing square, Poisson's and Tweedie's shifted and scaled exp
arguments, scale_pos_weight on y == 1 exactly, subnormal labels and weights, and weights that overflow the pair.

On every element where a float64 evaluation of the same formulas (with the kernels' clamps) is finite and normal, the
binary32 restatement is within ULP_BOUND units in the last place of the magnitudes it adds; where the float64 pair
overflows, the objectives that check finiteness write (0, 0) and count the row.  The edge grids are also the input of
tests/test_gpu_objective_gradients.py, which requires the GPU's pairs to equal the restatement's bit for bit."""
import numpy as np
import pytest

from tests import objective_reference as R

F = np.float32
FMAX = float(np.finfo(F).max)
TINY = float(np.finfo(F).tiny)
ULP_BOUND = 8


def f32(*v):
    return [float(F(x)) for x in v]


def around(x, k=2):
    """x in binary32 and its k neighbours on each side."""
    x = F(x)
    out, lo, hi = [float(x)], x, x
    for _ in range(k):
        lo, hi = np.nextafter(lo, F(-np.inf)), np.nextafter(hi, F(np.inf))
        out += [float(lo), float(hi)]
    return out


SUB = 2.0 ** -149
MARGINS = sorted(set(
    f32(0.0, SUB, -SUB, 2.0 ** -126, -(2.0 ** -126), 1e-8, -1e-8, 1.0, -1.0, 16.6, -16.6, 88.72, -88.72, -103.0,
        -103.0001, 104.0, -104.0, FMAX / 2, -FMAX / 2) + around(88.7) + around(-88.7)) | {-0.0}, key=lambda v: (v, str(v)))
WEIGHTS = f32(1.0, 0.0, SUB, 1e-30, 1e30, 0.5)
LABELS = {
    "reg:squarederror": f32(0.0, 1.0, 0.99999994, 1.0000001, -1.0, 3e38, -3e38) + around(3e38, 1),
    "binary:logistic": f32(0.0, 1.0, 0.99999994, 1.0000001, 0.5, -2.0, 3e38),
    "reg:logistic": f32(0.0, 1.0, 0.99999994, 0.5, SUB),
    "reg:squaredlogerror": f32(-0.99999994, -0.5, 0.0, 1.0, 0.99999994, 1.0000001, SUB, 1e-8, 3e38),
    "reg:pseudohubererror": f32(0.0, 1.0, 1.0000001, -1.0, 3e38, -3e38),
    "count:poisson": f32(0.0, 1.0, 0.99999994, 1.0000001, SUB, 3e38),
    "reg:gamma": f32(SUB, 2.0 ** -130, 1e-40, 2.0 ** -126, 1.0, 1.0000001, 3e38),
    "reg:tweedie": f32(0.0, 1.0, 0.99999994, SUB, 3e38),
}
LABELS["reg:linear"] = LABELS["reg:squarederror"]
LABELS["binary:logitraw"] = LABELS["reg:logistic"]
SPW = f32(1.0, 0.0, 1e-30, 1e30)


def param_sets(obj):
    """The parameter values each objective's grid runs with."""
    if obj in R.REG_LOSS:
        return [{"scale_pos_weight": s} for s in SPW]
    if obj == "reg:pseudohubererror":
        return [{"huber_slope": s} for s in f32(1.0, 1e-20, 1e20)]
    if obj == "count:poisson":
        return [{"max_delta_step": s} for s in f32(0.0, 0.7)]
    if obj == "reg:tweedie":
        return [{"tweedie_variance_power": r} for r in f32(1.0, 1.0 + 2.0 ** -23, 1.5, 2.0 - 2.0 ** -23)]
    return [{}]


def margins_for(params):
    """The common edge margins, and the margins where an objective's exp argument crosses 88.7 or -103."""
    obj, m = params["objective"], list(MARGINS)
    if obj == "count:poisson":
        m += around(float(F(88.7) - F(R.max_delta_step(params))))
    if obj == "reg:tweedie":
        rho = R.objective_param(params)
        for c in (F(1.0) - rho, F(2.0) - rho):
            if c != 0:
                for edge in (88.7, -103.0):
                    m += around(float(F(edge) / c))
    return np.array(m, F)


def edge_grid(params, weighted):
    """(margin, label, weight or None): every edge margin with every label of the objective, each with every edge
    weight when weighted, plus label == margin (z = 0 for pseudo-Huber).  For squared error and the logistic family,
    whose kernels have no finiteness flag, the rows whose pair overflows are left out: failing them is a separate
    design question (it needs a host sync per round), so their grids stay on finite pairs."""
    obj = params["objective"]
    m, y = margins_for(params), np.array(LABELS[obj], F)
    mm, yy = [a.reshape(-1) for a in np.meshgrid(m, y, indexing="ij")]
    if obj in ("reg:squarederror", "reg:linear", "reg:pseudohubererror", "binary:logistic"):
        fin = np.abs(m) <= FMAX   # every label is legal for these: add label == margin
        mm, yy = np.concatenate([mm, m[fin]]), np.concatenate([yy, m[fin]])
    w = None
    if weighted:
        k = len(mm)
        mm, yy = np.tile(mm, len(WEIGHTS)), np.tile(yy, len(WEIGHTS))
        w = np.repeat(np.array(WEIGHTS, F), k)
    if obj not in R.CHECKS_FINITE:
        g, h, _ = R.gradients(params, mm, yy, w)
        keep = np.isfinite(g) & np.isfinite(h)
        mm, yy = mm[keep], yy[keep]
        w = None if w is None else w[keep]
    return mm.astype(F), yy.astype(F), w


def all_cases(objectives=R.SCALAR_OBJECTIVES):
    """(params, weighted) for every objective and parameter set."""
    return [(dict(p, objective=o), wt) for o in objectives for p in param_sets(o) for wt in (False, True)]


def case_id(case):
    params, weighted = case
    extra = ",".join("%s=%g" % (k, v) for k, v in params.items() if k != "objective")
    return "%s[%s]%s" % (params["objective"], extra, "-w" if weighted else "")


# ---------------------------------------------------------------- float64 evaluation
def exp64(x):
    """b2_expf's clamps on the binary32 argument, the value in float64."""
    x32 = np.asarray(x, np.float64).astype(F)
    v = np.exp(np.minimum(np.asarray(x, np.float64), float(F(88.7))))
    return np.where(x32 < F(-103.0), 0.0, np.where(x32 > F(88.7), np.exp(float(F(88.7))), v))


def float64_pairs(params, p, y, w):
    """(g, h, scale of g, scale of h) in float64 with the kernels' clamps; the scales are the magnitudes of the terms
    added (times 1 + |argument| where an exp takes a rounded argument), so the tolerance allows for cancellation."""
    obj = params["objective"]
    p, y = p.astype(np.float64), y.astype(np.float64)
    w = np.ones_like(p) if w is None else w.astype(np.float64)
    with np.errstate(all="ignore"):
        if obj in R.REG_LOSS:
            w = np.where(y == 1.0, w * float(F(params.get("scale_pos_weight", 1.0))), w)
        if obj in ("reg:squarederror", "reg:linear"):
            g, h, gs, hs = p - y, np.ones_like(p), np.abs(p) + np.abs(y), np.ones_like(p)
        elif obj in R.LOGISTIC:
            s = 1.0 / (1.0 + exp64(np.minimum(-p, float(F(88.7)))) + float(F(1e-16)))
            h = np.maximum(s * (1 - s), float(F(1e-16)))
            g, gs, hs = s - y, s + np.abs(y), np.maximum(s, h)
        elif obj == "reg:squaredlogerror":
            q = np.maximum(p, float(F(-1.0) + F(1e-6)))
            lq, ly = np.log1p(q), np.log1p(y)
            g, gs = (lq - ly) / (q + 1), (np.abs(lq) + np.abs(ly)) / (q + 1)
            h = np.maximum((-lq + ly + 1) / (q + 1) ** 2, float(F(1e-6)))
            hs = np.maximum((np.abs(lq) + np.abs(ly) + 1) / (q + 1) ** 2, h)
        elif obj == "reg:pseudohubererror":
            d = float(R.objective_param(params))
            s = 1 + ((p - y) / d) ** 2
            g, h = (p - y) / np.sqrt(s), 1 / (s * np.sqrt(s))
            gs, hs = np.abs(g), h
        elif obj == "count:poisson":
            a = float(R.objective_param(params))
            g, h = exp64(p) - y, exp64(p + a)
            gs, hs = exp64(p) + y, h * (1 + np.abs(p + a))
        elif obj == "reg:gamma":
            r = y / exp64(p)
            g, h, gs, hs = 1 - r, r, 1 + r, r * (1 + np.abs(p))
        else:
            rho = float(R.objective_param(params))
            e1, e2 = exp64((1 - rho) * p), exp64((2 - rho) * p)
            g, h = -y * e1 + e2, -y * (1 - rho) * e1 + (2 - rho) * e2
            gs = (y * e1 + e2) * (1 + np.abs(p))
            hs = (y * abs(1 - rho) * e1 + (2 - rho) * e2) * (1 + np.abs(p))
        return g * w, h * w, gs * w, hs * w


def short_of_bits(params, p, y):
    """Rows where a binary32 intermediate that multiplies is subnormal (an exp result, gamma's y / exp(p), or Tweedie's
    y (1 - rho) for a subnormal label): it carries fewer than 24 bits, so the row is not held to the ulp bound."""
    obj = params["objective"]
    a = R.objective_param(params)
    if obj == "count:poisson":
        args = [p, p + a]
    elif obj == "reg:gamma":
        args = [p]
    elif obj == "reg:tweedie":
        args = [(F(1.0) - a) * p, (F(2.0) - a) * p]
    elif obj == "reg:pseudohubererror":   # h = 1 / (s sqrt(s)) before the weight
        with np.errstate(all="ignore"):
            sd = F(1.0) + ((p - y) / a) * ((p - y) / a)
            hu = np.abs(np.float64(1.0) / (sd.astype(np.float64) * np.sqrt(sd).astype(np.float64)))
        return (hu > 0) & (hu < TINY)
    else:
        return np.zeros(len(p), bool)
    with np.errstate(all="ignore"):
        v = [np.abs(R.expf_(x)) for x in args]
        if obj == "reg:gamma":
            v.append(np.abs(y.astype(np.float64) / v[0]))
        if obj == "reg:tweedie":
            v.append(np.abs(y * (F(1.0) - a)))
            v.append(np.where(a == F(1.0), F(0.0), np.abs(y)))
    return np.any([(x > 0) & (x < TINY) for x in v], axis=0)


def ulp(x):
    """A binary32 ulp at magnitude x, in float64 (x may exceed FLT_MAX: a scale sums several terms)."""
    return np.maximum(np.ldexp(1.0, np.frexp(np.abs(x))[1] - 24), SUB)


@pytest.mark.parametrize("case", all_cases(), ids=case_id)
def test_restatement_within_ulp_bound_of_float64(case):
    params, weighted = case
    obj = params["objective"]
    p, y, w = edge_grid(params, weighted)
    g, h, bad = R.gradients(params, p, y, w)
    rg, rh, gs, hs = float64_pairs(params, p, y, w)
    # the pseudo-Huber square overflows in binary32 for |z / huber_slope| > 1.8e19 while float64 keeps it: s = inf,
    # so g = z / inf = +-0 and h = 0 -- exact, finite, and not the float64 pair
    with np.errstate(all="ignore"):
        if obj == "reg:pseudohubererror":
            zd = (p - y) / R.objective_param(params)
            sq_over = ~(np.abs(zd * zd) <= FMAX) & np.isfinite(p - y)
            assert sq_over.any() or params["huber_slope"] > 1, "the grid must reach the overflowing square"
            assert np.all(g[sq_over] == 0) and np.all(h[sq_over] == 0)
            # a residual p - y that overflows binary32 (float64 keeps it) is a pair that is not finite: (0, 0), counted
            z_over = ~np.isfinite(p - y)
            assert z_over.any() and np.all(g[z_over] == 0) and np.all(h[z_over] == 0)
            sq_over |= z_over
            # s sqrt(s) overflows for |z / huber_slope| > 6.9e12: h = 1 / inf = 0 exactly, g stays held to the bound
            sd = F(1.0) + zd * zd
            h_over = ~(np.abs(sd * np.sqrt(sd)) <= FMAX) & ~sq_over
            assert np.all(h[h_over] == 0)
        else:
            sq_over = h_over = np.zeros(len(p), bool)
    # the kernels weight the pair last (after scale_pos_weight has scaled the weight): the unweighted pair must be
    # finite too
    ug, uh, _, _ = float64_pairs(dict(params, scale_pos_weight=1.0), p, y, None)
    band = FMAX * (1 + 2.0 ** -20)
    with np.errstate(invalid="ignore"):
        over = ~((np.abs(rg) <= band) & (np.abs(rh) <= band) & (np.abs(ug) <= band) & (np.abs(uh) <= band))   # NaN too
        fin64 = np.all([np.abs(v) <= FMAX * (1 - 2.0 ** -20) for v in (rg, rh, ug, uh)], axis=0)
    if obj in R.CHECKS_FINITE:
        zeroed = (g == 0) & (h == 0)
        assert np.all(zeroed[over & ~sq_over]), "a pair that overflows in float64 must come out as (0, 0)"
        assert bad >= np.count_nonzero(over & ~sq_over)
        assert bad <= np.count_nonzero(~fin64 | sq_over | short_of_bits(params, p, y)), "a finite float64 pair was flagged"
    else:
        assert bad == 0 and np.isfinite(g).all() and np.isfinite(h).all()
    ok = fin64 & ~sq_over & ~short_of_bits(params, p, y)
    assert ok.sum() >= len(p) // 10, "the grid is held to the bound"
    for got, want, scale, name, skip in ((g, rg, gs, "g", sq_over), (h, rh, hs, "h", h_over)):
        normal = ok & ~skip & ((want == 0) | (np.abs(want) >= TINY))
        err = np.abs(got[normal].astype(np.float64) - want[normal]) / ulp(scale[normal])
        i = int(np.argmax(err)) if err.size else 0
        assert err.size == 0 or err.max() <= ULP_BOUND, (
            name, err.max(), p[normal][i], y[normal][i], None if w is None else w[normal][i])


def test_grids_reach_the_edges():
    """The grids contain the rows the kernels' branches are about."""
    p, y, w = edge_grid({"objective": "binary:logistic", "scale_pos_weight": 1e30}, True)
    assert np.any(y == 1.0) and np.any(y == F(0.99999994)) and np.any(y == F(1.0000001))
    g, h, _ = R.gradients({"objective": "binary:logistic"}, p, y, w)
    assert np.any(h == F(1e-16))                                        # the hessian floor
    p, y, w = edge_grid({"objective": "reg:gamma"}, True)
    assert R.gradients({"objective": "reg:gamma"}, p, y, w)[2] > 0      # exp flushed to zero, and 1e30 weights
    p, y, w = edge_grid({"objective": "reg:squaredlogerror", "scale_pos_weight": 1.0}, False)
    assert np.any(p < F(-1.0) + F(1e-6)) and np.any(y == F(-0.99999994))
    g, h, _ = R.gradients({"objective": "reg:squaredlogerror"}, p, y)
    assert np.any(h == F(1e-6))                                         # the hessian floor
    for mds in (0.0, 0.7):
        params = {"objective": "count:poisson", "max_delta_step": mds}
        s = margins_for(params) + F(mds)
        assert np.any(s == F(88.7)) and np.any(s > F(88.7)) and np.any(s < F(88.7))
    for rho in f32(1.0 + 2.0 ** -23, 1.5, 2.0 - 2.0 ** -23):
        params = {"objective": "reg:tweedie", "tweedie_variance_power": rho}
        for c in (F(1.0) - F(rho), F(2.0) - F(rho)):
            s = c * margins_for(params)
            assert np.any(s > F(88.7)) and np.any(s < F(-103.0)) and np.any((s >= F(88.6)) & (s <= F(88.7)))


def test_weight_overflow_is_zeroed_and_counted():
    """A 1e30 weight pushes every objective that checks finiteness into the zero-and-flag path: rows whose unweighted
    pair is finite and whose weighted pair is not come out as (0, 0) and are counted."""
    for obj in R.CHECKS_FINITE:
        n_over = 0
        for params in param_sets(obj):
            params = dict(params, objective=obj)
            p, y, w = edge_grid(params, True)
            g, h, bad = R.gradients(params, p, y, w)
            big = w == F(1e30)
            gu, hu, bu = R.gradients(params, p[big], y[big])
            with np.errstate(all="ignore"):
                over = ~((np.abs(gu.astype(np.float64) * 1e30) <= FMAX) & (np.abs(hu.astype(np.float64) * 1e30) <= FMAX))
            assert np.all(g[big][over] == 0) and np.all(h[big][over] == 0)
            assert bad >= over.sum() + bu
            n_over += over.sum()
        assert n_over > 0, obj


def test_scale_pos_weight_only_on_label_one():
    """scale_pos_weight multiplies the weight of y == 1.0f exactly, not of its neighbours."""
    y = np.array([1.0, 0.99999994, 1.0000001, 0.0], F)
    p = np.zeros(4, F)
    for obj in ("binary:logistic", "reg:logistic", "binary:logitraw", "reg:squaredlogerror"):
        yy = y if obj != "reg:logistic" and obj != "binary:logitraw" else np.minimum(y, F(1.0))
        g1, h1, _ = R.gradients({"objective": obj}, p, yy)
        g2, h2, _ = R.gradients({"objective": obj, "scale_pos_weight": 4.0}, p, yy)
        one = yy == F(1.0)
        assert np.array_equal(g2[one], g1[one] * F(4)) and np.array_equal(h2[one], h1[one] * F(4))
        assert np.array_equal(g2[~one], g1[~one]) and np.array_equal(h2[~one], h1[~one])


def test_squared_error_is_the_weighted_residual():
    p, y, w = edge_grid({"objective": "reg:squarederror"}, True)
    g, h, bad = R.gradients({"objective": "reg:squarederror"}, p, y, w)
    assert bad == 0
    assert np.array_equal(g.view(np.uint32), ((p - y) * w).astype(F).view(np.uint32))
    assert np.array_equal(h.view(np.uint32), w.view(np.uint32))
    g2, h2, _ = R.gradients({"objective": "reg:linear"}, p, y, w)
    assert np.array_equal(g2.view(np.uint32), g.view(np.uint32)) and np.array_equal(h2.view(np.uint32), h.view(np.uint32))


@pytest.mark.parametrize("obj", ["reg:squarederror", "binary:logistic", "reg:pseudohubererror", "reg:squaredlogerror"])
def test_multi_target_form_is_per_column(obj):
    """gradients_multi_target lays column k's single-target pairs out as row k of [T][n]."""
    params = {"objective": obj}
    p, y, w = edge_grid(params, True)
    n, T = len(p), 5
    M = np.stack([np.roll(p, 3 * k) for k in range(T)], axis=1)
    Y = np.stack([np.roll(y, 3 * k) for k in range(T)], axis=1)
    g, h, bad = R.gradients_multi_target(params, M, Y, w)
    assert g.shape == (T, n) and h.shape == (T, n)
    total = 0
    for k in range(T):
        gk, hk, b = R.gradients(params, M[:, k], Y[:, k], w)
        assert np.array_equal(g[k].view(np.uint32), gk.view(np.uint32)) and np.array_equal(h[k].view(np.uint32), hk.view(np.uint32))
        total += b
    assert bad == total


@pytest.mark.parametrize("obj", ["reg:squarederror", "reg:linear", "binary:logistic", "reg:pseudohubererror"])
@pytest.mark.parametrize("bad_label", [np.nan, np.inf, -np.inf])
def test_nonfinite_labels_are_refused_by_the_reference(oracle, obj, bad_label):
    rng = np.random.RandomState(1)
    X = rng.uniform(size=(200, 3)).astype(F)
    y = np.full(200, 0.5, F)
    y[17] = bad_label
    with pytest.raises(ValueError, match="label must be finite for " + obj):
        R.train(oracle, {"objective": obj}, X, y, 1)
    y[17] = 0.5
    R.train(oracle, {"objective": obj}, X, y, 1)
