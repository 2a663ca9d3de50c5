"""Reference for survival:aft (accelerated failure time with censored label bounds): a binary64 NumPy restatement of
its gradients, loss, limits, label checks and metrics (DESIGN.md 4.4), and a trainer that grows trees with the CPU
oracle (oracle/hist_oracle.c) from those gradients through its custom-gradient path.

TEST INFRASTRUCTURE ONLY, like the oracle.  The gradients replay the binary64 sequence of objective_kernel.cu
(gradient_aft_kernel) operation for operation: NumPy's float64 +, -, *, / round correctly and never fuse, and exp, log
and erf are fdlibm's published algorithms (e_exp.c, e_log.c, s_erf.c) restated on float64 arrays, with the bit
handling done through `.view(np.uint64)`.  So gradients, and with them the trees, are bit-equal to the engine's.
"""
import numpy as np

from tests import objective_reference as OR

D = np.float64
F = np.float32
DISTRIBUTIONS = ("normal", "logistic", "extreme")
K_EPS = 1e-12
G_MIN, G_MAX = -15.0, 15.0
H_MIN, H_MAX = 1e-16, 15.0
INV_SQRT_2PI = 0.3989422804014327     # 1 / sqrt(2 pi), 0x3FD9884533D43651
SQRT1_2 = 0.7071067811865476          # 1 / sqrt(2), 0x3FE6A09E667F3BCD


def _bits(x):
    return np.ascontiguousarray(x, D).view(np.uint64)


def _dbl(u):
    return np.ascontiguousarray(u, np.uint64).view(D)


def _hi(x):
    """fdlibm's __HI: the high 32 bits as a signed int."""
    h = (_bits(x) >> np.uint64(32)).astype(np.int64)
    return np.where(h >= 2 ** 31, h - 2 ** 32, h)


def _add_exponent(y, k):
    """__HI(y) += k << 20 on every element."""
    return _dbl((_bits(y).astype(np.int64) + (np.asarray(k, np.int64) << 52)).astype(np.uint64))


# ------------------------------------------------------------------------------------------------ fdlibm, binary64
_LN2_HI, _LN2_LO = 6.93147180369123816490e-01, 1.90821492927058770002e-10
_INVLN2 = 1.44269504088896338700e+00
_O_THR, _U_THR = 7.09782712893383973096e+02, -7.45133219101941108420e+02
_TWOM1000 = 9.33263618503218878990e-302
_P = (1.66666666666666019037e-01, -2.77777777770155933842e-03, 6.61375632143793436117e-05,
      -1.65339022054652515390e-06, 4.13813679705723846039e-08)


def exp_(x):
    """fdlibm __ieee754_exp (e_exp.c)."""
    x = np.asarray(x, D)
    with np.errstate(all="ignore"):
        hx = _hi(x)
        xsb = (hx >> 31) & 1
        ahx = hx & 0x7fffffff
        xs = np.where(np.isfinite(x) & (np.abs(x) < 746.0), x, 0.0)
        mid = (ahx > 0x3fd62e42) & (ahx < 0x3FF0A2B2)
        far = ahx >= 0x3FF0A2B2
        tiny = ahx < 0x3e300000
        # |x| in (0.5 ln2, 1.5 ln2): k = +-1
        sgn = np.where(xsb == 0, 1.0, -1.0)
        hi_mid = xs - sgn * _LN2_HI
        lo_mid = sgn * _LN2_LO
        k_far = np.trunc(_INVLN2 * xs + np.where(xsb == 0, 0.5, -0.5)).astype(np.int64)
        t = k_far.astype(D)
        hi_far = xs - t * _LN2_HI
        lo_far = t * _LN2_LO
        k = np.where(mid, 1 - 2 * xsb, np.where(far, k_far, 0))
        hi = np.where(mid, hi_mid, hi_far)
        lo = np.where(mid, lo_mid, lo_far)
        r = np.where(k != 0, hi - lo, xs)
        t = r * r
        c = r - t * (_P[0] + t * (_P[1] + t * (_P[2] + t * (_P[3] + t * _P[4]))))
        y0 = 1.0 - ((r * c) / (c - 2.0) - r)
        y = 1.0 - ((lo - (r * c) / (2.0 - c)) - hi)
        ynorm = _add_exponent(y, k)
        ysub = _add_exponent(y, k + 1000) * _TWOM1000
        out = np.where(k == 0, y0, np.where(k >= -1021, ynorm, ysub))
        out = np.where(tiny, 1.0 + xs, out)
        out = np.where(x > _O_THR, np.inf, out)
        out = np.where(x < _U_THR, 0.0, out)
        out = np.where(np.isnan(x), x + x, out)
    return out


_LG = (6.666666666666735130e-01, 3.999999999940941908e-01, 2.857142874366239149e-01, 2.222219843214978396e-01,
       1.818357216161805012e-01, 1.531383769920937332e-01, 1.479819860511658591e-01)
_TWO54 = 1.80143985094819840000e+16


def log_(x):
    """fdlibm __ieee754_log (e_log.c)."""
    x = np.asarray(x, D)
    with np.errstate(all="ignore"):
        hx = _hi(x)
        sub = (hx < 0x00100000) & (x > 0)
        xs = np.where(sub, x * _TWO54, np.where(np.isfinite(x) & (x > 0), x, 1.0))
        k = np.where(sub, -54, 0)
        hx = _hi(xs)
        k = k + (hx >> 20) - 1023
        hx = hx & 0x000fffff
        i = (hx + 0x95f64) & 0x100000
        lo_bits = _bits(xs) & np.uint64(0xffffffff)
        xs = _dbl(((hx | (i ^ 0x3ff00000)).astype(np.uint64) << np.uint64(32)) | lo_bits)
        k = k + (i >> 20)
        f = xs - 1.0
        dk = k.astype(D)
        # |f| < 2^-20
        small = (0x000fffff & (2 + hx)) < 3
        Rs = f * f * (0.5 - 0.33333333333333333 * f)
        v_small = np.where(f == 0.0, np.where(k == 0, 0.0, dk * _LN2_HI + dk * _LN2_LO),
                           np.where(k == 0, f - Rs, dk * _LN2_HI - ((Rs - dk * _LN2_LO) - f)))
        s = f / (2.0 + f)
        z = s * s
        ii = hx - 0x6147a
        w = z * z
        j = 0x6b851 - hx
        t1 = w * (_LG[1] + w * (_LG[3] + w * _LG[5]))
        t2 = z * (_LG[0] + w * (_LG[2] + w * (_LG[4] + w * _LG[6])))
        ii = ii | j
        R = t2 + t1
        hfsq = 0.5 * f * f
        v_a = np.where(k == 0, f - (hfsq - s * (hfsq + R)), dk * _LN2_HI - ((hfsq - (s * (hfsq + R) + dk * _LN2_LO)) - f))
        v_b = np.where(k == 0, f - s * (f - R), dk * _LN2_HI - ((s * (f - R) - dk * _LN2_LO) - f))
        out = np.where(small, v_small, np.where(ii > 0, v_a, v_b))
        out = np.where(x == 0.0, -np.inf, out)
        out = np.where(x < 0.0, np.nan, out)
        out = np.where(~np.isfinite(x) & ~(x < 0.0), x + x, out)
    return out


_ERX = 8.45062911510467529297e-01
_EFX, _EFX8 = 1.28379167095512586316e-01, 1.02703333676410069053e+00
_PP = (1.28379167095512558561e-01, -3.25042107247001499370e-01, -2.84817495755985104766e-02,
       -5.77027029648944159157e-03, -2.37630166566501626084e-05)
_QQ = (3.97917223959155352819e-01, 6.50222499887672944485e-02, 5.08130628187576562776e-03,
       1.32494738004321644526e-04, -3.96022827877536812320e-06)
_PA = (-2.36211856075265944077e-03, 4.14856118683748331666e-01, -3.72207876035701323847e-01,
       3.18346619901161753674e-01, -1.10894694282396677476e-01, 3.54783043256182359371e-02,
       -2.16637559486879084300e-03)
_QA = (1.06420880400844228286e-01, 5.40397917702171048937e-01, 7.18286544141962662868e-02,
       1.26171219808761642112e-01, 1.36370839120290507362e-02, 1.19844998467991074170e-02)
_RA = (-9.86494403484714822705e-03, -6.93858572707181764372e-01, -1.05586262253232909814e+01,
       -6.23753324503260060396e+01, -1.62396669462573470355e+02, -1.84605092906711035994e+02,
       -8.12874355063065934246e+01, -9.81432934416914548592e+00)
_SA = (1.96512716674392571292e+01, 1.37657754143519042600e+02, 4.34565877475229228821e+02,
       6.45387271733267880336e+02, 4.29008140027567833386e+02, 1.08635005541779435134e+02,
       6.57024977031928170135e+00, -6.04244152148580987438e-02)
_RB = (-9.86494292470009928597e-03, -7.99283237680523006574e-01, -1.77579549177547519889e+01,
       -1.60636384855821916062e+02, -6.37566443368389627722e+02, -1.02509513161107724954e+03,
       -4.83519191608651397019e+02)
_SB = (3.03380607434824582924e+01, 3.25792512996573918826e+02, 1.53672958608443695994e+03,
       3.19985821950859553908e+03, 2.55305040643316442583e+03, 4.74528541206955367215e+02,
       -2.24409524465858183362e+01)


def erf_(x):
    """fdlibm erf (s_erf.c)."""
    x = np.asarray(x, D)
    with np.errstate(all="ignore"):
        hx = _hi(x)
        ix = hx & 0x7fffffff
        neg = hx < 0
        # |x| < 0.84375
        z = x * x
        r = _PP[0] + z * (_PP[1] + z * (_PP[2] + z * (_PP[3] + z * _PP[4])))
        s = 1.0 + z * (_QQ[0] + z * (_QQ[1] + z * (_QQ[2] + z * (_QQ[3] + z * _QQ[4]))))
        v0 = x + x * (r / s)
        v0 = np.where(ix < 0x3e300000, np.where(ix < 0x00800000, 0.125 * (8.0 * x + _EFX8 * x), x + _EFX * x), v0)
        # 0.84375 <= |x| < 1.25
        s = np.abs(x) - 1.0
        P = _PA[0] + s * (_PA[1] + s * (_PA[2] + s * (_PA[3] + s * (_PA[4] + s * (_PA[5] + s * _PA[6])))))
        Q = 1.0 + s * (_QA[0] + s * (_QA[1] + s * (_QA[2] + s * (_QA[3] + s * (_QA[4] + s * _QA[5])))))
        v1 = np.where(neg, -_ERX - P / Q, _ERX + P / Q)
        # 1.25 <= |x| < 6
        ax = np.abs(x)
        s = 1.0 / (ax * ax)
        Ra = _RA[0] + s * (_RA[1] + s * (_RA[2] + s * (_RA[3] + s * (_RA[4] + s * (_RA[5] + s * (_RA[6] + s * _RA[7]))))))
        Sa = 1.0 + s * (_SA[0] + s * (_SA[1] + s * (_SA[2] + s * (_SA[3] + s * (_SA[4] + s * (_SA[5] + s * (
            _SA[6] + s * _SA[7])))))))
        Rb = _RB[0] + s * (_RB[1] + s * (_RB[2] + s * (_RB[3] + s * (_RB[4] + s * (_RB[5] + s * _RB[6])))))
        Sb = 1.0 + s * (_SB[0] + s * (_SB[1] + s * (_SB[2] + s * (_SB[3] + s * (_SB[4] + s * (_SB[5] + s * _SB[6]))))))
        lo_a = ix < 0x4006DB6E
        R = np.where(lo_a, Ra, Rb)
        S = np.where(lo_a, Sa, Sb)
        zz = _dbl(_bits(ax) & np.uint64(0xffffffff00000000))
        rr = exp_(-zz * zz - 0.5625) * exp_((zz - ax) * (zz + ax) + R / S)
        v2 = np.where(neg, rr / ax - 1.0, 1.0 - rr / ax)
        v3 = np.where(neg, 1e-300 - 1.0, 1.0 - 1e-300)
        out = np.where(ix < 0x3feb0000, v0, np.where(ix < 0x3ff40000, v1, np.where(ix < 0x40180000, v2, v3)))
        out = np.where(ix >= 0x7ff00000, np.where(np.isnan(x), x + x, np.where(neg, -1.0, 1.0)), out)
    return out


# ------------------------------------------------------------------------------------------------ AFT distributions
def density(dist, z):
    """(pdf, cdf, pdf', pdf'') of the standardised distribution at z (arrays), the kernel's aft_density<D>."""
    z = np.asarray(z, D)
    with np.errstate(all="ignore"):
        if dist == "normal":
            pdf = exp_(((-z) * z) * 0.5) * INV_SQRT_2PI
            cdf = 0.5 * (1.0 + erf_(z * SQRT1_2))
            return pdf, cdf, (-z) * pdf, (z * z - 1.0) * pdf
        w = exp_(z)
        w2 = w * w
        inf_w = np.isinf(w)
        inf_w2 = inf_w | np.isinf(w2)
        if dist == "logistic":
            opw = 1.0 + w
            pdf = np.where(inf_w2, 0.0, w / (opw * opw))
            cdf = np.where(inf_w, 1.0, w / opw)
            dpdf = np.where(inf_w, 0.0, (pdf * (1.0 - w)) / opw)
            d2pdf = np.where(inf_w2, 0.0, (pdf * ((w2 - 4.0 * w) + 1.0)) / (opw * opw))
            return pdf, cdf, dpdf, d2pdf
        if dist == "extreme":
            ew = exp_(-w)
            pdf = np.where(inf_w, 0.0, w * ew)
            cdf = 1.0 - ew
            dpdf = np.where(inf_w, 0.0, (1.0 - w) * pdf)
            d2pdf = np.where(inf_w2, 0.0, ((w2 - 3.0 * w) + 1.0) * pdf)
            return pdf, cdf, dpdf, d2pdf
    raise ValueError("aft_loss_distribution must be normal, logistic or extreme, got %r" % (dist,))


def limit_grad(dist, z_sign, sigma):
    """g as the margin goes to -inf (z_sign) or +inf (not z_sign)."""
    if dist == "normal":
        return np.where(z_sign, G_MIN, G_MAX)
    if dist == "logistic":
        return np.where(z_sign, -1.0 / sigma, 1.0 / sigma)
    return np.where(z_sign, G_MIN, 1.0 / sigma)


def limit_hess(dist, z_sign, sigma):
    if dist == "normal":
        return np.full(np.shape(z_sign), 1.0 / (sigma * sigma))
    if dist == "logistic":
        return np.full(np.shape(z_sign), H_MIN)
    return np.where(z_sign, H_MAX, H_MIN)


def _clip(v, lo, hi):
    return np.where(v < lo, lo, np.where(v > hi, hi, v))


def sigma_of(params):
    return float(F(params.get("aft_loss_distribution_scale", 1.0)))


def dist_of(params):
    return params.get("aft_loss_distribution", "normal")


def _sides(dist, margin, lower, upper, sigma, exact_margin=False):
    """Per-row pieces shared by the loss and the gradient: uncensored mask, z, z_sign and the densities.  The engine's
    margins are binary32; exact_margin keeps a binary64 margin as it is (finite differences)."""
    m = np.asarray(margin, D) if exact_margin else np.asarray(margin, F).astype(D)
    lo = np.asarray(lower, F).astype(D)
    up = np.asarray(upper, F).astype(D)
    with np.errstate(all="ignore"):
        unc = lo == up
        has_u = ~np.isinf(up)
        has_l = lo > 0.0
        z_u = np.where(has_u, (log_(np.where(has_u, up, 1.0)) - m) / sigma, 0.0)
        z_l = np.where(has_l, (log_(np.where(has_l, lo, 1.0)) - m) / sigma, 0.0)
        fu, Fu, gu, hu = density(dist, z_u)
        fl, Fl, gl, hl = density(dist, z_l)
        fu, Fu, gu = np.where(has_u, fu, 0.0), np.where(has_u, Fu, 1.0), np.where(has_u, gu, 0.0)
        fl, Fl, gl = np.where(has_l, fl, 0.0), np.where(has_l, Fl, 0.0), np.where(has_l, gl, 0.0)
    return dict(unc=unc, lo=lo, z=z_l, z_sign=np.where(unc, z_l > 0.0, (z_u > 0.0) | (z_l > 0.0)),
                f=fl, fp=gl, fpp=hl, dF=Fu - Fl, df=fu - fl, dg=gu - gl)


def grad_hess64(dist, margin, lower, upper, sigma):
    """Binary64 (g, h) of every row before the weight: limits and clips applied, the kernel's sequence."""
    s = _sides(dist, margin, lower, upper, sigma)
    with np.errstate(all="ignore"):
        f, fp, fpp = s["f"], s["fp"], s["fpp"]
        g_num = np.where(s["unc"], fp, s["df"])
        g_den = np.where(s["unc"], sigma * f, sigma * s["dF"])
        sd = sigma * s["dF"]
        h_num = np.where(s["unc"], -(f * fpp - fp * fp), -(s["dF"] * s["dg"] - s["df"] * s["df"]))
        h_den = np.where(s["unc"], (sigma * sigma) * (f * f), sd * sd)
        g = g_num / g_den
        h = h_num / h_den
        g = np.where((g_den < K_EPS) & ~np.isfinite(g), limit_grad(dist, s["z_sign"], sigma), g)
        h = np.where((h_den < K_EPS) & ~np.isfinite(h), limit_hess(dist, s["z_sign"], sigma), h)
    return _clip(g, G_MIN, G_MAX), _clip(h, H_MIN, H_MAX)


def gradients(params, margin, lower, upper, weight=None):
    """(g, h, number of non-finite rows) in binary32: binary64 (g, h) times the weight, rounded once."""
    g, h = grad_hess64(dist_of(params), margin, lower, upper, sigma_of(params))
    w = np.ones(len(g), D) if weight is None else np.asarray(weight, F).astype(D)
    g, h = (g * w).astype(F), (h * w).astype(F)
    bad = ~(np.isfinite(g) & np.isfinite(h))
    g[bad] = 0.0
    h[bad] = 0.0
    return g, h, int(bad.sum())


def loss(dist, margin, lower, upper, sigma, exact_margin=False):
    """Per-row negative log-likelihood in binary64."""
    s = _sides(dist, margin, lower, upper, sigma, exact_margin)
    with np.errstate(all="ignore"):
        v_unc = -log_(np.maximum(s["f"] / (sigma * s["lo"]), K_EPS))
        v_cen = -log_(np.maximum(s["dF"], K_EPS))
    return np.where(s["unc"], v_unc, v_cen)


def check_bounds(lower, upper, n):
    """The engine's label check of survival:aft; raises ValueError with its message."""
    if lower is None or upper is None or len(lower) != n or len(upper) != n:
        raise ValueError("survival:aft needs label_lower_bound and label_upper_bound")
    lo, up = np.asarray(lower, F), np.asarray(upper, F)
    if np.any(np.isnan(lo) | np.isnan(up)):
        raise ValueError("label bounds must not be NaN")
    if np.any(~(lo >= 0) | np.isinf(lo)):
        raise ValueError("label_lower_bound must be finite and >= 0")
    if np.any(up < lo):
        raise ValueError("label_upper_bound must be >= label_lower_bound")
    if np.any((lo == up) & (lo <= 0)):
        raise ValueError("an uncensored row (lower == upper) needs a label > 0")


def metric(name, params, margin, lower, upper, weight=None):
    """aft-nloglik / interval-regression-accuracy: weighted means with float64 sums."""
    w = np.ones(len(lower), D) if weight is None else np.asarray(weight, F).astype(D)
    if name == "aft-nloglik":
        v = loss(dist_of(params), margin, lower, upper, sigma_of(params))
    elif name == "interval-regression-accuracy":
        p = exp_(np.asarray(margin, F).astype(D))
        v = ((np.asarray(lower, F).astype(D) <= p) & (p <= np.asarray(upper, F).astype(D))).astype(D)
    else:
        raise KeyError(name)
    return float(np.sum(v * w) / np.sum(w))


def base_margin(params):
    """logf(base_score) on the host, like the log-link objectives; base_score defaults to 0.5 and is never estimated."""
    return OR.base_margin("count:poisson", params.get("base_score", 0.5))


class Model(OR.Model):
    def predict(self, X):
        return OR.expf_(self.predict_margin(X))

    def metric(self, name, margin, lower, upper, weight=None):
        return metric(name, self.params, margin, lower, upper, weight)


def train(oracle, params, X, lower, upper, rounds, weight=None, is_cat=None, base_margin_rows=None):
    """Trees of `rounds` rounds: the oracle's tree growth fed with this module's gradients through its custom-gradient
    path, like objective_reference.train."""
    X = np.ascontiguousarray(X, F)
    check_bounds(lower, upper, X.shape[0])
    if dist_of(params) not in DISTRIBUTIONS:
        raise ValueError("aft_loss_distribution must be normal, logistic or extreme")
    if not sigma_of(params) > 0:
        raise ValueError("aft_loss_distribution_scale must be > 0")
    b = float(F(params.get("base_score", 0.5)))
    oparams = {k: v for k, v in params.items() if k not in ("objective", "base_score", "eval_metric",
                                                             "aft_loss_distribution", "aft_loss_distribution_scale")}
    oparams.update(objective="reg:squarederror", base_score=base_margin(params))
    cuts = oracle.Cuts.from_data(X, int(params.get("max_bin", 256)), np.nan, is_cat=is_cat, weight=weight)
    bins = cuts.bin(X)
    bst = oracle.Booster(oparams, cuts)
    bst.init_margin(X.shape[0], base_margin_rows)
    y = np.zeros(X.shape[0], F)
    for _ in range(rounds):
        g, h, bad = gradients(params, bst.margin[:, 0], lower, upper, weight)
        if bad:
            raise FloatingPointError("survival:aft: a gradient or hessian is not finite")
        bst.boost(bins, y, weight, custom_g=g, custom_h=h)
    return Model(dict(params, objective="survival:aft"), bst, b)
