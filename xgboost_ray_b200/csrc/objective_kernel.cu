// objective_kernel.cu -- objective gradients, fixed-point quantisation, metrics, tree traversal.
//
// Replaces the objective / metric / predictor stages that the reference reaches through
// xgb.train() and Booster.predict() (xgboost_ray/main.py:745-752, 804; SURVEY.md 8a rows a9, a14;
// Appendix A.4, A.9, A.10).  Compiled with --fmad=false: b2_expf (objective_common.cuh) and b2_log1pf below are fixed sequences
// of IEEE-754 binary32 operations, replayed identically on the host by the test references (the CPU oracle,
// tests/objective_reference.py), so gradients are bit-equal.
#include <cfloat>
#include <cmath>
#include "common.cuh"
#include "sampling.cuh"
#include "objective_common.cuh"

namespace b2 {

// log1p as a fixed binary32 sequence (tests/objective_reference.py replays it): the classic fdlibm reduction.  1+x = 2^k (1+f)
// with sqrt(2)/2 <= 1+f < sqrt(2), c corrects the rounding of 1+x, and log(1+f) = f - f^2/2 + s (f^2/2 + R(s^2)) with
// s = f / (2+f), with fdlibm's polynomial coefficients Lg1..Lg4 (about 1 ulp on (-1, inf)).
__device__ __forceinline__ float b2_log1pf(float x) {
  const uint32_t ix = __float_as_uint(x);
  if (!(x > -1.0f)) return x == -1.0f ? -INFINITY : NAN;
  if (x == INFINITY) return x;
  if ((ix & 0x7fffffffu) < 0x33800000u) return x;   // |x| < 2^-24: log1p(x) = x within half an ulp
  const float ln2_hi = __uint_as_float(0x3f317180u), ln2_lo = __uint_as_float(0x3717f7d1u);
  const float Lg1 = __uint_as_float(0x3f2aaaaau), Lg2 = __uint_as_float(0x3ecccce1u);
  const float Lg3 = __uint_as_float(0x3e91e9eeu), Lg4 = __uint_as_float(0x3e789e26u);
  int k = 1;
  float f = x, c = 0.0f;
  if (ix < 0x3ed413d0u || (ix >> 31)) {               // 1+x < sqrt(2)
    if (ix <= 0xbe95f619u) k = 0;                      // sqrt(2)/2 <= 1+x: no reduction
  }
  if (k) {
    const float u = __fadd_rn(1.0f, x);
    uint32_t iu = __float_as_uint(u) + (0x3f800000u - 0x3f3504f3u);
    k = (int)(iu >> 23) - 0x7f;
    if (k < 25) {
      c = k >= 2 ? __fadd_rn(1.0f, -__fadd_rn(u, -x)) : __fadd_rn(x, -__fadd_rn(u, -1.0f));
      c = __fdiv_rn(c, u);
    }
    iu = (iu & 0x007fffffu) + 0x3f3504f3u;
    f = __fadd_rn(__uint_as_float(iu), -1.0f);
  }
  const float s = __fdiv_rn(f, __fadd_rn(2.0f, f));
  const float z = __fmul_rn(s, s), w = __fmul_rn(z, z);
  const float t1 = __fmul_rn(w, __fadd_rn(Lg2, __fmul_rn(w, Lg4)));
  const float t2 = __fmul_rn(z, __fadd_rn(Lg1, __fmul_rn(w, Lg3)));
  const float R = __fadd_rn(t2, t1);
  const float hfsq = __fmul_rn(__fmul_rn(0.5f, f), f);
  const float dk = (float)k;
  float r = __fadd_rn(__fadd_rn(__fmul_rn(dk, ln2_lo), -hfsq), f);
  r = __fadd_rn(r, c);
  r = __fadd_rn(__fmul_rn(s, __fadd_rn(hfsq, R)), r);
  return __fadd_rn(r, __fmul_rn(dk, ln2_hi));
}

__device__ double b2_erf(double x) {
  const int hx = __double2hiint(x), ix = hx & 0x7fffffff;
  if (ix >= 0x7ff00000) return x != x ? B2_DA(x, x) : (hx < 0 ? -1.0 : 1.0);
  if (ix < 0x3feb0000) {                                  // |x| < 0.84375
    if (ix < 0x3e300000) {                                // |x| < 2^-28
      if (ix < 0x00800000) return B2_DM(0.125, B2_DA(B2_DM(8.0, x), B2_DM(1.02703333676410069053e+00, x)));
      return B2_DA(x, B2_DM(1.28379167095512586316e-01, x));
    }
    const double z = B2_DM(x, x);
    const double r = B2_DA(1.28379167095512558561e-01, B2_DM(z, B2_DA(-3.25042107247001499370e-01, B2_DM(z,
                     B2_DA(-2.84817495755985104766e-02, B2_DM(z, B2_DA(-5.77027029648944159157e-03,
                     B2_DM(z, -2.37630166566501626084e-05))))))));
    const double s = B2_DA(1.0, B2_DM(z, B2_DA(3.97917223959155352819e-01, B2_DM(z, B2_DA(6.50222499887672944485e-02,
                     B2_DM(z, B2_DA(5.08130628187576562776e-03, B2_DM(z, B2_DA(1.32494738004321644526e-04,
                     B2_DM(z, -3.96022827877536812320e-06))))))))));
    return B2_DA(x, B2_DM(x, B2_DD(r, s)));
  }
  if (ix < 0x3ff40000) {                                  // 0.84375 <= |x| < 1.25
    const double s = B2_DS(fabs(x), 1.0);
    const double P = B2_DA(-2.36211856075265944077e-03, B2_DM(s, B2_DA(4.14856118683748331666e-01, B2_DM(s,
                     B2_DA(-3.72207876035701323847e-01, B2_DM(s, B2_DA(3.18346619901161753674e-01, B2_DM(s,
                     B2_DA(-1.10894694282396677476e-01, B2_DM(s, B2_DA(3.54783043256182359371e-02,
                     B2_DM(s, -2.16637559486879084300e-03))))))))))));
    const double Q = B2_DA(1.0, B2_DM(s, B2_DA(1.06420880400844228286e-01, B2_DM(s, B2_DA(5.40397917702171048937e-01,
                     B2_DM(s, B2_DA(7.18286544141962662868e-02, B2_DM(s, B2_DA(1.26171219808761642112e-01,
                     B2_DM(s, B2_DA(1.36370839120290507362e-02, B2_DM(s, 1.19844998467991074170e-02))))))))))));
    const double erx = 8.45062911510467529297e-01;
    return hx >= 0 ? B2_DA(erx, B2_DD(P, Q)) : B2_DS(-erx, B2_DD(P, Q));
  }
  if (ix >= 0x40180000) return hx >= 0 ? B2_DS(1.0, 1e-300) : B2_DS(1e-300, 1.0);   // |x| >= 6
  const double ax = fabs(x), s = B2_DD(1.0, B2_DM(ax, ax));
  double R, S;
  if (ix < 0x4006DB6E) {                                  // |x| < 1/0.35
    R = B2_DA(-9.86494403484714822705e-03, B2_DM(s, B2_DA(-6.93858572707181764372e-01, B2_DM(s,
        B2_DA(-1.05586262253232909814e+01, B2_DM(s, B2_DA(-6.23753324503260060396e+01, B2_DM(s,
        B2_DA(-1.62396669462573470355e+02, B2_DM(s, B2_DA(-1.84605092906711035994e+02, B2_DM(s,
        B2_DA(-8.12874355063065934246e+01, B2_DM(s, -9.81432934416914548592e+00))))))))))))));
    S = B2_DA(1.0, B2_DM(s, B2_DA(1.96512716674392571292e+01, B2_DM(s, B2_DA(1.37657754143519042600e+02, B2_DM(s,
        B2_DA(4.34565877475229228821e+02, B2_DM(s, B2_DA(6.45387271733267880336e+02, B2_DM(s,
        B2_DA(4.29008140027567833386e+02, B2_DM(s, B2_DA(1.08635005541779435134e+02, B2_DM(s,
        B2_DA(6.57024977031928170135e+00, B2_DM(s, -6.04244152148580987438e-02))))))))))))))));
  } else {
    R = B2_DA(-9.86494292470009928597e-03, B2_DM(s, B2_DA(-7.99283237680523006574e-01, B2_DM(s,
        B2_DA(-1.77579549177547519889e+01, B2_DM(s, B2_DA(-1.60636384855821916062e+02, B2_DM(s,
        B2_DA(-6.37566443368389627722e+02, B2_DM(s, B2_DA(-1.02509513161107724954e+03,
        B2_DM(s, -4.83519191608651397019e+02))))))))))));
    S = B2_DA(1.0, B2_DM(s, B2_DA(3.03380607434824582924e+01, B2_DM(s, B2_DA(3.25792512996573918826e+02, B2_DM(s,
        B2_DA(1.53672958608443695994e+03, B2_DM(s, B2_DA(3.19985821950859553908e+03, B2_DM(s,
        B2_DA(2.55305040643316442583e+03, B2_DM(s, B2_DA(4.74528541206955367215e+02,
        B2_DM(s, -2.24409524465858183362e+01))))))))))))));
  }
  const double z = __hiloint2double(__double2hiint(ax), 0);
  const double r = B2_DM(b2_exp(B2_DS(B2_DM(-z, z), 0.5625)), b2_exp(B2_DA(B2_DM(B2_DS(z, ax), B2_DA(z, ax)), B2_DD(R, S))));
  return hx >= 0 ? B2_DS(1.0, B2_DD(r, ax)) : B2_DS(B2_DD(r, ax), 1.0);
}

// objective ids (engine.cu kObj*): 0 reg:squarederror, 1 binary:logistic, 2 multi:softprob, 3 reg:logistic,
// 4 binary:logitraw, 5 reg:squaredlogerror, 6 reg:pseudohubererror, 7 count:poisson, 8 reg:gamma, 9 reg:tweedie,
// 10 survival:aft
constexpr int kObjRegLogistic = 3, kObjLogitRaw = 4, kObjSquaredLog = 5, kObjPseudoHuber = 6, kObjPoisson = 7,
              kObjGamma = 8, kObjTweedie = 9, kObjAft = 10;
// the parameter of an objective that has one: huber_slope, max_delta_step (Poisson hessian), tweedie_variance_power
struct ObjParam { float a; };

// margin -> prediction of one scalar output (ObjFunction::PredTransform): sigmoid, exp or identity
__device__ __forceinline__ float b2_pred_transform(int objective, float m) {
  if (objective == 1 || objective == kObjRegLogistic) return b2_sigmoid(m);
  if (objective == kObjPoisson || objective == kObjGamma || objective == kObjTweedie || objective == kObjAft) return b2_expf(m);
  return m;
}

// (g, h) of one row before the weight, for the objectives added after the first three (the same IEEE sequence as
// tests/objective_reference.py::gradients); `a` is the objective's parameter
template <int kObjective>
__device__ __forceinline__ float2 scalar_grad(float p, float y, float a) {
  if (kObjective == kObjSquaredLog) {
    const float kMin = -1.0f + 1e-6f;
    const float q = p < kMin ? kMin : p;
    const float lq = b2_log1pf(q), ly = b2_log1pf(y), q1 = __fadd_rn(q, 1.0f);
    const float g = __fdiv_rn(__fadd_rn(lq, -ly), q1);
    float h = __fdiv_rn(__fadd_rn(__fadd_rn(-lq, ly), 1.0f), __fmul_rn(q1, q1));
    if (h < 1e-6f) h = 1e-6f;
    return make_float2(g, h);
  } else if (kObjective == kObjPseudoHuber) {
    const float z = __fadd_rn(p, -y), zd = __fdiv_rn(z, a);
    const float s = __fadd_rn(1.0f, __fmul_rn(zd, zd)), sq = __fsqrt_rn(s);
    return make_float2(__fdiv_rn(z, sq), __fdiv_rn(1.0f, __fmul_rn(s, sq)));
  } else if (kObjective == kObjPoisson) {
    return make_float2(__fadd_rn(b2_expf(p), -y), b2_expf(__fadd_rn(p, a)));
  } else if (kObjective == kObjGamma) {
    const float r = __fdiv_rn(y, b2_expf(p));
    return make_float2(__fadd_rn(1.0f, -r), r);
  } else {   // kObjTweedie, a = rho
    const float e1 = b2_expf(__fmul_rn(__fadd_rn(1.0f, -a), p)), e2 = b2_expf(__fmul_rn(__fadd_rn(2.0f, -a), p));
    const float g = __fadd_rn(-__fmul_rn(y, e1), e2);
    const float h = __fadd_rn(__fmul_rn(__fmul_rn(-y, __fadd_rn(1.0f, -a)), e1), __fmul_rn(__fadd_rn(2.0f, -a), e2));
    return make_float2(g, h);
  }
}

// gh layout: class-major [K][n] float2 so that each class tree reads a contiguous slice.
// absmax (nullable, [K][2] uint32 float bit patterns, zeroed by the caller): max |g|, max |h| per class, gathered in
// the same pass (the fixed-point scale of each class tree needs it; a separate pass re-read 8 bytes per row).
constexpr int kFusedMaxK = 16;   // classes whose running maxima fit in registers; more classes use absmax_kernel

// scalar objectives (reg:squarederror, binary:logistic and its variants): their own kernel so that the register budget
// of the softprob path (2 x 16 running maxima) does not cut the occupancy of this streaming loop (72 registers -> 3 blocks
// per SM made the 10M-row launch take 63 us instead of ~25)
template <int kObjective>
__global__ void __launch_bounds__(256)
gradient_scalar_kernel(const float* __restrict__ margin, const float* __restrict__ label, const float* __restrict__ weight,
                       int64_t n, float scale_pos_weight, float2* __restrict__ gh, uint32_t* __restrict__ absmax) {
  float mg = 0.0f, mh = 0.0f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float w = weight ? weight[i] : 1.0f;
    const float y = label[i], m = margin[i];
    float2 v;
    if (kObjective == 0) {
      v = make_float2(__fmul_rn(__fadd_rn(m, -y), w), w);
    } else {
      if (y == 1.0f) w = __fmul_rn(w, scale_pos_weight);   // RegLossObj: positive rows
      const float p = b2_sigmoid(m);
      float hh = __fmul_rn(p, __fadd_rn(1.0f, -p));
      if (hh < 1e-16f) hh = 1e-16f;
      v = make_float2(__fmul_rn(__fadd_rn(p, -y), w), __fmul_rn(hh, w));
    }
    gh[i] = v;
    mg = fmaxf(mg, fabsf(v.x)); mh = fmaxf(mh, fabsf(v.y));
  }
  if (absmax) absmax_publish(mg, mh, absmax);
}

// the objectives whose gradient can leave the finite range (exp, division by exp): a row with a non-finite g or h is
// written as (0, 0), so that the quantisation scale and the tree of this round stay finite, and raises *err (zeroed by
// the caller, read at the end of the round), which fails the round before its trees join the model
template <int kObjective>
__global__ void __launch_bounds__(256)
gradient_param_kernel(const float* __restrict__ margin, const float* __restrict__ label, const float* __restrict__ weight,
                      int64_t n, float scale_pos_weight, ObjParam op, float2* __restrict__ gh, uint32_t* __restrict__ absmax,
                      uint32_t* __restrict__ err) {
  float mg = 0.0f, mh = 0.0f;
  bool bad = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float w = weight ? weight[i] : 1.0f;
    const float y = label[i], m = margin[i];
    if (kObjective == kObjSquaredLog && y == 1.0f) w = __fmul_rn(w, scale_pos_weight);   // RegLossObj: positive rows
    const float2 r = scalar_grad<kObjective>(m, y, op.a);
    float2 v = make_float2(__fmul_rn(r.x, w), __fmul_rn(r.y, w));
    if (!(fabsf(v.x) <= FLT_MAX && fabsf(v.y) <= FLT_MAX)) { bad = true; v = make_float2(0.0f, 0.0f); }
    gh[i] = v;
    mg = fmaxf(mg, fabsf(v.x)); mh = fmaxf(mh, fabsf(v.y));
  }
  if (bad && err) atomicOr(err, 1u);
  if (absmax) absmax_publish(mg, mh, absmax);
}

// ---- survival:aft (accelerated failure time).  log y = margin + sigma Z with Z standard normal, logistic or extreme
// (Gumbel-min); a row gives a bound pair [lower, upper]: lower == upper is an exact time, upper = +inf right-censored,
// lower = 0 left-censored, otherwise interval-censored.  With z = (log y - margin) / sigma, f the pdf and F the CDF of Z:
//   uncensored  loss -log(max(f(z) / (sigma y), kEps)),   g = f'/(sigma f),   h = -(f'' f - f'^2) / (sigma^2 f^2)
//   censored    loss -log(max(F(z_u) - F(z_l), kEps)),   g = (f_u - f_l) / (sigma dF),
//               h = ((f_u - f_l)^2 - (f'_u - f'_l) dF) / (sigma^2 dF^2)
// in binary64 (tests/survival_reference.py replays the sequence).  A quotient that is not finite while its denominator
// is below kEps takes its limit as the margin goes to -inf (z > 0; z_u > 0 or z_l > 0 for censored rows) or +inf; then
// g is clipped to [-15, 15] and h to [1e-16, 15].
constexpr int kAftNormal = 0, kAftLogistic = 1, kAftExtreme = 2;
constexpr double kAftEps = 1e-12;
struct AftDensity { double pdf, cdf, dpdf, d2pdf; };

template <int kDist>
__device__ __forceinline__ AftDensity aft_density(double z) {
  AftDensity d;
  if (kDist == kAftNormal) {
    d.pdf = B2_DM(b2_exp(B2_DM(B2_DM(-z, z), 0.5)), 0.3989422804014327);     // 1 / sqrt(2 pi)
    d.cdf = B2_DM(0.5, B2_DA(1.0, b2_erf(B2_DM(z, 0.7071067811865476))));   // erf(z / sqrt(2))
    d.dpdf = B2_DM(-z, d.pdf);
    d.d2pdf = B2_DM(B2_DS(B2_DM(z, z), 1.0), d.pdf);
  } else {
    const double w = b2_exp(z), w2 = B2_DM(w, w);
    const bool inf_w = isinf(w), inf_w2 = inf_w || isinf(w2);
    if (kDist == kAftLogistic) {
      const double opw = B2_DA(1.0, w);
      d.pdf = inf_w2 ? 0.0 : B2_DD(w, B2_DM(opw, opw));
      d.cdf = inf_w ? 1.0 : B2_DD(w, opw);
      d.dpdf = inf_w ? 0.0 : B2_DD(B2_DM(d.pdf, B2_DS(1.0, w)), opw);
      d.d2pdf = inf_w2 ? 0.0 : B2_DD(B2_DM(d.pdf, B2_DA(B2_DS(w2, B2_DM(4.0, w)), 1.0)), B2_DM(opw, opw));
    } else {
      const double ew = b2_exp(-w);
      d.pdf = inf_w ? 0.0 : B2_DM(w, ew);
      d.cdf = B2_DS(1.0, ew);
      d.dpdf = inf_w ? 0.0 : B2_DM(B2_DS(1.0, w), d.pdf);
      d.d2pdf = inf_w2 ? 0.0 : B2_DM(B2_DA(B2_DS(w2, B2_DM(3.0, w)), 1.0), d.pdf);
    }
  }
  return d;
}

template <int kDist>
__device__ __forceinline__ double aft_limit_grad(bool z_sign, double sigma) {
  if (kDist == kAftNormal) return z_sign ? -15.0 : 15.0;
  if (kDist == kAftLogistic) return z_sign ? B2_DD(-1.0, sigma) : B2_DD(1.0, sigma);
  return z_sign ? -15.0 : B2_DD(1.0, sigma);
}
template <int kDist>
__device__ __forceinline__ double aft_limit_hess(bool z_sign, double sigma) {
  if (kDist == kAftNormal) return B2_DD(1.0, B2_DM(sigma, sigma));
  if (kDist == kAftLogistic) return 1e-16;
  return z_sign ? 15.0 : 1e-16;
}

// the pieces of one row that the loss and the gradient share
struct AftRow {
  bool unc, z_sign;
  double f, fp, fpp;       // uncensored: density, f', f'' at z
  double dF, df, dg;       // censored: F_u - F_l, f_u - f_l, f'_u - f'_l
};
template <int kDist>
__device__ __forceinline__ AftRow aft_row(double m, float lower, float upper, double sigma) {
  AftRow r;
  r.unc = lower == upper;
  if (r.unc) {
    const double z = B2_DD(B2_DS(b2_log((double)lower), m), sigma);
    const AftDensity d = aft_density<kDist>(z);
    r.z_sign = z > 0.0; r.f = d.pdf; r.fp = d.dpdf; r.fpp = d.d2pdf;
    r.dF = r.df = r.dg = 0.0;
  } else {
    double z_u = 0.0, z_l = 0.0, f_u = 0.0, F_u = 1.0, g_u = 0.0, f_l = 0.0, F_l = 0.0, g_l = 0.0;
    if (!isinf(upper)) {
      z_u = B2_DD(B2_DS(b2_log((double)upper), m), sigma);
      const AftDensity d = aft_density<kDist>(z_u);
      f_u = d.pdf; F_u = d.cdf; g_u = d.dpdf;
    }
    if (lower > 0.0f) {
      z_l = B2_DD(B2_DS(b2_log((double)lower), m), sigma);
      const AftDensity d = aft_density<kDist>(z_l);
      f_l = d.pdf; F_l = d.cdf; g_l = d.dpdf;
    }
    r.z_sign = z_u > 0.0 || z_l > 0.0;
    r.dF = B2_DS(F_u, F_l); r.df = B2_DS(f_u, f_l); r.dg = B2_DS(g_u, g_l);
    r.f = r.fp = r.fpp = 0.0;
  }
  return r;
}

template <int kDist>
__device__ __forceinline__ double aft_loss(double m, float lower, float upper, double sigma) {
  const AftRow r = aft_row<kDist>(m, lower, upper, sigma);
  if (r.unc) return -b2_log(fmax(B2_DD(r.f, B2_DM(sigma, (double)lower)), kAftEps));
  return -b2_log(fmax(r.dF, kAftEps));
}

// gradient pairs of survival:aft, one instantiation per distribution; weight applied in binary64, rounded once.  A row
// whose pair is not finite (a NaN margin) is written as (0, 0) and raises *err, like gradient_param_kernel.
template <int kDist>
__global__ void __launch_bounds__(256)
gradient_aft_kernel(const float* __restrict__ margin, const float* __restrict__ lower, const float* __restrict__ upper,
                    const float* __restrict__ weight, int64_t n, double sigma, float2* __restrict__ gh,
                    uint32_t* __restrict__ absmax, uint32_t* __restrict__ err) {
  float mg = 0.0f, mh = 0.0f;
  bool bad = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const AftRow r = aft_row<kDist>((double)margin[i], lower[i], upper[i], sigma);
    double g_num, g_den, h_num, h_den;
    if (r.unc) {
      g_num = r.fp; g_den = B2_DM(sigma, r.f);
      h_num = -B2_DS(B2_DM(r.f, r.fpp), B2_DM(r.fp, r.fp)); h_den = B2_DM(B2_DM(sigma, sigma), B2_DM(r.f, r.f));
    } else {
      const double sd = B2_DM(sigma, r.dF);
      g_num = r.df; g_den = sd;
      h_num = -B2_DS(B2_DM(r.dF, r.dg), B2_DM(r.df, r.df)); h_den = B2_DM(sd, sd);
    }
    double g = B2_DD(g_num, g_den), h = B2_DD(h_num, h_den);
    if (g_den < kAftEps && !isfinite(g)) g = aft_limit_grad<kDist>(r.z_sign, sigma);
    if (h_den < kAftEps && !isfinite(h)) h = aft_limit_hess<kDist>(r.z_sign, sigma);
    g = g < -15.0 ? -15.0 : (g > 15.0 ? 15.0 : g);
    h = h < 1e-16 ? 1e-16 : (h > 15.0 ? 15.0 : h);
    const double w = weight ? (double)weight[i] : 1.0;
    float2 v = make_float2(__double2float_rn(B2_DM(g, w)), __double2float_rn(B2_DM(h, w)));
    if (!(fabsf(v.x) <= FLT_MAX && fabsf(v.y) <= FLT_MAX)) { bad = true; v = make_float2(0.0f, 0.0f); }
    gh[i] = v;
    mg = fmaxf(mg, fabsf(v.x)); mh = fmaxf(mh, fabsf(v.y));
  }
  if (bad && err) atomicOr(err, 1u);
  if (absmax) absmax_publish(mg, mh, absmax);
}

// label bounds of survival:aft (once per train matrix): bad[0] a NaN bound, bad[1] lower < 0 or not finite,
// bad[2] upper < lower, bad[3] an uncensored row with y <= 0 (max-reduced over the workers, so one word per rule)
__global__ void aft_bounds_check_kernel(const float* __restrict__ lower, const float* __restrict__ upper, int64_t n,
                                        uint32_t* __restrict__ bad) {
  bool b0 = false, b1 = false, b2 = false, b3 = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float lo = lower[i], up = upper[i];
    b0 |= lo != lo || up != up;
    b1 |= !(lo >= 0.0f) || isinf(lo);
    b2 |= up < lo;
    b3 |= lo == up && lo <= 0.0f;
  }
  if (__any_sync(0xffffffffu, b0) && (threadIdx.x & 31) == 0) atomicOr(&bad[0], 1u);
  if (__any_sync(0xffffffffu, b1) && (threadIdx.x & 31) == 0) atomicOr(&bad[1], 1u);
  if (__any_sync(0xffffffffu, b2) && (threadIdx.x & 31) == 0) atomicOr(&bad[2], 1u);
  if (__any_sync(0xffffffffu, b3) && (threadIdx.x & 31) == 0) atomicOr(&bad[3], 1u);
}

// aft-nloglik (metric 14) and interval-regression-accuracy (metric 15): (sum w v, sum w) in double
template <int kDist>
__device__ __forceinline__ double aft_metric_value(int metric, float m, float lower, float upper, double sigma) {
  if (metric == 14) return aft_loss<kDist>((double)m, lower, upper, sigma);
  const double p = b2_exp((double)m);
  return ((double)lower <= p && p <= (double)upper) ? 1.0 : 0.0;
}
__global__ void aft_metric_kernel(int dist, int metric, double sigma, const float* __restrict__ margin,
                                  const float* __restrict__ lower, const float* __restrict__ upper,
                                  const float* __restrict__ weight, int64_t n, double* __restrict__ out) {
  double s = 0.0, ws = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double w = weight ? (double)weight[i] : 1.0;
    const double v = dist == kAftNormal ? aft_metric_value<kAftNormal>(metric, margin[i], lower[i], upper[i], sigma)
                   : dist == kAftLogistic ? aft_metric_value<kAftLogistic>(metric, margin[i], lower[i], upper[i], sigma)
                   : aft_metric_value<kAftExtreme>(metric, margin[i], lower[i], upper[i], sigma);
    s += v * w; ws += w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); ws += __shfl_xor_sync(0xffffffffu, ws, o); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(&out[0], s); atomicAdd(&out[1], ws); }
}

__global__ void gradient_softprob_kernel(int K, const float* __restrict__ margin, const float* __restrict__ label,
                                         const float* __restrict__ weight, int64_t n, float2* __restrict__ gh,
                                         uint32_t* __restrict__ absmax) {
  const bool fused = absmax != nullptr && K <= kFusedMaxK;
  float mg[kFusedMaxK], mh[kFusedMaxK];
#pragma unroll
  for (int k = 0; k < kFusedMaxK; ++k) { mg[k] = 0.0f; mh[k] = 0.0f; }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float w = weight ? weight[i] : 1.0f;
    const float* m = margin + i * K;
    float mx = m[0];
    for (int k = 1; k < K; ++k) if (m[k] > mx) mx = m[k];
    float s = 0.0f;
    for (int k = 0; k < K; ++k) s = __fadd_rn(s, b2_expf(__fadd_rn(m[k], -mx)));
    const int y = (int)label[i];
    if (fused) {
#pragma unroll
      for (int k = 0; k < kFusedMaxK; ++k) {
        if (k < K) {
          const float p = __fdiv_rn(b2_expf(__fadd_rn(m[k], -mx)), s);
          float hh = __fmul_rn(__fmul_rn(2.0f, p), __fadd_rn(1.0f, -p));
          if (hh < 1e-16f) hh = 1e-16f;
          const float g = (k == y) ? __fadd_rn(p, -1.0f) : p;
          const float2 v = make_float2(__fmul_rn(g, w), __fmul_rn(hh, w));
          gh[(int64_t)k * n + i] = v;
          mg[k] = fmaxf(mg[k], fabsf(v.x)); mh[k] = fmaxf(mh[k], fabsf(v.y));
        }
      }
    } else {
      for (int k = 0; k < K; ++k) {
        const float p = __fdiv_rn(b2_expf(__fadd_rn(m[k], -mx)), s);
        float hh = __fmul_rn(__fmul_rn(2.0f, p), __fadd_rn(1.0f, -p));
        if (hh < 1e-16f) hh = 1e-16f;
        const float g = (k == y) ? __fadd_rn(p, -1.0f) : p;
        gh[(int64_t)k * n + i] = make_float2(__fmul_rn(g, w), __fmul_rn(hh, w));
      }
    }
  }
  if (fused) {
#pragma unroll
    for (int k = 0; k < kFusedMaxK; ++k)
      if (k < K) absmax_publish(mg[k], mh[k], absmax + 2 * k);
  }
}

// row sampling (subsample < 1): rows whose hash falls above the threshold get a zero gradient pair for this tree
// (sampling.cuh); they stay in the row partition and still receive the leaf value.
__global__ void subsample_kernel(float2* __restrict__ gh, int64_t n, uint32_t seed, uint32_t tree, uint32_t rank, uint32_t thr) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (!(b2_hash4(seed, tree, rank, (uint32_t)i) < thr)) gh[i] = make_float2(0.0f, 0.0f);
}

// exact sums of one gradient-pair array in fixed point (bits relative to the quantisation exponents): int64 atomics
// of block partials, so the result does not depend on the order of rows, blocks or GPUs (base_score estimation)
__global__ void sum_fixed_kernel(const float2* __restrict__ gh, int64_t n, const int32_t* __restrict__ qexp, int bits,
                                 long long* __restrict__ out /*[2]*/) {
  const double kg = ldexp(1.0, bits - qexp[0]), kh = ldexp(1.0, bits - qexp[1]);
  long long ag = 0, ah = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float2 v = gh[i];
    ag += __double2ll_rn(__dmul_rn((double)v.x, kg));
    ah += __double2ll_rn(__dmul_rn((double)v.y, kh));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { ag += __shfl_xor_sync(0xffffffffu, ag, o); ah += __shfl_xor_sync(0xffffffffu, ah, o); }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd((unsigned long long*)&out[0], (unsigned long long)ag);
    atomicAdd((unsigned long long*)&out[1], (unsigned long long)ah);
  }
}

// interleave user-supplied gradients (custom objective): g,h row-major [n][K] -> gh [K][n]
__global__ void pack_custom_kernel(const float* __restrict__ g, const float* __restrict__ h, int K, int64_t n,
                                   float2* __restrict__ gh) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n * K; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / K; const int k = (int)(i % K);
    gh[(int64_t)k * n + row] = make_float2(g[i], h[i]);
  }
}

// absmax[0] = max|g|, absmax[1] = max|h| as float bit patterns (non-negative floats order as uints)
__global__ void absmax_kernel(const float2* __restrict__ gh, int64_t n, uint32_t* __restrict__ absmax) {
  float mg = 0.0f, mh = 0.0f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float2 v = gh[i];
    mg = fmaxf(mg, fabsf(v.x)); mh = fmaxf(mh, fabsf(v.y));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, o));
    mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMax(&absmax[0], __float_as_uint(mg));
    atomicMax(&absmax[1], __float_as_uint(mh));
  }
}

// exponent e with vmax < 2^e (frexp convention), q = rint(v * 2^(qbits - e))
__device__ __forceinline__ int frexp_exponent(uint32_t bits) {
  if (bits == 0) return 0;
  return (int)((bits >> 23) & 0xffu) - 126;
}
__global__ void quant_exponent_kernel(const uint32_t* __restrict__ absmax, int32_t* __restrict__ qexp) {
  if (threadIdx.x < 2) qexp[threadIdx.x] = frexp_exponent(absmax[threadIdx.x]);
}
__global__ void quantize_kernel(const float2* __restrict__ gh, int64_t n, const int32_t* __restrict__ qexp, int qbits,
                                int2* __restrict__ q) {
  const float sg = ldexpf(1.0f, qbits - qexp[0]), sh = ldexpf(1.0f, qbits - qexp[1]);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float2 v = gh[i];
    q[i] = make_int2((int)rintf(__fmul_rn(v.x, sg)), (int)rintf(__fmul_rn(v.y, sh)));
  }
}

// metric sums (sum loss*w, sum w, rows with an invalid class label) -> out[3] doubles.  Metrics see the TRANSFORMED prediction (ObjFunction::EvalTransform,
// src/learner.cc): the probability for binary:logistic / reg:logistic, exp(margin) for the log-link objectives, the raw
// value otherwise.  metric: 0 rmse, 1 logloss, 2 error, 3 mlogloss, 4 merror, 5 mae, 7 rmsle, 8 mape, 9 mphe (a = huber
// slope), 10 poisson-nloglik, 11 gamma-nloglik, 12 gamma-deviance, 13 tweedie-nloglik (a = rho); 6 (auc) is auc_kernel.cu.
// the elementwise metrics of the objectives added after the first three, on the transformed prediction q
__device__ __forceinline__ double scalar_metric(int metric, float a, double q, double y) {
  if (metric == 7) { const double d = log1p(y) - log1p(fmax(q, -1.0 + 1e-6)); return d * d; }
  if (metric == 8) return fabs((y - q) / y);
  if (metric == 9) { const double z = (y - q) / (double)a; return (double)a * (double)a * (sqrt(1.0 + z * z) - 1.0); }
  if (metric == 10) { const double qq = fmax(q, 1e-16); return lgamma(y + 1.0) + qq - y * log(qq); }
  if (metric == 11) return y / q + log(q);
  if (metric == 12) { const double qq = q + 1e-6, yy = y + 1e-6; return 2.0 * (log(qq / yy) + yy / qq - 1.0); }
  const double r = (double)a;
  return -y * pow(q, 1.0 - r) / (1.0 - r) + pow(q, 2.0 - r) / (2.0 - r);
}

// a multi-class label is a class index in [0, K): non-integer labels truncate (2.7 -> class 2); NaN is outside
__device__ __forceinline__ bool b2_class_label_ok(float y, int K) { return y >= 0.0f && y < (float)K; }

// out[2] counts the rows of mlogloss / merror whose label is not a class index: they add nothing to the sums (r[y] is
// never read for them) and the caller fails the evaluation
__global__ void metric_kernel(int objective, int metric, int K, float a, const float* __restrict__ margin,
                              const float* __restrict__ label, const float* __restrict__ weight, int64_t n,
                              double* __restrict__ out) {
  double s = 0.0, ws = 0.0;
  unsigned bad = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double w = weight ? (double)weight[i] : 1.0;
    double v = 0.0;
    if (metric <= 2 || metric == 5) {
      const float p = b2_pred_transform(objective, margin[i]);
      if (metric == 0) { const double d = (double)p - (double)label[i]; v = d * d; }
      else if (metric == 5) v = fabs((double)p - (double)label[i]);
      else if (metric == 1) {
        const float eps = 1e-16f; const float y = label[i];
        const float pn = 1.0f - p; const float a = p < eps ? eps : p, b = pn < eps ? eps : pn;
        v = -((double)y * log((double)a) + (1.0 - (double)y) * log((double)b));
      } else v = ((p > 0.5f) != (label[i] > 0.5f)) ? 1.0 : 0.0;
    }
    else if (metric >= 7) v = scalar_metric(metric, a, (double)b2_pred_transform(objective, margin[i]), (double)label[i]);
    else {
      const float yf = label[i];
      if (!b2_class_label_ok(yf, K)) { ++bad; continue; }
      const float* r = margin + i * K; const int y = (int)yf; float mx = r[0]; int am = 0;
      for (int k = 1; k < K; ++k) if (r[k] > mx) { mx = r[k]; am = k; }
      if (metric == 4) v = (am != y) ? 1.0 : 0.0;
      else {
        float ssum = 0.0f;
        for (int k = 0; k < K; ++k) ssum = __fadd_rn(ssum, b2_expf(__fadd_rn(r[k], -mx)));
        float p = __fdiv_rn(b2_expf(__fadd_rn(r[y], -mx)), ssum);
        if (p < 1e-16f) p = 1e-16f;
        v = -log((double)p);
      }
    }
    s += v * w; ws += w;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); ws += __shfl_xor_sync(0xffffffffu, ws, o); }
  bad = __reduce_add_sync(0xffffffffu, bad);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&out[0], s); atomicAdd(&out[1], ws);
    if (bad) atomicAdd(&out[2], (double)bad);
  }
}

// label domain of an objective (checked once per train matrix): *bad |= 1 when some label is outside it (NaN included);
// K is the class count of multi:softprob
__global__ void label_check_kernel(int objective, int K, const float* __restrict__ label, int64_t n, uint32_t* __restrict__ bad) {
  bool any = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float y = label[i];
    bool ok = true;
    if (objective == 2) ok = b2_class_label_ok(y, K);
    else if (objective == kObjRegLogistic || objective == kObjLogitRaw) ok = y >= 0.0f && y <= 1.0f;
    else if (objective == kObjSquaredLog) ok = y > -1.0f;
    else if (objective == kObjPoisson || objective == kObjTweedie) ok = y >= 0.0f;
    else if (objective == kObjGamma) ok = y > 0.0f;
    any |= !ok;
  }
  if (__any_sync(0xffffffffu, any) && (threadIdx.x & 31) == 0) atomicOr(bad, 1u);
}

// A.9 traversal on raw floats (the node step is b2_tree_step, common.cuh).  nodes of all trees are
// concatenated; tree_offset[t] is the first node of tree t; tree t adds to class (t / npt) % K (xgboost lays the
// num_parallel_tree trees of a class out next to each other, GBTree::BoostNewTrees).
__global__ void predict_kernel(const float* __restrict__ X, int64_t n, int F, float missing, int missing_is_nan,
                               const B2TreeNodeDev* __restrict__ nodes, const int32_t* __restrict__ tree_offset,
                               const uint32_t* __restrict__ cat_table, int tree_begin, int tree_end, int K, int npt,
                               float* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float* x = X + i * F;
    for (int t = tree_begin; t < tree_end; ++t) {
      float v;
      b2_tree_leaf(nodes + tree_offset[t], x, missing, missing_is_nan, cat_table, &v);
      out[i * K + ((t / npt) % K)] += v;
    }
  }
}

__global__ void fill_kernel(float* out, int64_t n, float v) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = v;
}

// margin -> prediction transform in place (sigmoid / exp / softmax)
__global__ void transform_kernel(int objective, int K, float* __restrict__ m, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (objective == 2) {
      float* r = m + i * K; float mx = r[0];
      for (int k = 1; k < K; ++k) if (r[k] > mx) mx = r[k];
      float s = 0.0f;
      for (int k = 0; k < K; ++k) { r[k] = b2_expf(__fadd_rn(r[k], -mx)); s = __fadd_rn(s, r[k]); }
      for (int k = 0; k < K; ++k) r[k] = __fdiv_rn(r[k], s);
    } else {
      m[i] = b2_pred_transform(objective, m[i]);
    }
  }
}

}  // namespace b2

static inline int grid_for(int64_t n, int num_sms) {
  int64_t g = (n + 255) / 256;
  int64_t cap = (int64_t)num_sms * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

extern "C" {
int b2_gradient_fused_max_classes() { return b2::kFusedMaxK; }
int b2_launch_gradient(int objective, int K, const float* margin, const float* label, const float* weight, int64_t n,
                       float scale_pos_weight, float obj_param, float2* gh, uint32_t* absmax, uint32_t* err, int num_sms,
                       cudaStream_t s) {
  if (n <= 0) return 0;
  const int g = grid_for(n, num_sms);
  const b2::ObjParam op{obj_param};
  switch (objective) {
    case 0: b2::gradient_scalar_kernel<0><<<g, 256, 0, s>>>(margin, label, weight, n, scale_pos_weight, gh, absmax); break;
    case 1: case b2::kObjRegLogistic: case b2::kObjLogitRaw:   // the logistic variants differ only in the transform
      b2::gradient_scalar_kernel<1><<<g, 256, 0, s>>>(margin, label, weight, n, scale_pos_weight, gh, absmax); break;
    case 2: b2::gradient_softprob_kernel<<<g, 256, 0, s>>>(K, margin, label, weight, n, gh, absmax); break;
#define B2_PARAM_OBJ(id) \
    case id: b2::gradient_param_kernel<id><<<g, 256, 0, s>>>(margin, label, weight, n, scale_pos_weight, op, gh, absmax, err); break;
    B2_PARAM_OBJ(b2::kObjSquaredLog) B2_PARAM_OBJ(b2::kObjPseudoHuber) B2_PARAM_OBJ(b2::kObjPoisson)
    B2_PARAM_OBJ(b2::kObjGamma) B2_PARAM_OBJ(b2::kObjTweedie)
#undef B2_PARAM_OBJ
    default: return (int)cudaErrorInvalidValue;
  }
  return (int)cudaGetLastError();
}
int b2_launch_gradient_aft(int dist, double sigma, const float* margin, const float* lower, const float* upper,
                           const float* weight, int64_t n, float2* gh, uint32_t* absmax, uint32_t* err, int num_sms,
                           cudaStream_t s) {
  if (n <= 0) return 0;
  const int g = grid_for(n, num_sms);
  switch (dist) {
#define B2_AFT(d) \
    case d: b2::gradient_aft_kernel<d><<<g, 256, 0, s>>>(margin, lower, upper, weight, n, sigma, gh, absmax, err); break;
    B2_AFT(b2::kAftNormal) B2_AFT(b2::kAftLogistic) B2_AFT(b2::kAftExtreme)
#undef B2_AFT
    default: return (int)cudaErrorInvalidValue;
  }
  return (int)cudaGetLastError();
}
int b2_launch_aft_bounds_check(const float* lower, const float* upper, int64_t n, uint32_t* bad, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::aft_bounds_check_kernel<<<grid_for(n, num_sms), 256, 0, s>>>(lower, upper, n, bad);
  return (int)cudaGetLastError();
}
int b2_launch_aft_metric(int dist, int metric, double sigma, const float* margin, const float* lower, const float* upper,
                         const float* weight, int64_t n, double* out, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::aft_metric_kernel<<<grid_for(n, num_sms), 256, 0, s>>>(dist, metric, sigma, margin, lower, upper, weight, n, out);
  return (int)cudaGetLastError();
}
int b2_launch_label_check(int objective, int K, const float* label, int64_t n, uint32_t* bad, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::label_check_kernel<<<grid_for(n, num_sms), 256, 0, s>>>(objective, K, label, n, bad);
  return (int)cudaGetLastError();
}
int b2_launch_subsample(float2* gh, int64_t n, uint32_t seed, uint32_t tree, uint32_t rank, double subsample, int num_sms,
                        cudaStream_t s) {
  if (n <= 0) return 0;
  b2::subsample_kernel<<<grid_for(n, num_sms), 256, 0, s>>>(gh, n, seed, tree, rank, b2_subsample_threshold(subsample));
  return (int)cudaGetLastError();
}
int b2_launch_sum_fixed(const float2* gh, int64_t n, const int32_t* qexp, int bits, long long* out, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::sum_fixed_kernel<<<grid_for(n, num_sms), 256, 0, s>>>(gh, n, qexp, bits, out);
  return (int)cudaGetLastError();
}
int b2_launch_pack_custom(const float* g, const float* h, int K, int64_t n, float2* gh, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::pack_custom_kernel<<<grid_for(n * K, num_sms), 256, 0, s>>>(g, h, K, n, gh);
  return (int)cudaGetLastError();
}
int b2_launch_absmax(const float2* gh, int64_t n, uint32_t* absmax, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::absmax_kernel<<<grid_for(n, num_sms), 256, 0, s>>>(gh, n, absmax);
  return (int)cudaGetLastError();
}
int b2_launch_quant_exponent(const uint32_t* absmax, int32_t* qexp, cudaStream_t s) {
  b2::quant_exponent_kernel<<<1, 32, 0, s>>>(absmax, qexp);
  return (int)cudaGetLastError();
}
int b2_launch_quantize(const float2* gh, int64_t n, const int32_t* qexp, int qbits, int2* q, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::quantize_kernel<<<grid_for(n, num_sms), 256, 0, s>>>(gh, n, qexp, qbits, q);
  return (int)cudaGetLastError();
}
int b2_launch_metric(int objective, int metric, int K, float metric_param, const float* margin, const float* label,
                     const float* weight, int64_t n, double* out, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::metric_kernel<<<grid_for(n, num_sms), 256, 0, s>>>(objective, metric, K, metric_param, margin, label, weight, n, out);
  return (int)cudaGetLastError();
}
int b2_launch_predict(const float* X, int64_t n, int F, float missing, const B2TreeNodeDev* nodes,
                      const int32_t* tree_offset, const uint32_t* cat_table, int tree_begin, int tree_end, int K, int npt,
                      float* out, int num_sms, cudaStream_t s) {
  if (n <= 0 || tree_end <= tree_begin) return 0;
  b2::predict_kernel<<<grid_for(n, num_sms), 256, 0, s>>>(X, n, F, missing, missing != missing ? 1 : 0, nodes, tree_offset,
                                                         cat_table, tree_begin, tree_end, K, npt < 1 ? 1 : npt, out);
  return (int)cudaGetLastError();
}
int b2_launch_fill(float* out, int64_t n, float v, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::fill_kernel<<<grid_for(n, num_sms), 256, 0, s>>>(out, n, v);
  return (int)cudaGetLastError();
}
int b2_launch_transform(int objective, int K, float* m, int64_t n, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::transform_kernel<<<grid_for(n, num_sms), 256, 0, s>>>(objective, K, m, n);
  return (int)cudaGetLastError();
}
}
