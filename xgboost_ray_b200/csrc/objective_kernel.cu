// objective_kernel.cu -- objective gradients, fixed-point quantisation, metrics, tree traversal.
//
// Replaces the objective / metric / predictor stages that the reference reaches through
// xgb.train() and Booster.predict() (xgboost_ray/main.py:745-752, 804; SURVEY.md 8a rows a9, a14;
// Appendix A.4, A.9, A.10).  Compiled with --fmad=false: b2_expf and b2_log1pf below are fixed sequences
// of IEEE-754 binary32 operations, replayed identically on the host by the test references (the CPU oracle,
// tests/objective_reference.py), so gradients are bit-equal.
#include <cfloat>
#include <cmath>
#include "common.cuh"
#include "sampling.cuh"

namespace b2 {

__device__ __forceinline__ float b2_expf(float x) {
  if (x > 88.7f) x = 88.7f;
  if (x < -103.0f) return 0.0f;
  const float log2e = 1.44269504088896341f;
  const float ln2_hi = 0.693359375f;
  const float ln2_lo = -2.12194440e-4f;
  float t = __fmul_rn(x, log2e);
  float n = rintf(t);
  float r = __fadd_rn(x, -__fmul_rn(n, ln2_hi));
  r = __fadd_rn(r, -__fmul_rn(n, ln2_lo));
  float p = 1.9875691500e-4f;
  p = __fadd_rn(__fmul_rn(p, r), 1.3981999507e-3f);
  p = __fadd_rn(__fmul_rn(p, r), 8.3334519073e-3f);
  p = __fadd_rn(__fmul_rn(p, r), 4.1665795894e-2f);
  p = __fadd_rn(__fmul_rn(p, r), 1.6666665459e-1f);
  p = __fadd_rn(__fmul_rn(p, r), 5.0000001201e-1f);
  float r2 = __fmul_rn(r, r);
  float e = __fadd_rn(__fmul_rn(p, r2), r);
  e = __fadd_rn(e, 1.0f);
  int ni = (int)n;
  int n1 = ni / 2, n2 = ni - n1;
  e = __fmul_rn(e, __uint_as_float((uint32_t)(n1 + 127) << 23));
  e = __fmul_rn(e, __uint_as_float((uint32_t)(n2 + 127) << 23));
  return e;
}
__device__ __forceinline__ float b2_sigmoid(float x) {
  float nx = -x;
  if (nx > 88.7f) nx = 88.7f;
  float denom = __fadd_rn(b2_expf(nx), 1.0f);
  denom = __fadd_rn(denom, 1e-16f);
  return __fdiv_rn(1.0f, denom);
}

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

// objective ids (engine.cu kObj*): 0 reg:squarederror, 1 binary:logistic, 2 multi:softprob, 3 reg:logistic,
// 4 binary:logitraw, 5 reg:squaredlogerror, 6 reg:pseudohubererror, 7 count:poisson, 8 reg:gamma, 9 reg:tweedie
constexpr int kObjRegLogistic = 3, kObjLogitRaw = 4, kObjSquaredLog = 5, kObjPseudoHuber = 6, kObjPoisson = 7,
              kObjGamma = 8, kObjTweedie = 9;
// the parameter of an objective that has one: huber_slope, max_delta_step (Poisson hessian), tweedie_variance_power
struct ObjParam { float a; };

// margin -> prediction of one scalar output (ObjFunction::PredTransform): sigmoid, exp or identity
__device__ __forceinline__ float b2_pred_transform(int objective, float m) {
  if (objective == 1 || objective == kObjRegLogistic) return b2_sigmoid(m);
  if (objective == kObjPoisson || objective == kObjGamma || objective == kObjTweedie) return b2_expf(m);
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

// block maxima -> two atomicMax per BLOCK (one per warp made 38K same-address atomics of a 10M-row launch cost more
// than the gradient arithmetic itself: 67 us against 23 us for the plain kernel)
__device__ __forceinline__ void absmax_publish(float mg, float mh, uint32_t* __restrict__ out) {
  __shared__ float s_mg[32], s_mh[32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, o));
    mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, o));
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = (blockDim.x + 31) >> 5;
  __syncthreads();                                   // the shared slots may still be read by the previous class
  if (lane == 0) { s_mg[warp] = mg; s_mh[warp] = mh; }
  __syncthreads();
  if (warp == 0) {
    mg = lane < n_warps ? s_mg[lane] : 0.0f; mh = lane < n_warps ? s_mh[lane] : 0.0f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mg = fmaxf(mg, __shfl_xor_sync(0xffffffffu, mg, o));
      mh = fmaxf(mh, __shfl_xor_sync(0xffffffffu, mh, o));
    }
    if (lane == 0) { atomicMax(&out[0], __float_as_uint(mg)); atomicMax(&out[1], __float_as_uint(mh)); }
  }
}

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

// metric sums (sum loss*w, sum w) -> out[2] doubles.  Metrics see the TRANSFORMED prediction (ObjFunction::EvalTransform,
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

__global__ void metric_kernel(int objective, int metric, int K, float a, const float* __restrict__ margin,
                              const float* __restrict__ label, const float* __restrict__ weight, int64_t n,
                              double* __restrict__ out) {
  double s = 0.0, ws = 0.0;
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
      const float* r = margin + i * K; const int y = (int)label[i]; float mx = r[0]; int am = 0;
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
  if ((threadIdx.x & 31) == 0) { atomicAdd(&out[0], s); atomicAdd(&out[1], ws); }
}

// label domain of an objective (checked once per train matrix): *bad |= 1 when some label is outside it (NaN included)
__global__ void label_check_kernel(int objective, const float* __restrict__ label, int64_t n, uint32_t* __restrict__ bad) {
  bool any = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float y = label[i];
    bool ok = true;
    if (objective == kObjRegLogistic || objective == kObjLogitRaw) ok = y >= 0.0f && y <= 1.0f;
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
int b2_launch_label_check(int objective, const float* label, int64_t n, uint32_t* bad, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::label_check_kernel<<<grid_for(n, num_sms), 256, 0, s>>>(objective, label, n, bad);
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
