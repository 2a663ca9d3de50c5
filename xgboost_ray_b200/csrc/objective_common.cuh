// objective_common.cuh -- what the objective and ranking gradient kernels share: the fixed IEEE-754 sequences of
// exp / sigmoid (binary32) and exp / log (binary64), and the block epilogue that publishes the |g|, |h| maxima.  Every
// file that includes it is compiled with --fmad=false, so each operation rounds once and the host references
// (tests/objective_reference.py, tests/survival_reference.py) replay the results bit for bit.
#pragma once
#include <cstdint>
#include <cmath>

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

// binary64 exp and log for survival:aft and the ranking objectives (erf: objective_kernel.cu): fdlibm's published
// algorithms (e_exp.c, e_log.c) written out in __dadd_rn / __dmul_rn / __ddiv_rn, so that tests/survival_reference.py
// replays them bit for bit (CUDA's own exp / log are not fixed sequences a host can repeat).  Both are within 1 ulp of
// the correctly rounded value.
#define B2_DA __dadd_rn
#define B2_DS(a, b) __dadd_rn(a, -(b))
#define B2_DM __dmul_rn
#define B2_DD __ddiv_rn
__device__ __forceinline__ double b2_add_exponent(double y, int k) {
  return __longlong_as_double(__double_as_longlong(y) + ((long long)k << 52));
}
__device__ __forceinline__ double b2_exp(double x) {
  const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10;
  const double P1 = 1.66666666666666019037e-01, P2 = -2.77777777770155933842e-03, P3 = 6.61375632143793436117e-05,
               P4 = -1.65339022054652515390e-06, P5 = 4.13813679705723846039e-08;
  const int hx0 = __double2hiint(x), xsb = (hx0 >> 31) & 1, hx = hx0 & 0x7fffffff;
  if (hx >= 0x40862E42) {                                 // |x| >= 709.78
    if (hx >= 0x7ff00000) return x != x ? B2_DA(x, x) : (xsb ? 0.0 : x);
    if (x > 7.09782712893383973096e+02) return INFINITY;
    if (x < -7.45133219101941108420e+02) return 0.0;
  }
  double hi = x, lo = 0.0;
  int k = 0;
  if (hx > 0x3fd62e42) {                                  // |x| > 0.5 ln2
    if (hx < 0x3FF0A2B2) {                                // and |x| < 1.5 ln2
      hi = xsb ? B2_DA(x, ln2_hi) : B2_DS(x, ln2_hi); lo = xsb ? -ln2_lo : ln2_lo; k = 1 - xsb - xsb;
    } else {
      k = (int)B2_DA(B2_DM(1.44269504088896338700e+00, x), xsb ? -0.5 : 0.5);
      const double t = (double)k;
      hi = B2_DS(x, B2_DM(t, ln2_hi)); lo = B2_DM(t, ln2_lo);
    }
    x = B2_DS(hi, lo);
  } else if (hx < 0x3e300000) {                           // |x| < 2^-28
    return B2_DA(1.0, x);
  }
  const double t = B2_DM(x, x);
  const double c = B2_DS(x, B2_DM(t, B2_DA(P1, B2_DM(t, B2_DA(P2, B2_DM(t, B2_DA(P3, B2_DM(t, B2_DA(P4, B2_DM(t, P5))))))))));
  if (k == 0) return B2_DS(1.0, B2_DS(B2_DD(B2_DM(x, c), B2_DS(c, 2.0)), x));
  const double y = B2_DS(1.0, B2_DS(B2_DS(lo, B2_DD(B2_DM(x, c), B2_DS(2.0, c))), hi));
  if (k >= -1021) return b2_add_exponent(y, k);
  return B2_DM(b2_add_exponent(y, k + 1000), 9.33263618503218878990e-302);
}
__device__ __forceinline__ double b2_log(double x) {
  const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10;
  const double Lg1 = 6.666666666666735130e-01, Lg2 = 3.999999999940941908e-01, Lg3 = 2.857142874366239149e-01,
               Lg4 = 2.222219843214978396e-01, Lg5 = 1.818357216161805012e-01, Lg6 = 1.531383769920937332e-01,
               Lg7 = 1.479819860511658591e-01;
  int hx = __double2hiint(x);
  const int lx = __double2loint(x);
  int k = 0;
  if (hx < 0x00100000) {                                  // x < 2^-1022
    if (((hx & 0x7fffffff) | lx) == 0) return -INFINITY;
    if (hx < 0) return NAN;
    k -= 54; x = B2_DM(x, 1.80143985094819840000e+16);   // subnormal: scale up
    hx = __double2hiint(x);
  }
  if (hx >= 0x7ff00000) return B2_DA(x, x);
  k += (hx >> 20) - 1023;
  hx &= 0x000fffff;
  int i = (hx + 0x95f64) & 0x100000;
  x = __hiloint2double(hx | (i ^ 0x3ff00000), __double2loint(x));   // normalise x or x/2
  k += i >> 20;
  const double f = B2_DS(x, 1.0), dk = (double)k;
  if ((0x000fffff & (2 + hx)) < 3) {                      // |f| < 2^-20
    if (f == 0.0) return k == 0 ? 0.0 : B2_DA(B2_DM(dk, ln2_hi), B2_DM(dk, ln2_lo));
    const double R = B2_DM(B2_DM(f, f), B2_DS(0.5, B2_DM(0.33333333333333333, f)));
    return k == 0 ? B2_DS(f, R) : B2_DS(B2_DM(dk, ln2_hi), B2_DS(B2_DS(R, B2_DM(dk, ln2_lo)), f));
  }
  const double s = B2_DD(f, B2_DA(2.0, f)), z = B2_DM(s, s), w = B2_DM(z, z);
  i = hx - 0x6147a;
  const int j = 0x6b851 - hx;
  const double t1 = B2_DM(w, B2_DA(Lg2, B2_DM(w, B2_DA(Lg4, B2_DM(w, Lg6)))));
  const double t2 = B2_DM(z, B2_DA(Lg1, B2_DM(w, B2_DA(Lg3, B2_DM(w, B2_DA(Lg5, B2_DM(w, Lg7)))))));
  i |= j;
  const double R = B2_DA(t2, t1);
  if (i > 0) {
    const double hfsq = B2_DM(B2_DM(0.5, f), f);
    if (k == 0) return B2_DS(f, B2_DS(hfsq, B2_DM(s, B2_DA(hfsq, R))));
    return B2_DS(B2_DM(dk, ln2_hi), B2_DS(B2_DS(hfsq, B2_DA(B2_DM(s, B2_DA(hfsq, R)), B2_DM(dk, ln2_lo))), f));
  }
  if (k == 0) return B2_DS(f, B2_DM(s, B2_DS(f, R)));
  return B2_DS(B2_DM(dk, ln2_hi), B2_DS(B2_DS(B2_DM(s, B2_DS(f, R)), B2_DM(dk, ln2_lo)), f));
}

// the |g|, |h| maxima of a gradient kernel's block, published to out[0], out[1] (float bit patterns, zeroed by the
// caller).  Block maxima -> two atomicMax per BLOCK (one per warp made 38K same-address atomics of a 10M-row launch
// cost more than the gradient arithmetic itself: 67 us against 23 us for the plain kernel)
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

}  // namespace b2
