// raw_keys.cuh -- how the sketch reads a raw value: the missing-value rule and the order-preserving uint32 key of a float.
// Shared by the dense key extraction and binning (sketch.cu) and the CSR entry keys (sparse_kernel.cu), so that a CSR
// matrix and its dense twin give the sketch the same keys and categorical statistics.
#pragma once
#include <stdint.h>

namespace b2 {

__device__ __forceinline__ uint32_t f2key(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) {
  uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(u);
}
__device__ __forceinline__ bool is_missing(float x, float missing, int missing_is_nan) {
  return isnan(x) || (!missing_is_nan && x == missing);
}
// the sketch key of a non-missing value: -0 and +0 are one value
__device__ __forceinline__ uint32_t sketch_key(float x) {
  if (x == 0.0f) x = 0.0f;
  return f2key(x);
}

// Categorical columns (HistogramCuts::AddCategories, src/common/quantile.cc): the cuts are the codes 0..max, so the
// only statistics needed are the largest code, whether a value is missing and which values are not valid codes.
// stats [n_cat][3] int32 = {max code (init -1), has_missing, largest invalid value (init INT_MIN) as the signed
// order-preserving key f2key(x) ^ 0x80000000, so the error can name it}; merged with an allreduce(max).  x is one value
// of categorical feature ci.
__device__ __forceinline__ void cat_stats_update(float x, float missing, int missing_is_nan, int32_t* stats, int ci) {
  if (is_missing(x, missing, missing_is_nan)) { if (stats[ci * 3 + 1] == 0) atomicMax(&stats[ci * 3 + 1], 1); return; }
  if (!(x >= 0.0f) || x > 255.0f || x != (float)(int)x) {
    atomicMax(&stats[ci * 3 + 2], (int32_t)(f2key(x) ^ 0x80000000u));
    return;
  }
  const int c = (int)x;
  if (stats[ci * 3] < c) atomicMax(&stats[ci * 3], c);
}

}  // namespace b2
