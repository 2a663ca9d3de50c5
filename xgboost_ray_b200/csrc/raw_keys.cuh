// raw_keys.cuh -- how the sketch reads a raw value: the missing-value rule and the order-preserving uint32 key of a float.
// Shared by the dense key extraction and binning (sketch.cu) and the CSR key extraction (sparse_kernel.cu), so that a
// CSR matrix and its dense twin give the sketch the same keys.
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

}  // namespace b2
