// auc_kernel.cu -- ROC AUC (`auc`) and precision-recall AUC (`aucpr`) of one worker's rows, binary or one-vs-rest over
// the classes of a softmax model (SURVEY.md A.10; DESIGN.md §2 item 17).
//
// Restates xgboost's BinaryAUC / MultiClassOVR (src/metric/auc.cc): for each class the rows are sorted by descending
// prediction, positive / negative weights are accumulated, and the area is summed over the segments between
// consecutive DISTINCT prediction values (ties form one step): trapezoids for ROC, the Davis & Goadrich interpolation
// of precision over recall for PR.  Every worker contributes one triple per class -- ROC (area, fp_total * tp_total,
// tp_total), PR (aucpr or NaN, 1, 1) -- and the host combines the triples summed over the workers.  The sort is
// cub::DeviceRadixSort (library sort on a once-per-evaluation path); scans are cub primitives.  The per-block areas are
// summed in a fixed order by one CTA (no floating-point atomics), so a value is the same from call to call.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "launch.h"

namespace b2 {

__device__ __forceinline__ uint32_t desc_key(float v) {
  uint32_t u = __float_as_uint(v);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);   // ascending order-preserving key
  return ~u;                                        // descending
}

// keys of class c: pred is [n, K] row-major
__global__ void auc_keys_kernel(const float* __restrict__ pred, int K, int c, int64_t n, uint32_t* __restrict__ keys,
                                int32_t* __restrict__ idx) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    keys[i] = desc_key(pred[i * K + c]); idx[i] = (int32_t)i;
  }
}
// per sorted position: positive / negative weight and "last row of its tie group" marker.  K == 1: y is the label;
// K > 1: y = [label == c].  bad (nullable): += the rows whose label is not in [0, K)
__global__ void auc_weights_kernel(const uint32_t* __restrict__ keys, const int32_t* __restrict__ idx, const float* __restrict__ label,
                                   const float* __restrict__ weight, int64_t n, int K, int c, double* __restrict__ pos,
                                   double* __restrict__ neg, int32_t* __restrict__ end_mark, double* __restrict__ bad) {
  int nbad = 0;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    const int32_t i = idx[p];
    const float yf = label[i];
    const double w = weight ? (double)weight[i] : 1.0;
    const double y = K == 1 ? (double)yf : (yf == (float)c ? 1.0 : 0.0);
    nbad += !(yf >= 0.0f && yf < (float)K);
    pos[p] = y * w; neg[p] = (1.0 - y) * w;
    end_mark[p] = (p == n - 1 || keys[p] != keys[p + 1]) ? (int32_t)p : -1;
  }
  if (bad) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nbad += __shfl_xor_sync(0xffffffffu, nbad, o);
    if ((threadIdx.x & 31) == 0 && nbad) atomicAdd(bad, (double)nbad);   // integer counts: exact in any order
  }
}

// PR area of the segment (tp0, fp0) -> (tp1, fp1), P the total positive weight: the integral of the precision
// tp / (tp + fp) over the recall tp / P, fp linear in tp along the segment.  With d = tp1 - tp0, e = fp1 - fp0 this is
// DESIGN.md's (t1 - t0)/a - (b/a^2) ln((a t1 + b)/(a t0 + b)) with a = (d + e)/d, b P = (fp0 d - e tp0)/d and
// a t + b = (tp + fp)/P at both ends, written so that it stays finite when d is a rounding residue of the prefix sums
// (a tie group without positive weight can leave tp1 an ulp away from tp0)
__device__ __forceinline__ double pr_segment(double tp0, double fp0, double tp1, double fp1, double P) {
  const double d = tp1 - tp0, e = fp1 - fp0, s = d + e;
  if (!(d > 0.0) || !(s > 0.0)) return 0.0;
  const double c = fp0 * d - e * tp0;                  // b P d
  const double r = d / s;                              // 1/a
  if (c == 0.0) return r * d / P;                      // b = 0
  return r * (d - c / s * log1p(s / (tp0 + fp0))) / P;
}

// per-CTA sum of the segment areas of the tie groups ending in the CTA's positions; pr: 0 ROC (trapezoids), 1 PR
__global__ void auc_area_kernel(int pr, const double* __restrict__ tp, const double* __restrict__ fp, const int32_t* __restrict__ end_mark,
                                const int32_t* __restrict__ last_end /* inclusive max-scan of end_mark */, int64_t n,
                                double* __restrict__ partial /* [gridDim.x] */) {
  __shared__ double sh[32];
  const double P = tp[n - 1];
  double area = 0.0;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    if (end_mark[p] < 0) continue;
    const int32_t prev = p > 0 ? last_end[p - 1] : -1;
    const double tp0 = prev >= 0 ? tp[prev] : 0.0, fp0 = prev >= 0 ? fp[prev] : 0.0;
    area += pr ? pr_segment(tp0, fp0, tp[p], fp[p], P) : fabs(fp[p] - fp0) * (tp[p] + tp0) * 0.5;
  }
  area = b2_block_sum_fixed(area, sh);
  if (threadIdx.x == 0) partial[blockIdx.x] = area;
}
// one CTA: the class's contribution out3 = ROC (area, fp * tp, tp) or PR (aucpr, 1, 1), aucpr NaN without positive or
// without negative weight
__global__ void auc_finish_kernel(int pr, const double* __restrict__ partial, int g, const double* __restrict__ tp,
                                  const double* __restrict__ fp, int64_t n, double* __restrict__ out3) {
  __shared__ double sh[32];
  double s = 0.0;
  for (int i = threadIdx.x; i < g; i += blockDim.x) s += partial[i];
  s = b2_block_sum_fixed(s, sh);
  if (threadIdx.x == 0) {
    const double P = n > 0 ? tp[n - 1] : 0.0, N = n > 0 ? fp[n - 1] : 0.0;
    if (pr) { out3[0] = (P > 0.0 && N > 0.0) ? s : __longlong_as_double(0x7ff8000000000000LL); out3[1] = 1.0; out3[2] = 1.0; }
    else    { out3[0] = s; out3[1] = N * P; out3[2] = P; }
  }
}

struct MaxOp {
  __device__ __forceinline__ int32_t operator()(int32_t a, int32_t b) const { return a > b ? a : b; }
};

static size_t cub_bytes_for(int64_t n) {
  size_t sort_bytes = 0, scan_d = 0, scan_i = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int32_t*)nullptr,
                                  (int32_t*)nullptr, (int)n);
  cub::DeviceScan::InclusiveSum(nullptr, scan_d, (const double*)nullptr, (double*)nullptr, (int)n);
  cub::DeviceScan::InclusiveScan(nullptr, scan_i, (const int32_t*)nullptr, (int32_t*)nullptr, MaxOp(), (int)n);
  size_t cub_bytes = sort_bytes > scan_d ? sort_bytes : scan_d;
  if (scan_i > cub_bytes) cub_bytes = scan_i;
  return (cub_bytes + 255) & ~(size_t)255;
}

}  // namespace b2

extern "C" {
// bytes of scratch memory b2_auc needs for n rows (any K: the classes reuse it one after the other)
size_t b2_auc_temp_bytes(int64_t n) {
  if (n < 1) n = 1;
  const size_t per_row = 2 * sizeof(uint32_t) + 2 * sizeof(int32_t) + 4 * sizeof(double) + 2 * sizeof(int32_t);
  const size_t partials = (size_t)((n + 255) / 256) * sizeof(double);
  return b2::cub_bytes_for(n) + (size_t)n * per_row + partials + 4096;
}
// pr: 0 `auc` (ROC), 1 `aucpr`.  pred: transformed predictions [n, K]; K == 1 is the binary metric on the label as it
// is, K > 1 one-vs-rest over the classes.  out: [3K + 1] doubles (device), zeroed here: per class the worker's
// triple (see auc_finish_kernel), then (K > 1) the number of rows whose label is not in [0, K).  Returns a cudaError.
int b2_auc(int pr, int K, const float* pred, const float* label, const float* weight, int64_t n, void* temp,
           size_t temp_bytes, double* out, int num_sms, cudaStream_t s) {
  if (K < 1) return (int)cudaErrorInvalidValue;
  cudaMemsetAsync(out, 0, (3 * (size_t)K + 1) * sizeof(double), s);
  if (temp_bytes < b2_auc_temp_bytes(n)) return (int)cudaErrorInvalidValue;
  const size_t cub_bytes = b2::cub_bytes_for(n < 1 ? 1 : n);
  const int64_t m = n < 1 ? 1 : n;
  char* p = (char*)temp;
  void* cub_tmp = p; p += cub_bytes;
  double* pos = (double*)p; p += (size_t)m * 8;
  double* neg = (double*)p; p += (size_t)m * 8;
  double* tp = (double*)p; p += (size_t)m * 8;
  double* fp = (double*)p; p += (size_t)m * 8;
  double* partial = (double*)p; p += (size_t)((m + 255) / 256) * 8;
  uint32_t* keys = (uint32_t*)p; p += (size_t)m * 4;
  uint32_t* keys_s = (uint32_t*)p; p += (size_t)m * 4;
  int32_t* idx = (int32_t*)p; p += (size_t)m * 4;
  int32_t* idx_s = (int32_t*)p; p += (size_t)m * 4;
  int32_t* end_mark = (int32_t*)p; p += (size_t)m * 4;
  int32_t* last_end = (int32_t*)p; p += (size_t)m * 4;
  int64_t g = (n + 255) / 256; if (g > (int64_t)num_sms * 16) g = (int64_t)num_sms * 16;
  for (int c = 0; c < K; ++c) {
    if (n > 0) {
      b2::auc_keys_kernel<<<(int)g, 256, 0, s>>>(pred, K, c, n, keys, idx);
      size_t tb = cub_bytes;
      cub::DeviceRadixSort::SortPairs(cub_tmp, tb, keys, keys_s, idx, idx_s, (int)n, 0, 32, s);
      b2::auc_weights_kernel<<<(int)g, 256, 0, s>>>(keys_s, idx_s, label, weight, n, K, c, pos, neg, end_mark,
                                                    K > 1 && c == 0 ? out + 3 * K : nullptr);
      tb = cub_bytes; cub::DeviceScan::InclusiveSum(cub_tmp, tb, pos, tp, (int)n, s);
      tb = cub_bytes; cub::DeviceScan::InclusiveSum(cub_tmp, tb, neg, fp, (int)n, s);
      tb = cub_bytes; cub::DeviceScan::InclusiveScan(cub_tmp, tb, end_mark, last_end, b2::MaxOp(), (int)n, s);
      b2::auc_area_kernel<<<(int)g, 256, 0, s>>>(pr, tp, fp, end_mark, last_end, n, partial);
    }
    b2::auc_finish_kernel<<<1, 256, 0, s>>>(pr, partial, n > 0 ? (int)g : 0, tp, fp, n, out + 3 * c);
  }
  return (int)cudaGetLastError();
}
}
