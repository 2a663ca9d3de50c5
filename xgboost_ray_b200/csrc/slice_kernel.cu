// slice_kernel.cu -- DMatrix.slice on the device (B2_MatrixSlice): rows rows[0..n) of a parent matrix, in that order and
// with duplicates allowed, gathered out of the parent's device buffers.  Dense values and the per-row side arrays are a
// row gather; CSR values keep their CSR form (row lengths, a scan for the new row pointers, then the entries of every
// row copied as one segment).  Every value is copied bit for bit.
#include <stdint.h>

#include <algorithm>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "launch.h"

namespace b2 {

constexpr int kSliceThreads = 256;

// dst [n][vw] = src [rows[i]][vw], in vectors of V (float4 / float2 / float: the widest the row width allows, so that a
// row of F floats moves in 16-byte loads when F % 4 == 0)
template <typename V>
__global__ void __launch_bounds__(kSliceThreads)
gather_rows_kernel(const V* __restrict__ src, int64_t vw, const int64_t* __restrict__ rows, int64_t n, V* __restrict__ dst) {
  const int64_t total = n * vw;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / vw, c = i - r * vw;
    dst[i] = __ldg(src + __ldg(rows + r) * vw + c);
  }
}

// lengths[i] = entries of parent row rows[i]; out_indptr[0] = 0 (the scan writes out_indptr[1..n])
__global__ void __launch_bounds__(kSliceThreads)
csr_slice_lengths_kernel(const int64_t* __restrict__ indptr, const int64_t* __restrict__ rows, int64_t n,
                         int64_t* __restrict__ lengths, int64_t* __restrict__ out_indptr) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = __ldg(rows + i);
    lengths[i] = __ldg(indptr + r + 1) - __ldg(indptr + r);
    if (i == 0) out_indptr[0] = 0;
  }
}

// one warp per slice row: the row's entries [indptr[r], indptr[r+1]) go to [out_indptr[i], out_indptr[i+1])
__global__ void __launch_bounds__(kSliceThreads)
csr_slice_entries_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                         const uint32_t* __restrict__ values, const int64_t* __restrict__ rows, int64_t n,
                         const int64_t* __restrict__ out_indptr, int32_t* __restrict__ out_indices,
                         uint32_t* __restrict__ out_values) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < n; i += warps) {
    const int64_t r = __ldg(rows + i), b = __ldg(indptr + r), len = __ldg(indptr + r + 1) - b, o = out_indptr[i];
    for (int64_t k = lane; k < len; k += 32) {
      out_indices[o + k] = __ldg(indices + b + k);
      out_values[o + k] = __ldg(values + b + k);
    }
  }
}

}  // namespace b2

static inline int slice_grid(int64_t work, int num_sms) {
  int64_t g = (work + b2::kSliceThreads - 1) / b2::kSliceThreads, cap = (int64_t)num_sms * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

template <typename V>
static int gather_rows(const float* src, int64_t width, const int64_t* rows, int64_t n, float* dst, int num_sms, cudaStream_t s) {
  const int64_t vw = width / (int64_t)(sizeof(V) / sizeof(float));
  b2::gather_rows_kernel<V><<<slice_grid(n * vw, num_sms), b2::kSliceThreads, 0, s>>>(
      reinterpret_cast<const V*>(src), vw, rows, n, reinterpret_cast<V*>(dst));
  return (int)cudaGetLastError();
}

extern "C" {

int b2_launch_gather_rows(const float* src, int64_t width, const int64_t* rows, int64_t n, float* dst, int num_sms,
                          cudaStream_t s) {
  if (n <= 0 || width <= 0) return 0;
  if (width % 4 == 0) return gather_rows<float4>(src, width, rows, n, dst, num_sms, s);
  if (width % 2 == 0) return gather_rows<float2>(src, width, rows, n, dst, num_sms, s);
  return gather_rows<float>(src, width, rows, n, dst, num_sms, s);
}

size_t b2_csr_slice_temp_bytes(int64_t n) {
  size_t bytes = 0;
  cub::DeviceScan::InclusiveSum(nullptr, bytes, (const int64_t*)nullptr, (int64_t*)nullptr, (int)std::max<int64_t>(n, 1));
  return bytes;
}

int b2_launch_csr_slice_indptr(const int64_t* indptr, const int64_t* rows, int64_t n, int64_t* lengths, int64_t* out_indptr,
                               void* temp, size_t temp_bytes, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::csr_slice_lengths_kernel<<<slice_grid(n, num_sms), b2::kSliceThreads, 0, s>>>(indptr, rows, n, lengths, out_indptr);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  return (int)cub::DeviceScan::InclusiveSum(temp, temp_bytes, lengths, out_indptr + 1, (int)n, s);
}

int b2_launch_csr_slice_entries(const int64_t* indptr, const int32_t* indices, const float* values, const int64_t* rows,
                                int64_t n, const int64_t* out_indptr, int32_t* out_indices, float* out_values, int num_sms,
                                cudaStream_t s) {
  if (n <= 0) return 0;
  const int warps_per_cta = b2::kSliceThreads / 32;
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n + warps_per_cta - 1) / warps_per_cta, (int64_t)num_sms * 8));
  b2::csr_slice_entries_kernel<<<grid, b2::kSliceThreads, 0, s>>>(indptr, indices, reinterpret_cast<const uint32_t*>(values),
                                                                 rows, n, out_indptr, out_indices,
                                                                 reinterpret_cast<uint32_t*>(out_values));
  return (int)cudaGetLastError();
}

}  // extern "C"
