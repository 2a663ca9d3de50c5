// sparse_kernel.cu -- the raw values of a CSR matrix (B2_MatrixCreateFromCSR): validation of the three arrays, dense
// row tiles for the kernels that read raw rows, and the sketch's entry keys and categorical statistics read straight
// from the stored entries.
//
// An entry a row does not store is missing.  A stored entry is copied bit for bit, so every kernel that reads a tile
// sees exactly the floats of the matrix's dense twin (the same matrix with NaN in every absent cell).
#include <stdint.h>

#include <algorithm>

#include "common.cuh"
#include "launch.h"
#include "raw_keys.cuh"

namespace b2 {

constexpr int kSparseThreads = 256;
constexpr int kDensifyCells = 4096;      // cells of one CTA step (rows * F), so that narrow matrices fill the CTA
constexpr int kDensifyMaxRows = 1024;    // rows of one CTA step (the row pointers staged in shared memory)

// bad = smallest row that breaks a rule: indptr[0] = 0, indptr[n] = nnz, indptr non-decreasing and inside [0, nnz],
// every column in [0, F) and the columns of a row strictly increasing (no duplicates).  One thread per row.
__global__ void __launch_bounds__(kSparseThreads)
csr_validate_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, int64_t n, int F, int64_t nnz,
                    unsigned long long* __restrict__ bad) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = indptr[i], e = indptr[i + 1];
    bool ok = b >= 0 && b <= e && e <= nnz && (i != 0 || b == 0) && (i != n - 1 || e == nnz);
    for (int64_t k = b, prev = -1; ok && k < e; ++k) {
      const int c = indices[k];
      ok = c > prev && c < F;   // prev = -1 first: a negative column fails too
      prev = c;
    }
    if (!ok) atomicMin(bad, (unsigned long long)i);
  }
}

// out [rows][F] = rows [r0, r0 + rows) of the CSR, NaN where a row stores nothing.  A CTA step covers `step` rows: it
// fills their cells with NaN, then scatters their stored entries (one thread per entry, its row found by a binary
// search of the step's row pointers in shared memory).  The entries of a step are contiguous in indices / values, so
// both phases read and write whole sectors.
__global__ void __launch_bounds__(kSparseThreads)
csr_densify_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const uint32_t* __restrict__ values,
                   int64_t r0, int64_t rows, int F, int step, uint32_t* __restrict__ out) {
  __shared__ int64_t sptr[kDensifyMaxRows + 1];
  const int64_t n_steps = (rows + step - 1) / step;
  for (int64_t blk = blockIdx.x; blk < n_steps; blk += gridDim.x) {
    const int64_t lr0 = blk * step;
    const int nr = (int)min((int64_t)step, rows - lr0);
    uint32_t* dst = out + lr0 * F;
    const int64_t cells = (int64_t)nr * F;
    for (int64_t c = threadIdx.x; c < cells; c += blockDim.x) dst[c] = 0x7fc00000u;   // NaN
    for (int i = threadIdx.x; i <= nr; i += blockDim.x) sptr[i] = indptr[r0 + lr0 + i];
    __syncthreads();
    const int64_t e1 = sptr[nr];
    for (int64_t e = sptr[0] + threadIdx.x; e < e1; e += blockDim.x) {
      int lo = 0, hi = nr;   // the last row of the step whose first entry is <= e
      while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (sptr[mid] <= e) lo = mid; else hi = mid; }
      dst[(int64_t)lo * F + __ldg(indices + e)] = __ldg(values + e);
    }
    __syncthreads();
  }
}

// counts [F] += the valid stored entries (not missing) of every numeric feature: the sizes of the sketch's segments
__global__ void __launch_bounds__(kSparseThreads)
csr_column_counts_kernel(const int32_t* __restrict__ indices, const float* __restrict__ values, int64_t nnz, float missing,
                         int missing_is_nan, const uint8_t* __restrict__ is_cat, unsigned long long* __restrict__ counts) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
    const int f = __ldg(indices + e);
    if (!is_missing(__ldg(values + e), missing, missing_is_nan) && !(is_cat && is_cat[f])) atomicAdd(counts + f, 1ull);
  }
}

// The sketch keys of features [f0, f0 + nf): every valid entry of a numeric feature f0 + j becomes (j << 32) | its
// sketch key, at the next free slot of feature j's segment (cursor [nf], started at the segment starts), with its row's
// integer weight when wq != nullptr.  The order inside a segment does not matter: the segments are sorted next.  One
// thread per row: a binary search finds the row's first column >= f0, then its entries in the window are keyed.
__global__ void __launch_bounds__(kSparseThreads)
csr_sketch_keys_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const float* __restrict__ values,
                       int64_t n, int f0, int nf, float missing, int missing_is_nan, const uint8_t* __restrict__ is_cat,
                       const int32_t* __restrict__ wq, unsigned int* __restrict__ cursor, uint64_t* __restrict__ keys,
                       int32_t* __restrict__ wq_out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t end = indptr[i + 1];
    int64_t lo = indptr[i], hi = end;
    while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (__ldg(indices + mid) < f0) lo = mid + 1; else hi = mid; }
    for (int64_t e = lo; e < end; ++e) {
      const int f = __ldg(indices + e), j = f - f0;
      if (j >= nf) break;
      const float x = __ldg(values + e);
      if (is_missing(x, missing, missing_is_nan) || (is_cat && is_cat[f])) continue;
      const unsigned int p = atomicAdd(cursor + j, 1u);
      keys[p] = ((uint64_t)j << 32) | sketch_key(x);
      if (wq) wq_out[p] = wq[i];
    }
  }
}

// Categorical statistics (cat_stats_update) from the stored entries, one thread per entry; cat_of [F] = the feature's
// index among the categorical features, or -1.  stored [n_cat] counts the entries, so that a feature some row does not
// store is marked missing by csr_cat_absent_kernel.
__global__ void __launch_bounds__(kSparseThreads)
csr_cat_stats_kernel(const int32_t* __restrict__ indices, const float* __restrict__ values, int64_t nnz, float missing,
                     int missing_is_nan, const int32_t* __restrict__ cat_of, unsigned long long* __restrict__ stored,
                     int32_t* __restrict__ stats) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
    const int ci = cat_of[__ldg(indices + e)];
    if (ci < 0) continue;
    atomicAdd(stored + ci, 1ull);
    cat_stats_update(__ldg(values + e), missing, missing_is_nan, stats, ci);
  }
}
__global__ void csr_cat_absent_kernel(const unsigned long long* __restrict__ stored, int n_cat, int64_t n, int32_t* __restrict__ stats) {
  for (int ci = blockIdx.x * blockDim.x + threadIdx.x; ci < n_cat; ci += gridDim.x * blockDim.x)
    if ((int64_t)stored[ci] < n) stats[ci * 3 + 1] = 1;
}

// out [n][F] = the dense bins of a CSR-layout matrix: the sentinel in every cell, then each row's stored bins (one
// thread per row)
__global__ void __launch_bounds__(kSparseThreads)
csr_bins_densify_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const uint8_t* __restrict__ ebins,
                        int64_t n, int F, uint8_t* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    uint8_t* row = out + i * F;
    for (int f = 0; f < F; ++f) row[f] = B2_MISSING_BIN;
    for (int64_t e = indptr[i]; e < indptr[i + 1]; ++e) row[indices[e]] = ebins[e];
  }
}

}  // namespace b2

static inline int sparse_grid(int64_t work, int num_sms) {
  int64_t g = (work + b2::kSparseThreads - 1) / b2::kSparseThreads, cap = (int64_t)num_sms * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

extern "C" {

int b2_launch_csr_validate(const int64_t* indptr, const int32_t* indices, int64_t n, int F, int64_t nnz, unsigned long long* bad,
                           int num_sms, cudaStream_t s) {
  cudaError_t e = cudaMemsetAsync(bad, 0xff, sizeof(unsigned long long), s);
  if (e != cudaSuccess || n <= 0) return (int)e;
  b2::csr_validate_kernel<<<sparse_grid(n, num_sms), b2::kSparseThreads, 0, s>>>(indptr, indices, n, F, nnz, bad);
  return (int)cudaGetLastError();
}

int b2_launch_csr_bins_densify(const int64_t* indptr, const int32_t* indices, const uint8_t* ebins, int64_t n, int F,
                               uint8_t* out, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  const int64_t want = (n + b2::kSparseThreads - 1) / b2::kSparseThreads, cap = (int64_t)num_sms * 8;
  b2::csr_bins_densify_kernel<<<(int)std::min(want, cap), b2::kSparseThreads, 0, s>>>(indptr, indices, ebins, n, F, out);
  return (int)cudaGetLastError();
}
int b2_launch_csr_densify(const int64_t* indptr, const int32_t* indices, const float* values, int64_t r0, int64_t rows, int F,
                          float* out, int num_sms, cudaStream_t s) {
  if (rows <= 0) return 0;
  const int step = F >= b2::kDensifyCells ? 1 : std::min(b2::kDensifyMaxRows, b2::kDensifyCells / F);
  const int64_t n_steps = (rows + step - 1) / step;
  const int grid = (int)std::min<int64_t>(n_steps, (int64_t)num_sms * 8);
  b2::csr_densify_kernel<<<grid, b2::kSparseThreads, 0, s>>>(indptr, indices, reinterpret_cast<const uint32_t*>(values), r0, rows,
                                                            F, step, reinterpret_cast<uint32_t*>(out));
  return (int)cudaGetLastError();
}

int b2_launch_csr_column_counts(const int32_t* indices, const float* values, int64_t nnz, float missing, const uint8_t* is_cat,
                                unsigned long long* counts, int num_sms, cudaStream_t s) {
  if (nnz <= 0) return 0;
  b2::csr_column_counts_kernel<<<sparse_grid(nnz, num_sms), b2::kSparseThreads, 0, s>>>(indices, values, nnz, missing,
                                                                                      missing != missing ? 1 : 0, is_cat, counts);
  return (int)cudaGetLastError();
}
int b2_launch_csr_sketch_keys(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int f0, int nf,
                              float missing, const uint8_t* is_cat, const int32_t* wq, unsigned int* cursor, uint64_t* keys,
                              int32_t* wq_out, int num_sms, cudaStream_t s) {
  if (n <= 0 || nf <= 0) return 0;
  b2::csr_sketch_keys_kernel<<<sparse_grid(n, num_sms), b2::kSparseThreads, 0, s>>>(indptr, indices, values, n, f0, nf, missing,
                                                                                  missing != missing ? 1 : 0, is_cat, wq, cursor,
                                                                                  keys, wq_out);
  return (int)cudaGetLastError();
}
int b2_launch_csr_cat_stats(const int32_t* indices, const float* values, int64_t nnz, int64_t n, float missing, const int32_t* cat_of,
                            int n_cat, unsigned long long* stored, int32_t* stats, int num_sms, cudaStream_t s) {
  if (n_cat <= 0) return 0;
  cudaError_t e = cudaMemsetAsync(stored, 0, (size_t)n_cat * sizeof(unsigned long long), s);
  if (e != cudaSuccess) return (int)e;
  if (nnz > 0)
    b2::csr_cat_stats_kernel<<<sparse_grid(nnz, num_sms), b2::kSparseThreads, 0, s>>>(indices, values, nnz, missing,
                                                                                    missing != missing ? 1 : 0, cat_of, stored, stats);
  b2::csr_cat_absent_kernel<<<1, 256, 0, s>>>(stored, n_cat, n, stats);
  return (int)cudaGetLastError();
}

}  // extern "C"
