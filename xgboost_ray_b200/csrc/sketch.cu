// sketch.cu -- GPU quantile cuts and binning of an actor's RayDMatrix shard.
//
// Replaces the DMatrix quantisation the reference triggers at xgboost_ray/main.py:386/418/437
// (SURVEY.md 8a rows a7, a8; Appendix A.2).  Per feature: order-preserving uint32 keys of the
// (global) column are radix sorted (cub::DeviceRadixSort -- library sort, one-time preprocessing),
// the exact distinct-value summary (value, rmin, rmax as int64 ranks) is built, XGBoost's
// WQSummary::SetPrune selection rule is evaluated with one thread per target rank, and the cut
// values are emitted.  Binning is bin = upper_bound(cuts_f, x) into the padded group-major row
// layout used by the histogram kernel.
#include <algorithm>

#include <cub/cub.cuh>

#include "common.cuh"
#include "launch.h"
#include "raw_keys.cuh"

namespace b2 {

// keys of kBatch consecutive feature columns in one pass: thread (row, j) reads X[row][f0+j], so a warp
// reads 4 rows x 32 contiguous bytes (whole sectors) instead of one float per 4*F-byte row.
constexpr int kExtractBatch = 8;
__global__ void extract_keys_kernel(const float* __restrict__ X, int64_t n, int F, int f0, int nf, float missing,
                                    int missing_is_nan, uint32_t* __restrict__ keys /*[kBatch][n_padded]*/, int64_t n_padded) {
  const int64_t total = n_padded * kExtractBatch;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / kExtractBatch; const int j = (int)(t % kExtractBatch);
    if (j >= nf) continue;
    uint32_t k = 0xffffffffu;
    if (i < n) {
      float x = X[i * F + f0 + j];
      if (!is_missing(x, missing, missing_is_nan)) k = sketch_key(x);
    }
    keys[(int64_t)j * n_padded + i] = k;
  }
}

// n_valid = number of keys below the missing/padding sentinel 0xffffffff in the sorted array
__global__ void count_valid_kernel(const uint32_t* __restrict__ sorted, int64_t n_total, long long* __restrict__ n_valid) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int64_t lo = 0, hi = n_total;
  while (lo < hi) { int64_t mid = (lo + hi) >> 1; if (sorted[mid] == 0xffffffffu) hi = mid; else lo = mid + 1; }
  *n_valid = lo;
}

// Key: uint32_t (one feature's keys, the all-ones sentinel = missing) or uint64_t (a batch's (feature << 32) | key,
// where a new feature starts a new run)
template <typename Key>
__global__ void head_flags_kernel(const Key* __restrict__ keys, int64_t n_total, int32_t* __restrict__ flags) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_total; i += (int64_t)gridDim.x * blockDim.x)
    flags[i] = (keys[i] != ~(Key)0 && (i == 0 || keys[i] != keys[i - 1])) ? 1 : 0;
}
__global__ void scatter_unique_kernel(const uint32_t* __restrict__ keys, const int32_t* __restrict__ flags,
                                      const int32_t* __restrict__ idx, int64_t n_total, float* __restrict__ uval,
                                      long long* __restrict__ rmin, int32_t* __restrict__ m_out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_total; i += (int64_t)gridDim.x * blockDim.x) {
    if (flags[i]) { uval[idx[i]] = key2f(keys[i]); rmin[idx[i]] = i; }
    if (i == n_total - 1) *m_out = idx[i] + flags[i];
  }
}

// ---- weighted sketch (sample weights; WQSummary ranks are sums of weights).  Weights are quantised to integers
// wq = rint(w * 2^(30 - e)), 2^e > max w over all ranks, so rank sums are exact int64 and independent of the order
// of rows and of the number of GPUs (same idea as the fixed-point gradient histograms).
__global__ void weight_absmax_kernel(const float* __restrict__ w, int64_t n, uint32_t* __restrict__ out /*[2]: max bits, invalid*/) {
  uint32_t mx = 0, bad = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = w[i];
    if (!(v >= 0.0f) || isinf(v)) bad = 1; else mx = max(mx, __float_as_uint(fabsf(v)));   // -0.0 is a valid weight of 0
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o)); bad |= __shfl_xor_sync(0xffffffffu, bad, o); }
  if ((threadIdx.x & 31) == 0) { if (mx) atomicMax(&out[0], mx); if (bad) atomicMax(&out[1], 1u); }
}
__global__ void weight_quantize_kernel(const float* __restrict__ w, int64_t n, int64_t n_padded, const uint32_t* __restrict__ absmax,
                                       int32_t* __restrict__ wq) {
  const int e = b2_frexp_exponent(absmax[0]);
  const float2 scale = b2_pow2_split(30 - e);          // exact powers of two; 2^(30 - e) alone overflows for max w < 2^-98
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_padded; i += (int64_t)gridDim.x * blockDim.x)
    wq[i] = i < n ? __float2int_rn(__fmul_rn(__fmul_rn(w[i], scale.x), scale.y)) : 0;
}
struct CastI64 { __host__ __device__ long long operator()(int32_t v) const { return (long long)v; } };
__global__ void scatter_unique_weighted_kernel(const uint32_t* __restrict__ keys, const int32_t* __restrict__ flags,
                                               const int32_t* __restrict__ idx, const long long* __restrict__ wpre,
                                               const int32_t* __restrict__ wq_sorted, const long long* __restrict__ n_valid_ptr,
                                               int64_t n_total, float* __restrict__ uval, long long* __restrict__ rmin,
                                               int32_t* __restrict__ m_out, long long* __restrict__ w_total) {
  const long long n_valid = *n_valid_ptr;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_total; i += (int64_t)gridDim.x * blockDim.x) {
    if (flags[i]) { uval[idx[i]] = key2f(keys[i]); rmin[idx[i]] = wpre[i]; }
    if (i == n_total - 1) *m_out = idx[i] + flags[i];
    if (i == n_valid - 1) *w_total = wpre[i] + wq_sorted[i];      // total weight of the non-missing values
  }
  if (n_valid == 0 && blockIdx.x == 0 && threadIdx.x == 0) *w_total = 0;
}

// A batch of features sorted as (feature << 32) | key, feature j's entries at [seg[j], seg[j+1]) (only valid keys): the
// summary entry of every distinct value, its rank relative to its feature's first entry -- the position, or with integer
// weights the prefix wpre of the weights -- exactly what scatter_unique(_weighted)_kernel computes for the feature alone.
__global__ void scatter_unique_segments_kernel(const uint64_t* __restrict__ keys, const int32_t* __restrict__ flags,
                                               const int32_t* __restrict__ idx, const long long* __restrict__ wpre,
                                               const int64_t* __restrict__ seg, int64_t n_total, float* __restrict__ uval,
                                               long long* __restrict__ rmin) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_total; i += (int64_t)gridDim.x * blockDim.x) {
    if (!flags[i]) continue;
    const uint64_t k = keys[i];
    const int64_t s = seg[k >> 32];
    uval[idx[i]] = key2f((uint32_t)k);
    rmin[idx[i]] = wpre ? wpre[i] - wpre[s] : i - s;
  }
}

// WQSummary::SetPrune + HistogramCuts::AddCutPoint on the exact summary of one feature (A.2), by one whole block:
// get_m() distinct values uval / rmin, n_valid non-missing values of n_global rows, rank_end the total rank (the last
// rmax: n_valid, or the total weight).
template <typename MFn>
__device__ __forceinline__ void prune_cuts(const float* __restrict__ uval, const long long* __restrict__ rmin, MFn get_m,
                                           long long n_valid, long long rank_end, long long n_global, int max_bin,
                                           float* __restrict__ cut_out /*[256]*/, int32_t* __restrict__ n_cut_out,
                                           float* __restrict__ min_out, int32_t* __restrict__ has_missing_out) {
  __shared__ int sel[260];
  __shared__ int choice[260];
  const bool any_missing = n_valid < n_global;
  const int max_bin_cap = (any_missing && max_bin > 255) ? 255 : max_bin;   // bin 255 is the missing sentinel
  if (threadIdx.x == 0) *has_missing_out = any_missing ? 1 : 0;
  const int m = n_valid > 0 ? get_m() : 0;
  if (m == 0) {
    if (threadIdx.x == 0) {
      float mval = 0.0f;
      float mn = __fadd_rn(__fadd_rn(mval, -fabsf(mval)), -1e-5f);
      *min_out = mn;
      cut_out[0] = __fadd_rn(mn, __fadd_rn(fabsf(mn), 1e-5f));
      *n_cut_out = 1;
    }
    return;
  }
  const int max_num_bins = m < max_bin_cap ? m : max_bin_cap;
  const int maxsize = max_num_bins + 1;
  int size = 0;
  auto RMAX = [&](int u) -> long long { return (u + 1 < m) ? rmin[u + 1] : rank_end; };
  if (m > maxsize) {
    const double begin = (double)RMAX(0);
    const double range = __dadd_rn((double)rmin[m - 1], -begin);
    const int n = maxsize - 1;
    for (int k = threadIdx.x; k < n; k += blockDim.x) {
      int c = -1;
      if (k >= 1) {
        const double dx2 = 2.0 * __dadd_rn(__ddiv_rn(__dmul_rn((double)k, range), (double)n), begin);
        // i = 1 + #{ j in [2, m-1] : rmin[j]+rmax[j] <= dx2 }
        int lo = 2, hi = m;  // first j in [2,m) with S(j) > dx2
        while (lo < hi) {
          int mid = (lo + hi) >> 1;
          double S = (double)(rmin[mid] + RMAX(mid));
          if (dx2 >= S) lo = mid + 1; else hi = mid;
        }
        const int i = lo - 1;
        if (i < m - 1) c = (dx2 < (double)(RMAX(i) + rmin[i + 1])) ? i : i + 1;
      }
      choice[k] = c;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      sel[size++] = 0;
      int lastidx = 0;
      for (int k = 1; k < n; ++k) {
        int c = choice[k];
        if (c < 0) break;
        if (c != lastidx) { sel[size++] = c; lastidx = c; }
      }
      if (lastidx != m - 1) sel[size++] = m - 1;
    }
  } else if (threadIdx.x == 0) {
    for (int i = 0; i < m; ++i) sel[size++] = i;
  }
  // the selected summary values are fetched by all threads at once (a serial chain of ~256 global loads by one
  // thread cost ~90 us per feature), the duplicate-dropping pass runs on shared memory
  __shared__ int s_size, s_nc;
  __shared__ float sval[260], scut[260];
  if (threadIdx.x == 0) s_size = size;
  __syncthreads();
  size = s_size;
  for (int i = threadIdx.x; i < size; i += blockDim.x) sval[i] = uval[sel[i]];
  __syncthreads();
  if (threadIdx.x == 0) {
    const float mval = sval[0];
    *min_out = __fadd_rn(__fadd_rn(mval, -fabsf(mval)), -1e-5f);
    const int required = size < max_num_bins ? size : max_num_bins;
    int nc = 0;
    for (int i = 1; i < required; ++i) {
      const float cpt = sval[i];
      if (i == 1 || cpt > scut[nc - 1]) scut[nc++] = cpt;
    }
    const float cpt = sval[size - 1];
    scut[nc++] = __fadd_rn(cpt, __fadd_rn(fabsf(cpt), 1e-5f));
    *n_cut_out = nc; s_nc = nc;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < s_nc; i += blockDim.x) cut_out[i] = scut[i];
}

// One block, the summary of b2_sketch_column.  w_total_ptr != nullptr: rmin holds weighted ranks and *w_total_ptr the
// total weight.
__global__ void __launch_bounds__(256)
prune_cuts_kernel(const float* __restrict__ uval, const long long* __restrict__ rmin, const int32_t* __restrict__ m_ptr,
                  const long long* __restrict__ n_valid_ptr, const long long* __restrict__ w_total_ptr, long long n_global, int max_bin,
                  float* __restrict__ cut_out /*[256]*/,
                  int32_t* __restrict__ n_cut_out, float* __restrict__ min_out, int32_t* __restrict__ has_missing_out) {
  const long long n_valid = *n_valid_ptr;
  const long long rank_end = w_total_ptr ? *w_total_ptr : n_valid;
  prune_cuts(uval, rmin, [&] { return *m_ptr; }, n_valid, rank_end, n_global, max_bin, cut_out, n_cut_out, min_out,
             has_missing_out);
}

// One block per feature of a batch (scatter_unique_segments_kernel's layout): feature f0 + j's summary is the slice of
// the batch's that starts at its first entry.  Only the owner rank (f % world) prunes; categorical features are skipped.
// Outputs are indexed by the global feature id.
__global__ void __launch_bounds__(256)
prune_cuts_segments_kernel(const float* __restrict__ uval, const long long* __restrict__ rmin, const int32_t* __restrict__ flags,
                           const int32_t* __restrict__ idx, const long long* __restrict__ wpre, const int32_t* __restrict__ wq_sorted,
                           const int64_t* __restrict__ seg, int f0, const uint8_t* __restrict__ is_cat, int world, int rank,
                           long long n_global, int max_bin, float* __restrict__ cuts /*[F][256]*/, int32_t* __restrict__ n_cuts,
                           float* __restrict__ mins, int32_t* __restrict__ has_missing) {
  const int f = f0 + blockIdx.x;
  if ((is_cat && is_cat[f]) || f % world != rank) return;
  const int64_t s = seg[blockIdx.x], e = seg[blockIdx.x + 1];
  const long long n_valid = e - s;
  const int64_t u0 = n_valid > 0 ? idx[s] : 0;
  const long long rank_end = !wpre ? n_valid : (n_valid > 0 ? wpre[e - 1] + wq_sorted[e - 1] - wpre[s] : 0);
  prune_cuts(uval + u0, rmin + u0, [&] { return idx[e - 1] + flags[e - 1] - (int)u0; }, n_valid, rank_end, n_global, max_bin,
             cuts + (size_t)f * 256, n_cuts + f, mins + f, has_missing + f);
}

// Categorical columns: the statistics of cat_stats_update (raw_keys.cuh), one thread per cell.
__global__ void cat_stats_kernel(const float* __restrict__ X, int64_t n, int F, float missing, int missing_is_nan,
                                 const int32_t* __restrict__ cat_feats, int n_cat, int32_t* __restrict__ stats) {
  const int64_t total = n * n_cat;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = e / n_cat; const int ci = (int)(e - row * n_cat);
    cat_stats_update(X[row * F + cat_feats[ci]], missing, missing_is_nan, stats, ci);
  }
}

// bin = upper_bound(cuts_f, x) clamped; missing -> 255.
// Categorical feature: bin = category code (clamped to the codes the cuts know).
__device__ __forceinline__ int bin_value(float x, int f, float missing, int missing_is_nan, const int32_t* __restrict__ cut_ptrs,
                                         const float* __restrict__ cut_vals, const uint8_t* __restrict__ is_cat) {
  int b;
  if (is_missing(x, missing, missing_is_nan)) b = B2_MISSING_BIN;
  else if (is_cat && is_cat[f]) {
    const int nf = cut_ptrs[f + 1] - cut_ptrs[f];
    b = x >= 0.0f ? (x > 255.0f ? 255 : (int)x) : 0;
    if (b >= nf) b = nf - 1;
  } else {
    const int p0 = cut_ptrs[f], nf = cut_ptrs[f + 1] - p0;
    const float* cv = cut_vals + p0;
    int lo = 0, hi = nf;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (__ldg(cv + mid) > x) hi = mid; else lo = mid + 1; }
    b = lo >= nf ? nf - 1 : lo;
  }
  return b;
}

// One thread per matrix element.
__global__ void bin_kernel(const float* __restrict__ X, int64_t n, int F, float missing, int missing_is_nan,
                           const int32_t* __restrict__ cut_ptrs, const float* __restrict__ cut_vals,
                           const int32_t* __restrict__ feat_byte, const uint8_t* __restrict__ is_cat, int row_stride,
                           uint8_t* __restrict__ bins, uint8_t* __restrict__ bins_col, int64_t col_stride) {
  const int64_t total = n * F;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = e / F; const int f = (int)(e - row * F);
    const int b = bin_value(X[e], f, missing, missing_is_nan, cut_ptrs, cut_vals, is_cat);
    bins[row * row_stride + feat_byte[f]] = (uint8_t)b;
    bins_col[(int64_t)f * col_stride + row] = (uint8_t)b;
  }
}

// Tiled variant (F <= kBinMaxF): a CTA stages kBinTileRows whole rows of X in shared memory (one contiguous,
// fully coalesced read), then each warp bins ONE feature for 32 rows at a time, so the 32 lanes search the same
// 1 KB cut table (few L1 wavefronts per step instead of 32 different tables), the feature-major copy is written
// 32 consecutive bytes per warp and the row-major tile leaves through shared memory as whole rows.
// (The one-thread-per-element kernel above spent 29.6 ms on C3, bound by L1 wavefronts of the divergent searches.)
constexpr int kBinTileRows = 64;
constexpr int kBinMaxF = 512;
__global__ void __launch_bounds__(256)
bin_tiled_kernel(const float* __restrict__ X, int64_t n, int F, float missing, int missing_is_nan,
                 const int32_t* __restrict__ cut_ptrs, const float* __restrict__ cut_vals,
                 const int32_t* __restrict__ feat_byte, const uint8_t* __restrict__ is_cat, int row_stride,
                 uint8_t* __restrict__ bins, uint8_t* __restrict__ bins_col, int64_t col_stride) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int ldx = F | 1;                                        // odd leading dimension: conflict-free column reads
  float* sx = reinterpret_cast<float*>(smem_raw);               // [kBinTileRows][ldx]
  uint8_t* so = smem_raw + (size_t)kBinTileRows * ldx * sizeof(float);   // [kBinTileRows][row_stride + 4]: padded rows
  const int sos = row_stride + 4, sow = sos / 4, rsw = row_stride / 4;   // (a 128-byte stride would put the 32 lanes' byte stores in one bank)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  const int64_t n_tiles = (n + kBinTileRows - 1) / kBinTileRows;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t row0 = tile * kBinTileRows;
    const int rows = (int)min((int64_t)kBinTileRows, n - row0);
    const float* src = X + row0 * F;
    for (int i = threadIdx.x; i < rows * F; i += blockDim.x) { const int r = i / F; sx[r * ldx + (i - r * F)] = src[i]; }
    for (int i = threadIdx.x; i < kBinTileRows * sow; i += blockDim.x) reinterpret_cast<uint32_t*>(so)[i] = 0u;
    __syncthreads();
    for (int f = warp; f < F; f += n_warps) {
      const int p0 = cut_ptrs[f], nf = cut_ptrs[f + 1] - p0;
      const float* cv = cut_vals + p0;
      const bool cat = is_cat && is_cat[f];
      const int fb = feat_byte[f];
#pragma unroll
      for (int half = 0; half < kBinTileRows / 32; ++half) {
        const int r = half * 32 + lane;
        if (r < rows) {
          const float x = sx[r * ldx + f];
          int b;
          if (is_missing(x, missing, missing_is_nan)) b = B2_MISSING_BIN;
          else if (cat) {
            b = x >= 0.0f ? (x > 255.0f ? 255 : (int)x) : 0;
            if (b >= nf) b = nf - 1;
          } else {
            int lo = 0, hi = nf;
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (__ldg(cv + mid) > x) hi = mid; else lo = mid + 1; }
            b = lo >= nf ? nf - 1 : lo;
          }
          so[r * sos + fb] = (uint8_t)b;
          bins_col[(int64_t)f * col_stride + row0 + r] = (uint8_t)b;
        }
      }
    }
    __syncthreads();
    uint32_t* dst = reinterpret_cast<uint32_t*>(bins + row0 * row_stride);        // row_stride is a multiple of 32
    for (int i = threadIdx.x; i < rows * rsw; i += blockDim.x) {
      const int r = i / rsw;
      dst[i] = reinterpret_cast<const uint32_t*>(so)[r * sow + (i - r * rsw)];
    }
    __syncthreads();
  }
}

// CSR bin layout: the bin of every stored entry (one thread per entry), by the rule of bin_kernel.  A stored NaN or
// `missing` gets the sentinel, as the same cell of the dense twin does.
__global__ void bin_csr_kernel(const int32_t* __restrict__ indices, const float* __restrict__ values, int64_t nnz, float missing,
                               int missing_is_nan, const int32_t* __restrict__ cut_ptrs, const float* __restrict__ cut_vals,
                               const uint8_t* __restrict__ is_cat, uint8_t* __restrict__ ebins) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x)
    ebins[e] = (uint8_t)bin_value(values[e], indices[e], missing, missing_is_nan, cut_ptrs, cut_vals, is_cat);
}

}  // namespace b2

static inline int sk_grid(int64_t n, int num_sms) {
  int64_t g = (n + 255) / 256, cap = (int64_t)num_sms * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

extern "C" {

int b2_extract_batch() { return b2::kExtractBatch; }

int b2_launch_extract_keys(const float* X, int64_t n, int F, int f0, int nf, float missing, uint32_t* keys, int64_t n_padded,
                           int num_sms, cudaStream_t s) {
  if (n_padded <= 0) return 0;
  b2::extract_keys_kernel<<<sk_grid(n_padded * b2::kExtractBatch, num_sms), 256, 0, s>>>(X, n, F, f0, nf, missing,
                                                                                      missing != missing ? 1 : 0, keys, n_padded);
  return (int)cudaGetLastError();
}

size_t b2_sort_temp_bytes(int64_t n) {
  size_t bytes = 0, b2 = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, n);
  cub::DeviceRadixSort::SortPairs(nullptr, b2, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int32_t*)nullptr,
                                  (int32_t*)nullptr, n);
  bytes = bytes > b2 ? bytes : b2;
  cub::DeviceScan::ExclusiveSum(nullptr, b2, (const int32_t*)nullptr, (int32_t*)nullptr, n);
  bytes = bytes > b2 ? bytes : b2;
  cub::TransformInputIterator<long long, b2::CastI64, const int32_t*> it((const int32_t*)nullptr, b2::CastI64());
  cub::DeviceScan::ExclusiveSum(nullptr, b2, it, (long long*)nullptr, n);
  return bytes > b2 ? bytes : b2;
}

// sample weights -> integer weights of the sketch (see weight_absmax_kernel).  absmax [2] must be zeroed; call
// b2_launch_weight_absmax, allreduce(max) absmax over the ranks, then b2_launch_weight_quantize.
int b2_launch_weight_absmax(const float* w, int64_t n, uint32_t* absmax, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::weight_absmax_kernel<<<sk_grid(n, num_sms), 256, 0, s>>>(w, n, absmax);
  return (int)cudaGetLastError();
}
int b2_launch_weight_quantize(const float* w, int64_t n, int64_t n_padded, const uint32_t* absmax, int32_t* wq, int num_sms,
                              cudaStream_t s) {
  if (n_padded <= 0) return 0;
  b2::weight_quantize_kernel<<<sk_grid(n_padded, num_sms), 256, 0, s>>>(w, n, n_padded, absmax, wq);
  return (int)cudaGetLastError();
}

// keys_in [n_total] (any order, 0xffffffff = missing/padding) -> cuts of one feature, no host round trip:
// n_valid is found on the device, the 255-bin cap of features with missing values is applied on the device.
// Scratch: keys_sorted [n_total], flags/idx int32 [n_total], uval float [n_total], rmin int64 [n_total].
// wq_in (nullable) [n_total]: integer sample weights aligned with keys_in; wq_sorted int32 [n_total], wpre int64 [n_total] and
// n_valid_scratch [2] are then needed as extra scratch.
int b2_sketch_column(const uint32_t* keys_in, const int32_t* wq_in, uint32_t* keys_sorted, int32_t* wq_sorted, long long* wpre,
                     int64_t n_total, long long n_global, void* temp,
                     size_t temp_bytes, int32_t* flags, int32_t* idx, float* uval, long long* rmin, int32_t* m_scratch,
                     long long* n_valid_scratch, int max_bin, float* cut_out, int32_t* n_cut_out, float* min_out,
                     int32_t* has_missing_out, int num_sms, cudaStream_t s) {
  cudaError_t e;
  if (n_total > 0) {
    if (wq_in) e = cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys_in, keys_sorted, wq_in, wq_sorted, n_total, 0, 32, s);
    else e = cub::DeviceRadixSort::SortKeys(temp, temp_bytes, keys_in, keys_sorted, n_total, 0, 32, s);
    if (e != cudaSuccess) return (int)e;
    b2::head_flags_kernel<uint32_t><<<sk_grid(n_total, num_sms), 256, 0, s>>>(keys_sorted, n_total, flags);
    e = cub::DeviceScan::ExclusiveSum(temp, temp_bytes, flags, idx, n_total, s);
    if (e != cudaSuccess) return (int)e;
  }
  b2::count_valid_kernel<<<1, 32, 0, s>>>(keys_sorted, n_total, n_valid_scratch);
  if (n_total > 0) {
    if (wq_in) {
      cub::TransformInputIterator<long long, b2::CastI64, const int32_t*> it(wq_sorted, b2::CastI64());
      e = cub::DeviceScan::ExclusiveSum(temp, temp_bytes, it, wpre, n_total, s);
      if (e != cudaSuccess) return (int)e;
      b2::scatter_unique_weighted_kernel<<<sk_grid(n_total, num_sms), 256, 0, s>>>(keys_sorted, flags, idx, wpre, wq_sorted,
                                                                                  n_valid_scratch, n_total, uval, rmin, m_scratch,
                                                                                  n_valid_scratch + 1);
    } else {
      b2::scatter_unique_kernel<<<sk_grid(n_total, num_sms), 256, 0, s>>>(keys_sorted, flags, idx, n_total, uval, rmin, m_scratch);
    }
  }
  b2::prune_cuts_kernel<<<1, 256, 0, s>>>(uval, rmin, m_scratch, n_valid_scratch, (wq_in && n_total > 0) ? n_valid_scratch + 1 : nullptr,
                                         n_global, max_bin, cut_out, n_cut_out, min_out, has_missing_out);
  return (int)cudaGetLastError();
}

size_t b2_sketch_batch_temp_bytes(int64_t n) {
  size_t bytes = 0, b2 = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, n);
  cub::DeviceRadixSort::SortPairs(nullptr, b2, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr,
                                  (int32_t*)nullptr, n);
  bytes = bytes > b2 ? bytes : b2;
  cub::DeviceScan::ExclusiveSum(nullptr, b2, (const int32_t*)nullptr, (int32_t*)nullptr, n);
  bytes = bytes > b2 ? bytes : b2;
  cub::TransformInputIterator<long long, b2::CastI64, const int32_t*> it((const int32_t*)nullptr, b2::CastI64());
  cub::DeviceScan::ExclusiveSum(nullptr, b2, it, (long long*)nullptr, n);
  return bytes > b2 ? bytes : b2;
}

// Cuts of features [f0, f0 + nf) from their stored entries: keys_in [n_sort] = (j << 32) | sketch key of every valid
// entry of feature f0 + j (any order; all-ones sentinels allowed after them, they sort last), wq_in (nullable) the
// entries' integer weights.  seg [nf + 1]: feature j's entries are [seg[j], seg[j+1]) of the sorted keys, seg[nf] of
// them valid.  One sort, one summary pass over the batch and one prune block per feature.  Scratch: keys_sorted,
// wq_sorted, flags, idx, uval, rmin, wpre [n_sort].
int b2_sketch_batch(const uint64_t* keys_in, const int32_t* wq_in, uint64_t* keys_sorted, int32_t* wq_sorted, long long* wpre,
                    int64_t n_sort, const int64_t* seg, const int64_t* h_seg, int f0, int nf, const uint8_t* is_cat, int world,
                    int rank, long long n_global, void* temp, size_t temp_bytes, int32_t* flags, int32_t* idx, float* uval,
                    long long* rmin, int max_bin, float* cuts, int32_t* n_cuts, float* mins, int32_t* has_missing, int num_sms,
                    cudaStream_t s) {
  if (nf <= 0) return 0;
  const int64_t n_valid = h_seg[nf];
  int end_bit = 32;
  while (end_bit < 64 && ((int64_t)1 << (end_bit - 32)) <= nf) ++end_bit;   // the feature bits of (nf - 1) and the sentinel
  cudaError_t e;
  if (n_valid > 0) {
    if (wq_in) e = cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys_in, keys_sorted, wq_in, wq_sorted, n_sort, 0, end_bit, s);
    else e = cub::DeviceRadixSort::SortKeys(temp, temp_bytes, keys_in, keys_sorted, n_sort, 0, end_bit, s);
    if (e != cudaSuccess) return (int)e;
    b2::head_flags_kernel<uint64_t><<<sk_grid(n_valid, num_sms), 256, 0, s>>>(keys_sorted, n_valid, flags);
    e = cub::DeviceScan::ExclusiveSum(temp, temp_bytes, flags, idx, n_valid, s);
    if (e != cudaSuccess) return (int)e;
    if (wq_in) {
      cub::TransformInputIterator<long long, b2::CastI64, const int32_t*> it(wq_sorted, b2::CastI64());
      e = cub::DeviceScan::ExclusiveSum(temp, temp_bytes, it, wpre, n_valid, s);
      if (e != cudaSuccess) return (int)e;
    }
    b2::scatter_unique_segments_kernel<<<sk_grid(n_valid, num_sms), 256, 0, s>>>(keys_sorted, flags, idx, wq_in ? wpre : nullptr,
                                                                               seg, n_valid, uval, rmin);
  }
  b2::prune_cuts_segments_kernel<<<nf, 256, 0, s>>>(uval, rmin, flags, idx, wq_in ? wpre : nullptr, wq_sorted, seg, f0, is_cat, world,
                                                   rank, n_global, max_bin, cuts, n_cuts, mins, has_missing);
  return (int)cudaGetLastError();
}

int b2_launch_bin(const float* X, int64_t n, int F, float missing, const int32_t* cut_ptrs, const float* cut_vals,
                  const int32_t* feat_byte, const uint8_t* is_cat, int row_stride, uint8_t* bins, uint8_t* bins_col,
                  int64_t col_stride, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  if (F <= b2::kBinMaxF) {
    const int smem = b2::kBinTileRows * ((F | 1) * (int)sizeof(float) + row_stride + 4);
    static bool attr_set = false;
    if (!attr_set) {
      cudaFuncSetAttribute(b2::bin_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
      attr_set = true;
    }
    const int64_t n_tiles = (n + b2::kBinTileRows - 1) / b2::kBinTileRows;
    int ctas_per_sm = (220 * 1024) / (smem + 1024);
    if (ctas_per_sm > 8) ctas_per_sm = 8;
    if (ctas_per_sm < 1) ctas_per_sm = 1;
    const int grid = (int)std::min<int64_t>(n_tiles, (int64_t)num_sms * ctas_per_sm);
    b2::bin_tiled_kernel<<<grid, 256, smem, s>>>(X, n, F, missing, missing != missing ? 1 : 0, cut_ptrs, cut_vals, feat_byte,
                                                 is_cat, row_stride, bins, bins_col, col_stride);
    return (int)cudaGetLastError();
  }
  b2::bin_kernel<<<sk_grid(n * F, num_sms), 256, 0, s>>>(X, n, F, missing, missing != missing ? 1 : 0, cut_ptrs, cut_vals,
                                                        feat_byte, is_cat, row_stride, bins, bins_col, col_stride);
  return (int)cudaGetLastError();
}
int b2_launch_bin_csr(const int32_t* indices, const float* values, int64_t nnz, float missing, const int32_t* cut_ptrs,
                      const float* cut_vals, const uint8_t* is_cat, uint8_t* ebins, int num_sms, cudaStream_t s) {
  if (nnz <= 0) return 0;
  b2::bin_csr_kernel<<<sk_grid(nnz, num_sms), 256, 0, s>>>(indices, values, nnz, missing, missing != missing ? 1 : 0, cut_ptrs,
                                                          cut_vals, is_cat, ebins);
  return (int)cudaGetLastError();
}
// stats must be initialised to {-1, 0, INT_MIN} per categorical feature
int b2_launch_cat_stats(const float* X, int64_t n, int F, float missing, const int32_t* cat_feats, int n_cat, int32_t* stats,
                        int num_sms, cudaStream_t s) {
  if (n <= 0 || n_cat <= 0) return 0;
  b2::cat_stats_kernel<<<sk_grid(n * n_cat, num_sms), 256, 0, s>>>(X, n, F, missing, missing != missing ? 1 : 0, cat_feats, n_cat,
                                                                  stats);
  return (int)cudaGetLastError();
}
}
