// dart_kernel.cu -- DART (booster=dart) margin rebuild on the bin matrix of the training rows.
//
// Before a round that drops trees, every training row needs two margins built from the whole model:
//   drop[c] = base + sum over the KEPT trees t of class c, in tree order, of fl(w_old[t] * leaf_t)   (gradients)
//   full[c] = base + sum over ALL old trees t of class c, in tree order, of fl(w_new[t] * leaf_t)    (the prefix the
//             round's new trees are then added to by the leaf pass, margin_update_kernel)
// One traversal yields both.  Every add is m = fl(m + fl(w * v)): a separate multiply and add (built with
// --fmad=false), the same sequence the weighted predict_kernel and the CPU reference use, so the margins are bit-equal.
//
// The walk reads bins, not floats (the raw matrix is usually released after quantisation): a numeric node goes left iff
// bin <= split_bin (B2TreeNodeDev::pad), the missing bin of a feature with missing values follows the default
// direction, a categorical node sends the codes in its set right.  A CTA stages the bin rows of its 128 rows in shared
// memory (one coalesced copy; the row pitch is padded by one word so that threads reading the same feature hit
// different banks) while the tree nodes stream through L1 / L2; rows too wide for shared memory read the bins from
// global memory instead.
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "launch.h"

namespace b2 {

constexpr int kDartRows = 128;                       // rows (threads) per CTA
constexpr size_t kDartMaxSmem = (size_t)200 * 1024;  // staged tile limit (227 KB per CTA on sm_90)

// one step of the bin-space walk from node nd, where b is the row's bin of nd.feature
__device__ __forceinline__ int dart_step(const B2TreeNodeDev& nd, int b, const uint8_t* __restrict__ has_missing,
                                         const uint32_t* __restrict__ cat_table) {
  if (b == B2_MISSING_BIN && __ldg(has_missing + nd.feature)) return nd.default_left ? nd.left : nd.right;
  if (nd.cat_slot >= 0) return ((__ldg(cat_table + (size_t)nd.cat_slot * 8 + (b >> 5)) >> (b & 31)) & 1u) ? nd.right : nd.left;
  return b <= nd.pad ? nd.left : nd.right;
}

// tree t's leaf value v added to the margins of row i: drop when the tree is kept, full always
__device__ __forceinline__ void dart_add(int64_t i, int t, float v, bool keep, int K, int npt, const float* __restrict__ w_drop,
                                         const float* __restrict__ w_full, float* __restrict__ drop, float* __restrict__ full) {
  const int64_t o = i * K + (t / npt) % K;
  if (keep) drop[o] = __fadd_rn(drop[o], __fmul_rn(__ldg(w_drop + t), v));
  full[o] = __fadd_rn(full[o], __fmul_rn(__ldg(w_full + t), v));
}

template <bool kSmem, bool kSingle>
__global__ void __launch_bounds__(kDartRows)
dart_margins_kernel(const uint8_t* __restrict__ bins, int64_t n, int row_stride, const int32_t* __restrict__ feat_byte,
                    const uint8_t* __restrict__ has_missing, const B2TreeNodeDev* __restrict__ nodes,
                    const int32_t* __restrict__ tree_offset, const uint32_t* __restrict__ cat_table, int T, int K, int npt,
                    const float* __restrict__ w_drop, const uint8_t* __restrict__ dropped, const float* __restrict__ w_full,
                    float* __restrict__ drop /* nullable: full margin only */, float* __restrict__ full) {
  extern __shared__ uint32_t s_tile[];
  const int words = row_stride >> 2, pitch = words + 1;   // row_stride is a multiple of 32 bytes
  for (int64_t row0 = (int64_t)blockIdx.x * kDartRows; row0 < n; row0 += (int64_t)gridDim.x * kDartRows) {
    const int rows = (int)(n - row0 < kDartRows ? n - row0 : kDartRows);
    const int64_t i = row0 + threadIdx.x;
    const uint8_t* row;
    if (kSmem) {
      __syncthreads();   // the previous tile is no longer read
      const uint32_t* src = (const uint32_t*)(bins + row0 * row_stride);
      for (int w = threadIdx.x; w < rows * words; w += kDartRows) s_tile[(w / words) * pitch + (w % words)] = __ldg(src + w);
      __syncthreads();
      row = (const uint8_t*)(s_tile + threadIdx.x * pitch);
    } else {
      row = bins + i * row_stride;
    }
    if (threadIdx.x >= rows) continue;
    float d1 = kSingle ? (drop ? drop[i] : 0.0f) : 0.0f, f1 = kSingle ? full[i] : 0.0f;
    for (int t = 0; t < T; ++t) {
      const B2TreeNodeDev* tn = nodes + __ldg(tree_offset + t);
      B2TreeNodeDev nd = tn[0];
      while (nd.feature >= 0) {
        const int b = kSmem ? row[__ldg(feat_byte + nd.feature)] : __ldg(row + __ldg(feat_byte + nd.feature));
        nd = tn[dart_step(nd, b, has_missing, cat_table)];
      }
      const float v = nd.value;
      const bool keep = drop && !__ldg(dropped + t);
      if (kSingle) {
        if (keep) d1 = __fadd_rn(d1, __fmul_rn(__ldg(w_drop + t), v));
        f1 = __fadd_rn(f1, __fmul_rn(__ldg(w_full + t), v));
      } else {
        dart_add(i, t, v, keep, K, npt, w_drop, w_full, drop, full);
      }
    }
    if (kSingle) {
      if (drop) drop[i] = d1;
      full[i] = f1;
    }
  }
}

// CSR bin layout: one thread per row, the bin of a node's feature found in the row's stored entries (b2_csr_bin)
__global__ void __launch_bounds__(kDartRows)
dart_margins_csr_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const uint8_t* __restrict__ ebins,
                        int64_t n, const uint8_t* __restrict__ has_missing, const B2TreeNodeDev* __restrict__ nodes,
                        const int32_t* __restrict__ tree_offset, const uint32_t* __restrict__ cat_table, int T, int K, int npt,
                        const float* __restrict__ w_drop, const uint8_t* __restrict__ dropped, const float* __restrict__ w_full,
                        float* __restrict__ drop, float* __restrict__ full) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    for (int t = 0; t < T; ++t) {
      const B2TreeNodeDev* tn = nodes + __ldg(tree_offset + t);
      B2TreeNodeDev nd = tn[0];
      while (nd.feature >= 0) nd = tn[dart_step(nd, b2_csr_bin(indptr, indices, ebins, i, nd.feature), has_missing, cat_table)];
      dart_add(i, t, nd.value, drop && !__ldg(dropped + t), K, npt, w_drop, w_full, drop, full);
    }
  }
}

}  // namespace b2

extern "C" {
// drop / full hold the starting margins (base_score or base_margin) on entry.  dropped[t] != 0: tree t is left out of
// drop.  drop == nullptr rebuilds the full margin only (w_drop / dropped unused).
int b2_launch_dart_margins(B2BinRows src, int64_t n, const uint8_t* has_missing, const B2TreeNodeDev* nodes,
                           const int32_t* tree_offset, const uint32_t* cat_table, int T, int K, int npt, const float* w_drop,
                           const uint8_t* dropped, const float* w_full, float* drop, float* full, int num_sms, cudaStream_t s) {
  if (n <= 0 || T <= 0) return 0;
  if (npt < 1) npt = 1;
  const int64_t tiles = (n + b2::kDartRows - 1) / b2::kDartRows;
  const int64_t cap = (int64_t)num_sms * 16;
  const int grid = (int)(tiles < cap ? tiles : cap);
  if (src.ebins) {
    b2::dart_margins_csr_kernel<<<grid, b2::kDartRows, 0, s>>>(src.indptr, src.indices, src.ebins, n, has_missing, nodes,
                                                              tree_offset, cat_table, T, K, npt, w_drop, dropped, w_full, drop,
                                                              full);
    return (int)cudaGetLastError();
  }
  const uint8_t* bins = src.bins; const int row_stride = src.row_stride; const int32_t* feat_byte = src.feat_byte;
  if (row_stride <= 0 || (row_stride & 31)) return (int)cudaErrorInvalidValue;
  const size_t smem = (size_t)b2::kDartRows * (size_t)(row_stride / 4 + 1) * 4;
  const bool single = K == 1;
#define B2_DART_LAUNCH(SMEM, SINGLE, BYTES)                                                                                  \
  b2::dart_margins_kernel<SMEM, SINGLE><<<grid, b2::kDartRows, BYTES, s>>>(bins, n, row_stride, feat_byte, has_missing,   \
                                                                          nodes, tree_offset, cat_table, T, K, npt,      \
                                                                          w_drop, dropped, w_full, drop, full)
  if (smem <= b2::kDartMaxSmem) {
    const int e = single ? (int)cudaFuncSetAttribute(b2::dart_margins_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                         : (int)cudaFuncSetAttribute(b2::dart_margins_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e) return e;
    if (single) B2_DART_LAUNCH(true, true, smem);
    else B2_DART_LAUNCH(true, false, smem);
  } else {
    if (single) B2_DART_LAUNCH(false, true, 0);
    else B2_DART_LAUNCH(false, false, 0);
  }
#undef B2_DART_LAUNCH
  return (int)cudaGetLastError();
}
}
