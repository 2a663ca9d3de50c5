// shap_kernel.cu -- SHAP contributions, SHAP interaction values and leaf indices on raw floats.
//
// Replaces what the reference reaches through model.predict(local_data, pred_contribs=True / pred_interactions=True /
// pred_leaf=True) at xgboost_ray/main.py:804 (xgboost's RegTree::CalculateContributions / TreeShap).
//
// Algorithm: exact path-dependent TreeSHAP (Lundberg et al. 2018) on the path table of common.cuh (one path per leaf,
// repeated features merged), in the warp-parallel form of GPUTreeShap (Mitchell et al. 2022): the lanes of a path hold
// its elements, the EXTEND recurrence runs across them with shuffles, and every lane then UNWINDS its own element.
//
// Warp mapping and determinism (DESIGN.md 4.6): a warp owns one row at a time and walks the path list of the tree
// range in order.  Paths of at most 16 elements go two at a time (half-warps of 16 lanes); a path of 17..32 elements
// (max_depth 16, or a deep model loaded from JSON) takes the whole warp on its own, and so does a short path whose
// successor is long.  Which width a path runs at depends only on the path table, and a path's values do not depend on
// it: lanes past its length never change the recurrences.  Contributions are accumulated in double in the warp's own
// accumulator -- shared memory for pred_contribs, the row's slice of a global scratch block for interactions (up to
// K (F+1)^2 doubles, far beyond shared memory) -- by plain read-modify-writes in a fixed order (half 0 before half 1,
// path after path), so the result is bit-identical from call to call and independent of how rows are sharded.  There
// are no atomics; each output value is written once per row.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "common.cuh"
#include "launch.h"

namespace b2 {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kHalf = 16;

// 1 if row x satisfies every merged split of the element, else 0
__device__ __forceinline__ double path_one_fraction(const B2PathElem& e, const float* __restrict__ x, float missing,
                                                    int missing_is_nan, const uint32_t* __restrict__ cat_table) {
  if (e.feature < 0) return 1.0;
  const float v = x[e.feature];
  const bool miss = isnan(v) || (!missing_is_nan && v == missing);
  if (miss) return (e.flags & B2_PATH_MISSING_OK) ? 1.0 : 0.0;
  if (e.cat_slot >= 0) {
    if (v >= 0.0f && v < 256.0f) {
      const int c = (int)v;
      return ((cat_table[(size_t)e.cat_slot * 8 + (c >> 5)] >> (c & 31)) & 1u) ? 1.0 : 0.0;
    }
    return (e.flags & B2_PATH_OUTSIDE_OK) ? 1.0 : 0.0;
  }
  return (v >= e.lo && (!(e.flags & B2_PATH_HAS_HI) || v < e.hi)) ? 1.0 : 0.0;
}

// EXTEND over elements 1..L-1 of this W-lane group's path (element 0, the bias, starts the path with weight 1), leaving
// out element `skip` (-1: none).  Lane s returns the permutation weight of position s; positions are compacted past
// `skip`.  Every lane of the warp calls this with the same Lmax = max(L) of the warp's groups.
template <int W>
__device__ __forceinline__ double path_extend(int sub, int L, int Lmax, double z, double o, int skip) {
  double w = sub == 0 ? 1.0 : 0.0;
  int pos = 0;
  for (int l = 1; l < Lmax; ++l) {
    const double zl = __shfl_sync(kFull, z, l, W), ol = __shfl_sync(kFull, o, l, W);
    const double wl = __shfl_up_sync(kFull, w, 1, W);
    if (l < L && l != skip) {
      ++pos;
      if (sub <= pos)
        w = w * zl * (double)(pos - sub) / (double)(pos + 1) + (sub > 0 ? wl * ol * (double)sub / (double)(pos + 1) : 0.0);
    }
  }
  return w;
}

// UNWOUND_PATH_SUM: total permutation weight of the path with this lane's element (z, o) removed, given the weights
// w of the Lp positions.  A lane whose element has o = z = 0 contributes nothing and returns 0 (never 0/0).
template <int W>
__device__ __forceinline__ double path_unwound_sum(int Lp, int Lpmax, double w, double z, double o, bool active) {
  const int l = Lp - 1;
  double next = __shfl_sync(kFull, w, l < 0 ? 0 : l, W);
  double total = 0.0;
  for (int j = Lpmax - 2; j >= 0; --j) {
    const double wj = __shfl_sync(kFull, w, j, W);
    if (active && j < l) {
      if (o != 0.0) {
        const double t = next * (double)(l + 1) / ((double)(j + 1) * o);
        total += t;
        next = wj - t * z * (double)(l - j) / (double)(l + 1);
      } else if (z != 0.0) {
        total += wj / z / ((double)(l - j) / (double)(l + 1));
      }
    }
  }
  return total;
}

struct PathLane {
  B2PathElem e;
  int L, cls;
  double v, z, o;
};

__device__ __forceinline__ PathLane load_path_lane(const B2PathElem* __restrict__ elems, const B2PathInfo* __restrict__ paths,
                                                   int q, int p_end, int sub, const float* __restrict__ x, float missing,
                                                   int missing_is_nan, const uint32_t* __restrict__ cat_table) {
  PathLane r;
  r.L = 0; r.cls = 0; r.v = 0.0; r.z = 0.0; r.o = 0.0;
  r.e.feature = -1; r.e.cat_slot = -1; r.e.lo = 0.0f; r.e.hi = 0.0f; r.e.flags = 0; r.e.pad = 0; r.e.zero_fraction = 0.0;
  if (q < p_end) {
    const B2PathInfo pi = paths[q];
    r.L = pi.len; r.cls = pi.cls; r.v = pi.value;
    if (sub < r.L) {
      r.e = elems[pi.elem_begin + sub];
      r.z = r.e.zero_fraction;
      r.o = path_one_fraction(r.e, x, missing, missing_is_nan, cat_table);
    }
  }
  return r;
}

// How the warp takes the paths from p on: 0 = path p alone on the full warp (more than 16 elements), 2 = paths p and
// p + 1 on the two half-warps, 1 = path p on half 0 alone (the next path is long, or p is the last).  Warp-uniform.
__device__ __forceinline__ int path_step(const B2PathInfo* __restrict__ paths, int p, int p_end) {
  if (paths[p].len > kHalf) return 0;
  return p + 1 < p_end && paths[p + 1].len <= kHalf ? 2 : 1;
}

// phi of one path per W-lane group (W = 16: group `part` of the warp holds path q; W = 32: part 0, the whole warp),
// added to the row accumulator group by group in path order
template <int W>
__device__ __forceinline__ void contribs_path(double* acc, int F1, const B2PathElem* __restrict__ elems,
                                              const B2PathInfo* __restrict__ paths, int q, int q_end, int sub, int part,
                                              const float* __restrict__ x, float missing, int missing_is_nan,
                                              const uint32_t* __restrict__ cat_table) {
  const PathLane pl = load_path_lane(elems, paths, q, q_end, sub, x, missing, missing_is_nan, cat_table);
  const int Lmax = W == 32 ? pl.L : max(pl.L, __shfl_xor_sync(kFull, pl.L, 16));
  const double w = path_extend<W>(sub, pl.L, Lmax, pl.z, pl.o, -1);
  const bool mine = sub > 0 && sub < pl.L;
  const double s = path_unwound_sum<W>(pl.L, Lmax, w, pl.z, pl.o, mine);
  const double c = s * (pl.o - pl.z) * pl.v;
#pragma unroll
  for (int h = 0; h < 32 / W; ++h) {
    if (part == h && mine) acc[pl.cls * F1 + pl.e.feature] += c;
    __syncwarp();
  }
}

// Phi_ij of one path per W-lane group, as contribs_path: phi_i on the diagonal, then the conditioning elements in order
template <int W>
__device__ __forceinline__ void interactions_path(double* acc, size_t mat, int F1, const B2PathElem* __restrict__ elems,
                                                  const B2PathInfo* __restrict__ paths, int q, int q_end, int sub, int part,
                                                  const float* __restrict__ x, float missing, int missing_is_nan,
                                                  const uint32_t* __restrict__ cat_table) {
  const PathLane pl = load_path_lane(elems, paths, q, q_end, sub, x, missing, missing_is_nan, cat_table);
  const int Lmax = W == 32 ? pl.L : max(pl.L, __shfl_xor_sync(kFull, pl.L, 16));
  const bool mine = sub > 0 && sub < pl.L;
  double* accc = acc + (size_t)pl.cls * mat;
  {   // phi_i of the full path, kept on the diagonal until the final correction
    const double w = path_extend<W>(sub, pl.L, Lmax, pl.z, pl.o, -1);
    const double c = path_unwound_sum<W>(pl.L, Lmax, w, pl.z, pl.o, mine) * (pl.o - pl.z) * pl.v;
#pragma unroll
    for (int h = 0; h < 32 / W; ++h) {
      if (part == h && mine) accc[(size_t)pl.e.feature * F1 + pl.e.feature] += c;
      __syncwarp();
    }
  }
  for (int cc = 1; cc < Lmax; ++cc) {
    const bool has_c = cc < pl.L;
    const double zc = __shfl_sync(kFull, pl.z, cc, W), oc = __shfl_sync(kFull, pl.o, cc, W);
    const int fc = __shfl_sync(kFull, pl.e.feature, cc, W);
    const int Lp = has_c ? pl.L - 1 : 0;
    const int Lpmax = W == 32 ? Lp : max(Lp, __shfl_xor_sync(kFull, Lp, 16));
    const double w = path_extend<W>(sub, has_c ? pl.L : 0, Lmax, pl.z, pl.o, cc);
    const bool act = has_c && mine && sub != cc;
    const double s = path_unwound_sum<W>(Lp, Lpmax, w, pl.z, pl.o, act);
    const double val = 0.5 * s * (pl.o - pl.z) * pl.v * (oc - zc);
#pragma unroll
    for (int h = 0; h < 32 / W; ++h) {
      if (part == h && act) accc[(size_t)fc * F1 + pl.e.feature] += val;
      __syncwarp();
    }
  }
}

// pred_contribs: out [rows][K][F+1] (float), row r of the block is global row row0 + r
__global__ void __launch_bounds__(256) shap_contribs_kernel(
    const float* __restrict__ X, int64_t row0, int64_t rows, int F, float missing, int missing_is_nan,
    const B2PathElem* __restrict__ elems, const B2PathInfo* __restrict__ paths, int p_begin, int p_end,
    const uint32_t* __restrict__ cat_table, int K, const double* __restrict__ bias_k, const float* __restrict__ base_margin,
    float base_value, double* __restrict__ gacc, int acc_in_smem, float* __restrict__ out) {
  extern __shared__ double smem_acc[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane & 15, half = lane >> 4;
  const int F1 = F + 1, stride = K * F1;
  const int64_t warps_total = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp; r < rows; r += warps_total) {
    double* acc = acc_in_smem ? smem_acc + (size_t)warp * stride : gacc + (size_t)r * stride;
    const int64_t row = row0 + r;
    const float* x = X + row * F;
    for (int i = lane; i < stride; i += 32) {
      const int k = i / F1, f = i - k * F1;
      acc[i] = f == F ? (double)(base_margin ? base_margin[row * K + k] : base_value) + bias_k[k] : 0.0;
    }
    __syncwarp();
    for (int p = p_begin; p < p_end;) {
      const int step = path_step(paths, p, p_end);
      if (step == 0) {
        contribs_path<32>(acc, F1, elems, paths, p, p + 1, lane, 0, x, missing, missing_is_nan, cat_table);
        p += 1;
      } else {
        contribs_path<kHalf>(acc, F1, elems, paths, p + half, p + step, sub, half, x, missing, missing_is_nan, cat_table);
        p += step;
      }
    }
    for (int i = lane; i < stride; i += 32) out[r * stride + i] = (float)acc[i];
    __syncwarp();
  }
}

// pred_interactions: out [rows][K][F+1][F+1] (float); gacc [rows][K][F+1][F+1] doubles of scratch.
//   Phi_ij (i != j < F) = 1/2 (phi_j | i present - phi_j | i absent): for every conditioning element c of a path, the
//   path without c is extended and unwound, and the contributions are scaled by one_fraction_c (present) and
//   zero_fraction_c (absent).  Phi_ii = phi_i - sum_{j != i} Phi_ij; the bias row / column is 0 except Phi_FF = bias.
__global__ void __launch_bounds__(256) shap_interactions_kernel(
    const float* __restrict__ X, int64_t row0, int64_t rows, int F, float missing, int missing_is_nan,
    const B2PathElem* __restrict__ elems, const B2PathInfo* __restrict__ paths, int p_begin, int p_end,
    const uint32_t* __restrict__ cat_table, int K, const double* __restrict__ bias_k, const float* __restrict__ base_margin,
    float base_value, double* __restrict__ gacc, float* __restrict__ out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane & 15, half = lane >> 4;
  const int F1 = F + 1;
  const size_t mat = (size_t)F1 * F1, stride = (size_t)K * mat;
  const int64_t warps_total = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp; r < rows; r += warps_total) {
    double* acc = gacc + (size_t)r * stride;
    const int64_t row = row0 + r;
    const float* x = X + row * F;
    for (size_t i = lane; i < stride; i += 32) acc[i] = 0.0;
    __syncwarp();
    for (int k = lane; k < K; k += 32)
      acc[k * mat + (size_t)F * F1 + F] = (double)(base_margin ? base_margin[row * K + k] : base_value) + bias_k[k];
    __syncwarp();
    for (int p = p_begin; p < p_end;) {
      const int step = path_step(paths, p, p_end);
      if (step == 0) {
        interactions_path<32>(acc, mat, F1, elems, paths, p, p + 1, lane, 0, x, missing, missing_is_nan, cat_table);
        p += 1;
      } else {
        interactions_path<kHalf>(acc, mat, F1, elems, paths, p + half, p + step, sub, half, x, missing, missing_is_nan,
                                 cat_table);
        p += step;
      }
    }
    for (int i = lane; i < K * F; i += 32) {
      const int k = i / F, f = i - k * F;
      double* rowp = acc + (size_t)k * mat + (size_t)f * F1;
      double off = 0.0;
      for (int j = 0; j < F; ++j) if (j != f) off += rowp[j];
      rowp[f] -= off;
    }
    __syncwarp();
    float* o = out + (size_t)r * stride;
    for (size_t i = lane; i < stride; i += 32) o[i] = (float)acc[i];
    __syncwarp();
  }
}

// pred_leaf: out [rows][tree_end - tree_begin] = node id of the leaf the row reaches (b2_tree_leaf, as predict_kernel)
template <typename Rows>
__global__ void leaf_index_kernel(Rows src, int64_t row0, int64_t rows, int F, float missing, int missing_is_nan,
                                  const B2TreeNodeDev* __restrict__ nodes, const int32_t* __restrict__ tree_offset,
                                  const uint32_t* __restrict__ cat_table, int tree_begin, int tree_end, float* __restrict__ out) {
  const int T = tree_end - tree_begin;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < rows * T; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / T;
    const int t = tree_begin + (int)(i - r * T);
    float v;
    out[i] = (float)b2_tree_leaf(nodes + tree_offset[t], b2_row(src, row0 + r, F), missing, missing_is_nan, cat_table, &v);
  }
}

}  // namespace b2

extern "C" {
// shared memory a contributions block needs for `warps` row accumulators; 0 = they go to global scratch
size_t b2_shap_contribs_smem(int K, int F, int warps) { return (size_t)warps * K * (F + 1) * sizeof(double); }

int b2_launch_shap_contribs(const float* X, int64_t row0, int64_t rows, int F, float missing, const B2PathElem* elems,
                            const B2PathInfo* paths, int p_begin, int p_end, const uint32_t* cat_table, int K,
                            const double* bias_k, const float* base_margin, float base_value, double* gacc, int warps,
                            size_t smem, float* out, int num_sms, cudaStream_t s) {
  if (rows <= 0) return 0;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(b2::shap_contribs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
  }
  int64_t g = (rows + warps - 1) / warps;
  const int64_t cap = (int64_t)num_sms * (warps <= 2 ? 16 : 8);
  if (g > cap) g = cap;
  b2::shap_contribs_kernel<<<(int)g, warps * 32, smem, s>>>(X, row0, rows, F, missing, missing != missing ? 1 : 0, elems, paths,
                                                              p_begin, p_end, cat_table, K, bias_k, base_margin, base_value, gacc,
                                                              smem > 0 ? 1 : 0, out);
  return (int)cudaGetLastError();
}

int b2_launch_shap_interactions(const float* X, int64_t row0, int64_t rows, int F, float missing, const B2PathElem* elems,
                                const B2PathInfo* paths, int p_begin, int p_end, const uint32_t* cat_table, int K,
                                const double* bias_k, const float* base_margin, float base_value, double* gacc, float* out,
                                int num_sms, cudaStream_t s) {
  if (rows <= 0) return 0;
  int64_t g = (rows + 7) / 8;
  const int64_t cap = (int64_t)num_sms * 8;
  if (g > cap) g = cap;
  b2::shap_interactions_kernel<<<(int)g, 256, 0, s>>>(X, row0, rows, F, missing, missing != missing ? 1 : 0, elems, paths, p_begin,
                                                     p_end, cat_table, K, bias_k, base_margin, base_value, gacc, out);
  return (int)cudaGetLastError();
}

int b2_launch_leaf_index(B2RawRows src, int64_t row0, int64_t rows, int F, float missing, const B2TreeNodeDev* nodes,
                         const int32_t* tree_offset, const uint32_t* cat_table, int tree_begin, int tree_end, float* out,
                         int num_sms, cudaStream_t s) {
  if (rows <= 0 || tree_end <= tree_begin) return 0;
  int64_t g = (rows * (tree_end - tree_begin) + 255) / 256;
  const int64_t cap = (int64_t)num_sms * 16;
  if (g > cap) g = cap;
  const int mnan = missing != missing ? 1 : 0;
  if (src.indptr)
    b2::leaf_index_kernel<<<(int)g, 256, 0, s>>>(B2CsrRows{src.indptr, src.indices, src.values}, row0, rows, F, missing, mnan, nodes,
                                                 tree_offset, cat_table, tree_begin, tree_end, out);
  else
    b2::leaf_index_kernel<B2DenseRows><<<(int)g, 256, 0, s>>>(src.X, row0, rows, F, missing, mnan, nodes, tree_offset, cat_table,
                                                 tree_begin, tree_end, out);
  return (int)cudaGetLastError();
}
}
