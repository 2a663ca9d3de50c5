// refresh_kernel.cu -- the refresh updater (process_type=update, updater=refresh; DESIGN.md 2 item 20, 4.8).
//
// Re-fits the node statistics of an existing tree to the rows of the train matrix without changing its structure
// (xgboost's TreeRefresher, src/tree/updater_refresh.cc):
//   refresh_kernel        one thread walks one raw row to its leaf (b2_tree_step, the traversal predict uses), writes the
//                         compact leaf index to pos[row] and adds the row's 40-bit fixed-point (g, h) to the leaf's sums
//   refresh_nodes_kernel  one CTA: every internal node's sums bottom-up as exact limb sums of its children, then sum_hess,
//                         base_weight, loss_chg and (refresh_leaf) the leaf values, into the tree's read-back block and
//                         the leaf table margin_update_kernel reads
// The sums use the round's quantisation exponents (max |g|, |h| over all ranks), so they are exact integers that do not
// depend on row order or sharding: only the leaf sums are exchanged, every rank derives the rest itself.
#include "common.cuh"
#include "launch.h"

namespace b2 {

constexpr int kRefreshThreads = 256;
constexpr size_t kRefreshSmemNodes = 96 * 1024;   // the tree's nodes stay in shared memory up to 3,072 nodes
constexpr size_t kRefreshSmemAcc = 64 * 1024;     // per-CTA leaf accumulators up to 4,096 leaves (16 bytes each)
constexpr int64_t kRefreshCtaRows = 1 << 22;      // rows per CTA at most: 2^22 x 2^40 < 2^63 keeps every CTA total exact
constexpr int kRefreshNodeThreads = 1024;

// x += q modulo 2^64 with x kept as two 32-bit shared words (leaf_accumulate_kernel's exact int64 trick): the carry out
// of the low word is read from the value the 32-bit atomic returns
__device__ __forceinline__ void refresh_add64(uint32_t* lo, uint32_t* hi, long long q) {
  const uint32_t l = (uint32_t)(unsigned long long)q, h = (uint32_t)((unsigned long long)q >> 32);
  const uint32_t old = atomicAdd(lo, l);
  const uint32_t hadd = h + ((uint32_t)(old + l) < old ? 1u : 0u);
  if (hadd != 0u) atomicAdd(hi, hadd);
}

// nodes[i].pad holds the compact leaf index of a leaf (-1 for a split).  sums: [n_leaves][g, h][hi, lo] limbs (zeroed
// by the caller).  kSmemNodes: the nodes are copied into shared memory; kSmemAcc: each CTA sums its rows in shared
// memory and adds one total per leaf, else every row adds to the global limbs with 64-bit atomics.  A tree is a full
// binary tree (n_nodes = 2 n_leaves - 1, checked by the host), so nodes that fit in shared memory imply leaves that do.
template <bool kSmemNodes, bool kSmemAcc, typename Rows>
__global__ void __launch_bounds__(kRefreshThreads)
refresh_kernel(Rows rows, int64_t n, int F, float missing, int missing_is_nan,
               const B2TreeNodeDev* __restrict__ nodes, int n_nodes, const uint32_t* __restrict__ cat_table, int n_leaves,
               const float2* __restrict__ gh, const int32_t* __restrict__ qexp, int leaf_bits,
               uint16_t* __restrict__ pos, long long* __restrict__ sums) {
  static_assert(kSmemAcc || !kSmemNodes, "nodes in shared memory imply leaf accumulators in shared memory");
  extern __shared__ __align__(16) unsigned char smem[];
  B2TreeNodeDev* s_nodes = reinterpret_cast<B2TreeNodeDev*>(smem);
  uint32_t* s_acc = reinterpret_cast<uint32_t*>(smem + (kSmemNodes ? (size_t)n_nodes * sizeof(B2TreeNodeDev) : 0));
  if (kSmemNodes)
    for (int i = threadIdx.x; i < n_nodes; i += blockDim.x) s_nodes[i] = nodes[i];
  if (kSmemAcc)
    for (int i = threadIdx.x; i < 4 * n_leaves; i += blockDim.x) s_acc[i] = 0u;
  __syncthreads();
  const B2TreeNodeDev* tn = kSmemNodes ? s_nodes : nodes;
  uint32_t *glo = s_acc, *ghi = s_acc + n_leaves, *hlo = s_acc + 2 * n_leaves, *hhi = s_acc + 3 * n_leaves;
  const double kg = ldexp(1.0, leaf_bits - qexp[0]), kh = ldexp(1.0, leaf_bits - qexp[1]);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const auto x = b2_row(rows, i, F);
    B2TreeNodeDev nd = tn[0];
    while (nd.feature >= 0) nd = tn[b2_tree_step(nd, b2_ldg_value(x, nd.feature), missing, missing_is_nan, cat_table)];
    const int leaf = nd.pad;
    pos[i] = (uint16_t)leaf;
    const float2 v = __ldg(gh + i);
    const long long qg = __double2ll_rn(__dmul_rn((double)v.x, kg)), qh = __double2ll_rn(__dmul_rn((double)v.y, kh));
    if (kSmemAcc) {
      refresh_add64(glo + leaf, ghi + leaf, qg);
      refresh_add64(hlo + leaf, hhi + leaf, qh);
    } else {
      b2_atomic_add_limbs(&sums[4 * leaf], qg);
      b2_atomic_add_limbs(&sums[4 * leaf + 2], qh);
    }
  }
  if (!kSmemAcc) return;
  __syncthreads();
  for (int j = threadIdx.x; j < 2 * n_leaves; j += blockDim.x) {   // j = 2 * leaf + (0: g, 1: h)
    const int leaf = j >> 1;
    const uint32_t lo = (j & 1) ? hlo[leaf] : glo[leaf], hi = (j & 1) ? hhi[leaf] : ghi[leaf];
    const long long t = (long long)(((unsigned long long)hi << 32) | (unsigned long long)lo);
    if (t != 0) b2_atomic_add_limbs(&sums[2 * j], t);
  }
}

__device__ __forceinline__ double refresh_gain(const long long* l, double kg, double kh, const B2CtlParams& p) {
  const double G = __ddiv_rn(b2_limbs_to_double(l[0], l[1]), kg), H = __ddiv_rn(b2_limbs_to_double(l[2], l[3]), kh);
  return b2_calc_gain(G, H, p.mcw, p.lambda, p.alpha, p.max_delta_step);
}

// order: node ids by depth, level_ptr[d] the first of depth d (n_levels + 1 entries).  limbs: scratch [n_nodes][4].
// Read-back block: sum_hess double[n_nodes], then base_weight, loss_chg, value float[n_nodes] each.  p.eta is the
// leaf scale eta / num_parallel_tree (fp32, as the grow path's leaf_values_kernel).
__global__ void __launch_bounds__(kRefreshNodeThreads)
refresh_nodes_kernel(const B2TreeNodeDev* __restrict__ nodes, int n_nodes, const int32_t* __restrict__ order,
                     const int32_t* __restrict__ level_ptr, int n_levels, const long long* __restrict__ sums,
                     const int32_t* __restrict__ qexp, int leaf_bits, B2CtlParams p, int refresh_leaf,
                     long long* __restrict__ limbs, unsigned char* __restrict__ block, float* __restrict__ leaf_table) {
  for (int d = n_levels - 1; d >= 0; --d) {   // children before parents: a node's sums are the exact sums of its rows
    for (int idx = level_ptr[d] + threadIdx.x; idx < level_ptr[d + 1]; idx += blockDim.x) {
      const int nid = order[idx];
      const B2TreeNodeDev nd = nodes[nid];
      long long* out = limbs + 4 * (size_t)nid;
      if (nd.feature < 0) {
        for (int c = 0; c < 4; ++c) out[c] = sums[4 * (size_t)nd.pad + c];
      } else {
        const long long* a = limbs + 4 * (size_t)nd.left; const long long* b = limbs + 4 * (size_t)nd.right;
        for (int c = 0; c < 4; ++c) out[c] = a[c] + b[c];
      }
    }
    __syncthreads();
  }
  const double kg = ldexp(1.0, leaf_bits - qexp[0]), kh = ldexp(1.0, leaf_bits - qexp[1]);
  double* sum_hess = reinterpret_cast<double*>(block);
  float* base_weight = reinterpret_cast<float*>(block + (size_t)n_nodes * 8);
  float* loss_chg = base_weight + n_nodes;
  float* value = loss_chg + n_nodes;
  for (int nid = threadIdx.x; nid < n_nodes; nid += blockDim.x) {
    const B2TreeNodeDev nd = nodes[nid];
    const long long* l = limbs + 4 * (size_t)nid;
    const double G = __ddiv_rn(b2_limbs_to_double(l[0], l[1]), kg), H = __ddiv_rn(b2_limbs_to_double(l[2], l[3]), kh);
    const float w = __double2float_rn(b2_calc_weight(G, H, p.mcw, p.lambda, p.alpha, p.max_delta_step));
    sum_hess[nid] = H;
    base_weight[nid] = w;
    if (nd.feature >= 0) {
      const double gl = refresh_gain(limbs + 4 * (size_t)nd.left, kg, kh, p);
      const double gr = refresh_gain(limbs + 4 * (size_t)nd.right, kg, kh, p);
      const double gp = b2_calc_gain(G, H, p.mcw, p.lambda, p.alpha, p.max_delta_step);
      loss_chg[nid] = __double2float_rn(__dadd_rn(__dadd_rn(gl, gr), -gp));
      value[nid] = w;
    } else {
      const float v = refresh_leaf ? __fmul_rn(w, p.eta) : nd.value;
      loss_chg[nid] = 0.0f;
      value[nid] = v;
      leaf_table[nd.pad] = v;
    }
  }
}

}  // namespace b2

extern "C" {
int b2_launch_refresh(B2RawRows src, int64_t n, int F, float missing, const B2TreeNodeDev* nodes, int n_nodes,
                      const uint32_t* cat_table, int n_leaves, const float2* gh, const int32_t* qexp, int leaf_bits,
                      uint16_t* pos, long long* sums, int num_sms, cudaStream_t stream) {
  if (n <= 0) return 0;
  const bool smem_acc = (size_t)n_leaves * 16 <= b2::kRefreshSmemAcc;
  const bool smem_nodes = smem_acc && (size_t)n_nodes * sizeof(B2TreeNodeDev) <= b2::kRefreshSmemNodes;
  const size_t smem = (smem_nodes ? (size_t)n_nodes * sizeof(B2TreeNodeDev) : 0) + (smem_acc ? (size_t)n_leaves * 16 : 0);
  const int64_t want = (n + b2::kRefreshThreads - 1) / b2::kRefreshThreads;
  int64_t cap = (int64_t)num_sms * 8;
  const int64_t exact_min = (n + b2::kRefreshCtaRows - 1) / b2::kRefreshCtaRows;
  if (cap < exact_min) cap = exact_min;
  const int grid = (int)(want < cap ? want : cap);
  const int missing_is_nan = isnan(missing) ? 1 : 0;
#define B2_REFRESH_LAUNCH(N, A, R, ROWS)                                                                                \
  do {                                                                                                                  \
    auto k = b2::refresh_kernel<N, A, R>;                                                                               \
    if (smem > 48 * 1024) {                                                                                             \
      const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);           \
      if (e != cudaSuccess) return (int)e;                                                                              \
    }                                                                                                                   \
    k<<<grid, b2::kRefreshThreads, smem, stream>>>(ROWS, n, F, missing, missing_is_nan, nodes, n_nodes, cat_table,        \
                                                   n_leaves, gh, qexp, leaf_bits, pos, sums);                           \
  } while (0)
#define B2_REFRESH_ROWS(R, ROWS)                                       \
  do {                                                                 \
    if (smem_nodes) B2_REFRESH_LAUNCH(true, true, R, ROWS);            \
    else if (smem_acc) B2_REFRESH_LAUNCH(false, true, R, ROWS);        \
    else B2_REFRESH_LAUNCH(false, false, R, ROWS);                     \
  } while (0)
  if (src.indptr) B2_REFRESH_ROWS(B2CsrRows, (B2CsrRows{src.indptr, src.indices, src.values}));
  else B2_REFRESH_ROWS(B2DenseRows, src.X);
#undef B2_REFRESH_ROWS
#undef B2_REFRESH_LAUNCH
  return (int)cudaGetLastError();
}
int b2_launch_refresh_nodes(const B2TreeNodeDev* nodes, int n_nodes, const int32_t* order, const int32_t* level_ptr, int n_levels,
                            const long long* sums, const int32_t* qexp, int leaf_bits, B2CtlParams p, int refresh_leaf,
                            long long* limbs, unsigned char* block, float* leaf_table, cudaStream_t stream) {
  b2::refresh_nodes_kernel<<<1, b2::kRefreshNodeThreads, 0, stream>>>(nodes, n_nodes, order, level_ptr, n_levels, sums, qexp,
                                                                       leaf_bits, p, refresh_leaf, limbs, block, leaf_table);
  return (int)cudaGetLastError();
}
}
