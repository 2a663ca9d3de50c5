// control_kernel.cu -- device-side tree bookkeeping so that growing a tree needs no host round trip.
//
// What xgboost's driver loop does on the host between the per-level kernels (src/tree/driver.h,
// updater_quantile_hist.cc: pick the best candidate, decide expand-or-leaf, allocate child ids in
// node order, choose the smaller-hessian child to build, emit work lists) is done here by single-CTA
// kernels that read and write device-resident tables.  The host enqueues the same fixed launch
// sequence for every tree and reads the finished tree back once (SURVEY.md 3.1 "host hot spots").
// All arithmetic that influences the model is IEEE fp64/fp32 with explicit rounding, identical to
// the oracle's host formulas (Appendix A.6/A.7).
#include <string.h>

#include "common.cuh"
#include "decide.cuh"
#include "launch.h"

namespace b2 {

constexpr int kCtlThreads = 1024;
constexpr int kPartChunkRows = 2048;   // leaf-segment work items; must match partition_kernel.cu kPartChunk

__device__ __forceinline__ float c_calc_weight(double G, double H, const B2CtlParams& p) {
  return __double2float_rn(b2_calc_weight(G, H, p.mcw, p.lambda, p.alpha, p.max_delta_step));
}

// ---- decide as its own launch: the NCCL and peer-memory exchanges (the candidates of all ranks are needed), matrices
// with categorical features (their scan runs after the numeric one) and the last level (no scan)
__global__ void __launch_bounds__(kCtlThreads)
decide_kernel(B2DecideArgs a, int use_p2p, B2P2P pp) {
  __shared__ DecideScratch<kCtlThreads> sm;
  decide_block<kCtlThreads>(sm, a, use_p2p != 0, pp);
}

// ---- leaves: chunked work list over the leaf segments
__global__ void __launch_bounds__(kCtlThreads)
leaf_plan_kernel(const B2LeafDev* __restrict__ leaves, const int32_t* __restrict__ n_leaves, B2SegWork* __restrict__ work,
                 B2LevelCtl* __restrict__ leaf_ctl) {
  __shared__ typename TileScan<kCtlThreads>::Scan::TempStorage tmp;
  const int n = *n_leaves;
  TileScan<kCtlThreads> scan(&tmp);
  for (int base = 0; base < n; base += kCtlThreads) {
    const int i = base + threadIdx.x;
    int chunks = 0; B2LeafDev lf; lf.nid = 0; lf.buf = 0; lf.begin = 0; lf.count = 0;
    if (i < n) { lf = leaves[i]; chunks = (lf.count + kPartChunkRows - 1) / kPartChunkRows; }
    const int cb = scan.step(chunks);
    if (i < n) {
      B2SegWork w; w.seg_begin = lf.begin; w.seg_count = lf.count; w.id = i; w.chunk_begin = cb; w.buf = lf.buf;
      w.pad0 = lf.nid == 0 ? 1 : 0;   // the root as a leaf: its rows are the identity list (no index list was ever written)
      w.pad1 = w.pad2 = 0; work[i] = w;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) { leaf_ctl->hist_n_work = n; leaf_ctl->hist_total_chunks = scan.carry; }
}

// leaf weight from the 40-bit fixed-point sums (A.7 leaf refinement; two limbs each, common.cuh), value = weight * eta (fp32); also keeps the
// tree's quantisation exponents in its read-back block (qexp_out)
__global__ void leaf_values_kernel(const B2LeafDev* __restrict__ leaves, const int32_t* __restrict__ n_leaves,
                                   const long long* __restrict__ sums, const int32_t* __restrict__ qexp, int leaf_bits,
                                   B2CtlParams p, float* __restrict__ leaf_value, B2TreeDev tree, int32_t* __restrict__ qexp_out) {
  const int n = *n_leaves;
  if (blockIdx.x == 0 && threadIdx.x < 2) qexp_out[threadIdx.x] = qexp[threadIdx.x];
  const double kg = ldexp(1.0, leaf_bits - qexp[0]), kh = ldexp(1.0, leaf_bits - qexp[1]);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const long long* s = sums + 4 * i;   // [g, h][hi, lo]
    const double G = __ddiv_rn(b2_limbs_to_double(s[0], s[1]), kg), H = __ddiv_rn(b2_limbs_to_double(s[2], s[3]), kh);
    const float w = c_calc_weight(G, H, p);
    const float v = __fmul_rn(w, p.eta);
    leaf_value[i] = v;
    tree.leaf_weight[leaves[i].nid] = w;
    tree.leaf_value[leaves[i].nid] = v;
  }
}

// vector-leaf tree: leaf i's value of target k from target k's 40-bit sums (sums + k * sums_stride, exponents qexp[2k..])
// -> leaf_vec[i][k] (the margin update's table) and tree_vec[nid][k] (the read-back block); also keeps the T exponent
// pairs in the read-back block (qexp_out)
__global__ void vector_leaf_values_kernel(const B2LeafDev* __restrict__ leaves, const int32_t* __restrict__ n_leaves,
                                          const long long* __restrict__ sums, size_t sums_stride, const int32_t* __restrict__ qexp,
                                          int T, int leaf_bits, B2CtlParams p, float* __restrict__ leaf_vec,
                                          float* __restrict__ tree_vec, int32_t* __restrict__ qexp_out) {
  const int n = *n_leaves;
  if (blockIdx.x == 0)
    for (int t = threadIdx.x; t < 2 * T; t += blockDim.x) qexp_out[t] = qexp[t];
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n * T; idx += gridDim.x * blockDim.x) {
    const int i = idx / T, k = idx - i * T;
    const long long* s = sums + (size_t)k * sums_stride + 4 * (size_t)i;
    const double kg = ldexp(1.0, leaf_bits - qexp[2 * k]), kh = ldexp(1.0, leaf_bits - qexp[2 * k + 1]);
    const double G = __ddiv_rn(b2_limbs_to_double(s[0], s[1]), kg), H = __ddiv_rn(b2_limbs_to_double(s[2], s[3]), kh);
    const float v = __fmul_rn(c_calc_weight(G, H, p), p.eta);
    leaf_vec[idx] = v;
    tree_vec[(size_t)leaves[i].nid * T + k] = v;
  }
}

// tree-start reset: root node, counters
__global__ void tree_init_kernel(B2TreeDev tree, B2LevelCtl* ctl0, B2NodeSeg* seg0, B2EvalNode* ev0, int32_t* n_leaves,
                                 int n_rows, B2HistWork* hist_work0) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    B2HistWork hw; hw.seg_begin = 0; hw.seg_count = n_rows; hw.hist_index = 0; hw.chunk_begin = 0; hist_work0[0] = hw;
    ctl0->leaf_base_next = 0;
    *tree.n_nodes = 1; *n_leaves = 0;
    tree.left[0] = -1; tree.right[0] = -1; tree.parent[0] = -1; tree.feature[0] = -1;
    ctl0->n_nodes = 1; ctl0->n_split = 0; ctl0->part_chunks = 0; ctl0->hist_n_work = 0; ctl0->hist_total_chunks = 0;
    ctl0->n_pairs = 0;
    B2NodeSeg s; s.nid = 0; s.buf = 0; s.begin = 0; s.count = n_rows; seg0[0] = s;
    B2EvalNode e; e.sum_g = 0; e.sum_h = 0; e.hist_index = 0; e.root_gain = 0.f; ev0[0] = e;
  }
}

}  // namespace b2

extern "C" {
int b2_launch_decide(const B2DecideArgs* a, const B2P2P* p2p, cudaStream_t s) {
  B2P2P pp;
  if (p2p) pp = *p2p; else memset(&pp, 0, sizeof(pp));
  b2::decide_kernel<<<1, b2::kCtlThreads, 0, s>>>(*a, p2p ? 1 : 0, pp);
  return (int)cudaGetLastError();
}
int b2_launch_leaf_plan(const B2LeafDev* leaves, const int32_t* n_leaves, B2SegWork* work, B2LevelCtl* leaf_ctl, cudaStream_t s) {
  b2::leaf_plan_kernel<<<1, b2::kCtlThreads, 0, s>>>(leaves, n_leaves, work, leaf_ctl);
  return (int)cudaGetLastError();
}
int b2_launch_leaf_values(const B2LeafDev* leaves, const int32_t* n_leaves, const long long* sums, const int32_t* qexp,
                          int leaf_bits, B2CtlParams p, float* leaf_value, B2TreeDev tree, int32_t* qexp_out, cudaStream_t s) {
  b2::leaf_values_kernel<<<8, 256, 0, s>>>(leaves, n_leaves, sums, qexp, leaf_bits, p, leaf_value, tree, qexp_out);
  return (int)cudaGetLastError();
}
int b2_launch_vector_leaf_values(const B2LeafDev* leaves, const int32_t* n_leaves, const long long* sums, size_t sums_stride,
                                 const int32_t* qexp, int T, int leaf_bits, B2CtlParams p, float* leaf_vec, float* tree_vec,
                                 int32_t* qexp_out, cudaStream_t s) {
  b2::vector_leaf_values_kernel<<<32, 256, 0, s>>>(leaves, n_leaves, sums, sums_stride, qexp, T, leaf_bits, p, leaf_vec, tree_vec,
                                                  qexp_out);
  return (int)cudaGetLastError();
}
int b2_launch_tree_init(B2TreeDev tree, B2LevelCtl* ctl0, B2NodeSeg* seg0, B2EvalNode* ev0, int32_t* n_leaves, int n_rows,
                        B2HistWork* hist_work0, cudaStream_t s) {
  b2::tree_init_kernel<<<1, 32, 0, s>>>(tree, ctl0, seg0, ev0, n_leaves, n_rows, hist_work0);
  return (int)cudaGetLastError();
}
}
