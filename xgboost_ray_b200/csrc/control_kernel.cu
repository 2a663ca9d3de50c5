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

#include <cub/block/block_scan.cuh>

#include "common.cuh"
#include "p2p.cuh"

namespace b2 {

constexpr int kCtlThreads = 1024;
constexpr int kPartChunkRows = 2048;   // leaf-segment work items; must match partition_kernel.cu kPartChunk
constexpr int kSplitChunkRows = 8192;  // split-node work items; must match partition_kernel.cu kSplitChunk

__device__ __forceinline__ double c_calc_gain(double G, double H, const B2CtlParams& p) {
  return b2_calc_gain(G, H, p.mcw, p.lambda, p.alpha, p.max_delta_step);
}
__device__ __forceinline__ float c_calc_weight(double G, double H, const B2CtlParams& p) {
  return __double2float_rn(b2_calc_weight(G, H, p.mcw, p.lambda, p.alpha, p.max_delta_step));
}

// exclusive scan of one int per item over n items handled as tiles of kCtlThreads; returns total
struct TileScan {
  typedef cub::BlockScan<int, kCtlThreads> Scan;
  Scan::TempStorage* tmp;
  int carry;
  __device__ TileScan(Scan::TempStorage* t) : tmp(t), carry(0) {}
  // call with the value of item (tile_base + tid) (0 when out of range); returns exclusive prefix
  __device__ int step(int v) {
    int ex, total;
    Scan(*tmp).ExclusiveSum(v, ex, total);
    __syncthreads();
    int r = carry + ex;
    carry += total;
    return r;
  }
};

// ---- decide: one thread per node of the level
__global__ void __launch_bounds__(kCtlThreads)
decide_kernel(B2LevelCtl* __restrict__ ctl_cur, B2LevelCtl* __restrict__ ctl_nxt, const B2NodeSeg* __restrict__ seg_cur,
              B2NodeSeg* __restrict__ seg_nxt, const B2EvalNode* __restrict__ ev_cur, B2EvalNode* __restrict__ ev_nxt,
              const B2SplitCand* __restrict__ cands, int cands_per_node, int cand_ranks, int cand_rank_stride, int can_split,
              B2TreeDev tree,
              B2SplitWork* __restrict__ split_work, int32_t* __restrict__ pair_parent_hist, B2LeafDev* __restrict__ leaves,
              int32_t* __restrict__ n_leaves, const uint8_t* __restrict__ has_missing, const int32_t* __restrict__ qexp,
              int qbits, B2CtlParams p, int32_t* __restrict__ part_counters, const B2SplitCand* __restrict__ local_cands,
              int use_p2p, B2P2P pp) {
  __shared__ typename TileScan::Scan::TempStorage tmp;
  __shared__ int s_node_base, s_leaf_base;
  const int n = ctl_cur->n_nodes;
  // the partition of this level counts its left / right rows per split node with atomics: start them at zero here
  if (part_counters) for (int i = threadIdx.x; i < 2 * n; i += kCtlThreads) part_counters[i] = 0;
  if (use_p2p && can_split) {
    // peer-memory candidate exchange (replaces ncclAllGather): this rank scanned only the feature slots it owns, so
    // its per-node candidates go into region `rank` of EVERY rank's table; `cands` is this rank's own table
    constexpr int kWords = sizeof(B2SplitCand) / 8;
    static_assert(sizeof(B2SplitCand) % 8 == 0, "candidates are copied as 64-bit words");
    const uint32_t epoch = p2p_next_epoch(pp, kSlotCand);
    const int total = n * cands_per_node * kWords;
    for (int w = 0; w < pp.world; ++w) {
      long long* dst = reinterpret_cast<long long*>(pp.cands[w] + (size_t)pp.rank * pp.cand_cap);
      for (int t = threadIdx.x; t < total; t += kCtlThreads) st_volatile_u64(dst + t, reinterpret_cast<const long long*>(local_cands)[t]);
    }
    __syncthreads();
    p2p_signal(pp, kSlotCand, epoch);
    p2p_wait(pp, kSlotCand, epoch);
    p2p_finish_single(pp, kSlotCand, epoch);
  }
  const double inv_sg = ldexp(1.0, qexp[0] - qbits), inv_sh = ldexp(1.0, qexp[1] - qbits);
  if (threadIdx.x == 0) { s_node_base = *tree.n_nodes; s_leaf_base = *n_leaves; }
  __syncthreads();
  TileScan scan_split(&tmp), scan_leaf(&tmp), scan_chunks(&tmp);
  for (int base = 0; base < n; base += kCtlThreads) {
    const int i = base + threadIdx.x;
    const bool in = i < n;
    B2SplitCand best; best.feature = -1; best.loss_chg = 0.f; best.order = 0xffffffffu; best.bin = 0; best.default_left = 0;
    best.left_g = 0; best.left_h = 0; best.is_cat = 0;
    B2EvalNode nd; nd.sum_g = 0; nd.sum_h = 0; nd.hist_index = 0; nd.root_gain = 0.f;
    B2NodeSeg sg; sg.nid = 0; sg.begin = 0; sg.count = 0; sg.buf = 0;
    bool expand = false;
    if (in) {
      nd = ev_cur[i]; sg = seg_cur[i];
      if (can_split) {
        for (int w = 0; w < cand_ranks; ++w)
          for (int g = 0; g < cands_per_node; ++g) {
            B2SplitCand c;
            if (use_p2p) {   // written by a peer while this kernel was already running: never the read-only / L1 path
              constexpr int kW = sizeof(B2SplitCand) / 8;
              const long long* src = reinterpret_cast<const long long*>(cands + (size_t)w * cand_rank_stride + (size_t)i * cands_per_node + g);
#pragma unroll
              for (int t = 0; t < kW; ++t) reinterpret_cast<unsigned long long*>(&c)[t] = ld_volatile_u64(src + t);
            } else c = cands[(size_t)w * cand_rank_stride + (size_t)i * cands_per_node + g];
            if (c.feature < 0) continue;
            if (best.feature < 0 || c.loss_chg > best.loss_chg || (c.loss_chg == best.loss_chg && c.order < best.order)) best = c;
          }
        if (best.feature >= 0)
          expand = best.loss_chg > 1e-6f && best.left_h != 0 && (nd.sum_h - best.left_h) != 0 && !(best.loss_chg < p.gamma);
      }
    }
    const int rank = scan_split.step(expand ? 1 : 0);
    const int lrank = scan_leaf.step((in && !expand) ? 1 : 0);
    const int chunks = expand ? (sg.count + kSplitChunkRows - 1) / kSplitChunkRows : 0;
    const int chunk_begin = scan_chunks.step(chunks);
    if (in && !expand) {
      B2LeafDev lf; lf.nid = sg.nid; lf.buf = sg.buf; lf.begin = sg.begin; lf.count = sg.count;
      leaves[s_leaf_base + lrank] = lf;
    }
    if (expand) {
      const int l = s_node_base + 2 * rank, r = l + 1;
      const int nid = sg.nid;
      tree.left[nid] = l; tree.right[nid] = r; tree.feature[nid] = best.feature; tree.split_bin[nid] = best.bin;
      tree.default_left[nid] = best.default_left; tree.loss_chg[nid] = best.loss_chg;
      tree.split_type[nid] = best.is_cat;
      if (best.is_cat) {
#pragma unroll
        for (int w8 = 0; w8 < 8; ++w8) tree.cat_bits[(size_t)nid * 8 + w8] = best.cat_bits[w8];
      }
      tree.left[l] = -1; tree.right[l] = -1; tree.feature[l] = -1; tree.parent[l] = nid;
      tree.left[r] = -1; tree.right[r] = -1; tree.feature[r] = -1; tree.parent[r] = nid;
      const long long lg = best.left_g, lh = best.left_h, rg = nd.sum_g - lg, rh = nd.sum_h - lh;
      tree.sum_g[l] = lg; tree.sum_h[l] = lh; tree.sum_g[r] = rg; tree.sum_h[r] = rh;
      B2SplitWork sw;
      sw.seg_begin = sg.begin; sw.seg_count = sg.count; sw.feature = best.feature; sw.split_bin = best.bin;
      sw.default_left = best.default_left; sw.has_missing = has_missing[best.feature]; sw.chunk_begin = chunk_begin;
      sw.is_cat = best.is_cat;
#pragma unroll
      for (int w8 = 0; w8 < 8; ++w8) sw.cat_bits[w8] = best.is_cat ? best.cat_bits[w8] : 0u;
      split_work[rank] = sw;
      pair_parent_hist[rank] = nd.hist_index;
      const double GL = __dmul_rn(__ll2double_rn(lg), inv_sg), HL = __dmul_rn(__ll2double_rn(lh), inv_sh);
      const double GR = __dmul_rn(__ll2double_rn(rg), inv_sg), HR = __dmul_rn(__ll2double_rn(rh), inv_sh);
      B2EvalNode el, er;
      el.sum_g = lg; el.sum_h = lh; el.hist_index = -1; el.root_gain = __double2float_rn(c_calc_gain(GL, HL, p));
      er.sum_g = rg; er.sum_h = rh; er.hist_index = -1; er.root_gain = __double2float_rn(c_calc_gain(GR, HR, p));
      ev_nxt[2 * rank] = el; ev_nxt[2 * rank + 1] = er;
      B2NodeSeg sl, sr;
      sl.nid = l; sl.buf = sg.buf ^ 1; sl.begin = sg.begin; sl.count = 0;
      sr.nid = r; sr.buf = sg.buf ^ 1; sr.begin = sg.begin; sr.count = sg.count;   // finalised after the partition
      seg_nxt[2 * rank] = sl; seg_nxt[2 * rank + 1] = sr;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int n_split = scan_split.carry;
    ctl_cur->n_split = n_split; ctl_cur->part_chunks = scan_chunks.carry;
    ctl_cur->leaf_base_next = s_leaf_base + scan_leaf.carry;   // leaf index of the first node of the next level (final_assign_kernel)
    ctl_nxt->n_nodes = 2 * n_split; ctl_nxt->n_split = 0; ctl_nxt->part_chunks = 0;
    ctl_nxt->hist_n_work = 0; ctl_nxt->hist_total_chunks = 0; ctl_nxt->n_pairs = 0;
    *tree.n_nodes = s_node_base + 2 * n_split;
    *n_leaves = s_leaf_base + scan_leaf.carry;
  }
}

// ---- leaves: chunked work list over the leaf segments
__global__ void __launch_bounds__(kCtlThreads)
leaf_plan_kernel(const B2LeafDev* __restrict__ leaves, const int32_t* __restrict__ n_leaves, B2SegWork* __restrict__ work,
                 B2LevelCtl* __restrict__ leaf_ctl) {
  __shared__ typename TileScan::Scan::TempStorage tmp;
  const int n = *n_leaves;
  TileScan scan(&tmp);
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

// leaf weight from the 40-bit fixed-point sums (A.7 leaf refinement), value = weight * eta (fp32); also keeps the
// tree's quantisation exponents in its read-back block (qexp_out)
__global__ void leaf_values_kernel(const B2LeafDev* __restrict__ leaves, const int32_t* __restrict__ n_leaves,
                                   const long long* __restrict__ sums, const int32_t* __restrict__ qexp, int leaf_bits,
                                   B2CtlParams p, float* __restrict__ leaf_value, B2TreeDev tree, int32_t* __restrict__ qexp_out) {
  const int n = *n_leaves;
  if (blockIdx.x == 0 && threadIdx.x < 2) qexp_out[threadIdx.x] = qexp[threadIdx.x];
  const double kg = ldexp(1.0, leaf_bits - qexp[0]), kh = ldexp(1.0, leaf_bits - qexp[1]);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double G = __ddiv_rn(__ll2double_rn(sums[2 * i]), kg), H = __ddiv_rn(__ll2double_rn(sums[2 * i + 1]), kh);
    const float w = c_calc_weight(G, H, p);
    const float v = __fmul_rn(w, p.eta);
    leaf_value[i] = v;
    tree.leaf_weight[leaves[i].nid] = w;
    tree.leaf_value[leaves[i].nid] = v;
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
int b2_launch_decide(B2LevelCtl* ctl_cur, B2LevelCtl* ctl_nxt, const B2NodeSeg* seg_cur, B2NodeSeg* seg_nxt,
                     const B2EvalNode* ev_cur, B2EvalNode* ev_nxt, const B2SplitCand* cands, int cands_per_node, int cand_ranks,
                     int cand_rank_stride, int can_split, B2TreeDev tree, B2SplitWork* split_work, int32_t* pair_parent_hist, B2LeafDev* leaves, int32_t* n_leaves,
                     const uint8_t* has_missing, const int32_t* qexp, int qbits, B2CtlParams p, int32_t* part_counters,
                     const B2SplitCand* local_cands, const void* p2p, cudaStream_t s) {
  B2P2P pp;
  if (p2p) pp = *reinterpret_cast<const B2P2P*>(p2p); else memset(&pp, 0, sizeof(pp));
  b2::decide_kernel<<<1, b2::kCtlThreads, 0, s>>>(ctl_cur, ctl_nxt, seg_cur, seg_nxt, ev_cur, ev_nxt, cands, cands_per_node,
                                                 cand_ranks, cand_rank_stride, can_split, tree, split_work, pair_parent_hist, leaves, n_leaves, has_missing, qexp, qbits, p,
                                                 part_counters, local_cands, p2p ? 1 : 0, pp);
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
int b2_launch_tree_init(B2TreeDev tree, B2LevelCtl* ctl0, B2NodeSeg* seg0, B2EvalNode* ev0, int32_t* n_leaves, int n_rows,
                        B2HistWork* hist_work0, cudaStream_t s) {
  b2::tree_init_kernel<<<1, 32, 0, s>>>(tree, ctl0, seg0, ev0, n_leaves, n_rows, hist_work0);
  return (int)cudaGetLastError();
}
}
