// decide.cuh -- the decision of one tree level: best candidate per node, expand or leaf, child ids, split work list.
//
// Run by ONE CTA of kThreads threads: decide_kernel (control_kernel.cu), or on one GPU the last CTA of the level's
// split scan (split_kernel.cu), which saves a single-CTA launch and its gap per level.
#pragma once
#include <stddef.h>

#include <cub/block/block_scan.cuh>

#include "common.cuh"
#include "p2p.cuh"

namespace b2 {

constexpr int kSplitChunkRows = 8192;  // split-node work items; must match partition_kernel.cu kSplitChunk

__device__ __forceinline__ double c_calc_gain(double G, double H, const B2CtlParams& p) {
  return b2_calc_gain(G, H, p.mcw, p.lambda, p.alpha, p.max_delta_step);
}

// exclusive scan of one int per item over n items handled as tiles of kThreads; returns total
template <int kThreads>
struct TileScan {
  typedef cub::BlockScan<int, kThreads> Scan;
  typename Scan::TempStorage* tmp;
  int carry;
  __device__ TileScan(typename Scan::TempStorage* t) : tmp(t), carry(0) {}
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

template <int kThreads>
struct DecideScratch {
  typename TileScan<kThreads>::Scan::TempStorage scan;
  int node_base, leaf_base;
};

// word w of a candidate: peer-written tables with ld.volatile, others at L2 (written by other CTAs of the same kernel
// when decide runs in the scan's last CTA)
__device__ __forceinline__ unsigned long long cand_word(const B2SplitCand* c, int w, bool vol) {
  const long long* src = reinterpret_cast<const long long*>(c) + w;
  return vol ? ld_volatile_u64(src) : (unsigned long long)__ldcg(src);
}

// cand_best[i] = the best candidate of node i over all ranks and scan CTAs, one warp per node.  The key
// (loss_chg bits, ~order) orders candidates as (loss_chg, then earlier enumeration): loss_chg > 0 for every
// candidate with a feature, and the enumeration order of a candidate is unique, so exactly one lane holds the maximum.
template <int kThreads>
__device__ void select_candidates(const B2DecideArgs& a, int n, bool vol) {
  constexpr int kWords = sizeof(B2SplitCand) / 8;
  static_assert(sizeof(B2SplitCand) % 8 == 0, "candidates are copied as 64-bit words");
  static_assert(offsetof(B2SplitCand, loss_chg) == 0 && offsetof(B2SplitCand, feature) == 4 && offsetof(B2SplitCand, order) == 32,
                "key words of a candidate");
  const int lane = threadIdx.x & 31, per_node = a.cand_ranks * a.cands_per_node;
  for (int i = threadIdx.x >> 5; i < n; i += kThreads / 32) {
    unsigned long long mine = 0ull;
    const B2SplitCand* mine_c = nullptr;
    for (int j = lane; j < per_node; j += 32) {
      const int w = j / a.cands_per_node, g = j - w * a.cands_per_node;
      const B2SplitCand* c = a.cands + (size_t)w * a.cand_rank_stride + (size_t)i * a.cands_per_node + g;
      const unsigned long long w0 = cand_word(c, 0, vol);
      if ((int32_t)(uint32_t)(w0 >> 32) < 0) continue;   // feature -1: no candidate
      const unsigned long long key = ((w0 & 0xffffffffull) << 32) | (0xffffffffull - (cand_word(c, 4, vol) & 0xffffffffull));
      if (key > mine) { mine = key; mine_c = c; }
    }
    unsigned long long kmax = mine;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, kmax, o);
      kmax = other > kmax ? other : kmax;
    }
    if (kmax == 0ull) {
      if (lane == 0) { B2SplitCand& e = a.cand_best[i]; e.feature = -1; e.loss_chg = 0.f; e.order = 0xffffffffu; e.is_cat = 0; }
    } else if (mine == kmax) {
      unsigned long long* dst = reinterpret_cast<unsigned long long*>(a.cand_best + i);
#pragma unroll
      for (int t = 0; t < kWords; ++t) dst[t] = cand_word(mine_c, t, vol);
    }
  }
}

// use_p2p: peer-memory exchange (replaces ncclAllGather) -- this rank scanned only the feature slots it owns, so
// its per-node candidates go into region `rank` of EVERY rank's table; `a.cands` is this rank's own table
template <int kThreads>
__device__ __forceinline__ void decide_block(DecideScratch<kThreads>& sm, const B2DecideArgs& a, bool use_p2p, const B2P2P& pp) {
  const B2TreeDev& tree = a.tree;
  const B2CtlParams& p = a.p;
  const int n = a.ctl_cur->n_nodes;
  // the partition of this level counts its left / right rows per split node with atomics: start them at zero here
  if (a.part_counters) for (int i = threadIdx.x; i < 2 * n; i += kThreads) a.part_counters[i] = 0;
  if (use_p2p && a.can_split) {
    constexpr int kWords = sizeof(B2SplitCand) / 8;
    const uint32_t epoch = p2p_next_epoch(pp, kSlotCand);
    const int total = n * a.cands_per_node * kWords;
    for (int w = 0; w < pp.world; ++w) {
      long long* dst = reinterpret_cast<long long*>(pp.cands[w] + (size_t)pp.rank * pp.cand_cap);
      for (int t = threadIdx.x; t < total; t += kThreads) st_volatile_u64(dst + t, reinterpret_cast<const long long*>(a.local_cands)[t]);
    }
    __syncthreads();
    p2p_signal(pp, kSlotCand, epoch);
    p2p_wait(pp, kSlotCand, epoch);
    p2p_finish_single(pp, kSlotCand, epoch);
  }
  if (a.can_split) select_candidates<kThreads>(a, n, use_p2p);
  const double inv_sg = ldexp(1.0, a.qexp[0] - a.qbits), inv_sh = ldexp(1.0, a.qexp[1] - a.qbits);
  if (threadIdx.x == 0) { sm.node_base = *tree.n_nodes; sm.leaf_base = *a.n_leaves; }
  __syncthreads();
  const int node_base = sm.node_base, leaf_base = sm.leaf_base;
  TileScan<kThreads> scan_split(&sm.scan), scan_leaf(&sm.scan), scan_chunks(&sm.scan);
  for (int base = 0; base < n; base += kThreads) {
    const int i = base + threadIdx.x;
    const bool in = i < n;
    B2SplitCand best; best.feature = -1; best.loss_chg = 0.f; best.order = 0xffffffffu; best.bin = 0; best.default_left = 0;
    best.left_g = 0; best.left_h = 0; best.is_cat = 0;
    B2EvalNode nd; nd.sum_g = 0; nd.sum_h = 0; nd.hist_index = 0; nd.root_gain = 0.f;
    B2NodeSeg sg; sg.nid = 0; sg.begin = 0; sg.count = 0; sg.buf = 0;
    bool expand = false;
    if (in) {
      nd = a.ev_cur[i]; sg = a.seg_cur[i];
      if (a.can_split) {
        best = a.cand_best[i];
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
      a.leaves[leaf_base + lrank] = lf;
    }
    if (expand) {
      const int l = node_base + 2 * rank, r = l + 1;
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
      sw.default_left = best.default_left; sw.has_missing = a.has_missing[best.feature]; sw.chunk_begin = chunk_begin;
      sw.is_cat = best.is_cat;
#pragma unroll
      for (int w8 = 0; w8 < 8; ++w8) sw.cat_bits[w8] = best.is_cat ? best.cat_bits[w8] : 0u;
      a.split_work[rank] = sw;
      a.pair_parent_hist[rank] = nd.hist_index;
      const double GL = __dmul_rn(__ll2double_rn(lg), inv_sg), HL = __dmul_rn(__ll2double_rn(lh), inv_sh);
      const double GR = __dmul_rn(__ll2double_rn(rg), inv_sg), HR = __dmul_rn(__ll2double_rn(rh), inv_sh);
      B2EvalNode el, er;
      el.sum_g = lg; el.sum_h = lh; el.hist_index = -1; el.root_gain = __double2float_rn(c_calc_gain(GL, HL, p));
      er.sum_g = rg; er.sum_h = rh; er.hist_index = -1; er.root_gain = __double2float_rn(c_calc_gain(GR, HR, p));
      a.ev_nxt[2 * rank] = el; a.ev_nxt[2 * rank + 1] = er;
      B2NodeSeg sl, sr;
      sl.nid = l; sl.buf = sg.buf ^ 1; sl.begin = sg.begin; sl.count = 0;
      sr.nid = r; sr.buf = sg.buf ^ 1; sr.begin = sg.begin; sr.count = sg.count;   // finalised after the partition
      a.seg_nxt[2 * rank] = sl; a.seg_nxt[2 * rank + 1] = sr;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int n_split = scan_split.carry;
    a.ctl_cur->n_split = n_split; a.ctl_cur->part_chunks = scan_chunks.carry;
    a.ctl_cur->leaf_base_next = leaf_base + scan_leaf.carry;   // leaf index of the first node of the next level (final_assign_kernel)
    a.ctl_nxt->n_nodes = 2 * n_split; a.ctl_nxt->n_split = 0; a.ctl_nxt->part_chunks = 0;
    a.ctl_nxt->hist_n_work = 0; a.ctl_nxt->hist_total_chunks = 0; a.ctl_nxt->n_pairs = 0;
    *tree.n_nodes = node_base + 2 * n_split;
    *a.n_leaves = leaf_base + scan_leaf.carry;
  }
}

}  // namespace b2
