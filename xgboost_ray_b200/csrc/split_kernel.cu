// split_kernel.cu -- split-gain scan over the (allreduced) level histograms.
//
// Replaces XGBoost's EvaluateSplits stage reached through xgb.train()
// (xgboost_ray/main.py:745-752; SURVEY.md 8a row a12, Appendix A.6).  One CTA per
// (node, 4 feature slots); a thread scans 4 bins of one slot (eval_node_cta).
// Prefix sums are exact int64, gains are IEEE fp64 with explicit round-to-nearest ops (no fma
// contraction), so every rank and the CPU oracle compute identical candidates.
#include <string.h>

#include <cub/block/block_scan.cuh>

#include "common.cuh"
#include "decide.cuh"
#include "sampling.cuh"

namespace b2 {

__device__ __forceinline__ double calc_gain(double G, double H, const B2TrainParamDev& p) {
  return b2_calc_gain(G, H, p.min_child_weight, p.lambda, p.alpha, p.max_delta_step);
}

struct Best {
  unsigned long long key;  // (loss_chg bits << 32) | ~order ; 0 = none
  int32_t bin, default_left;
  long long lg, lh;
};

__device__ __forceinline__ void consider(Best& b, float chg, uint32_t order, int bin, int dl, long long lg, long long lh) {
  if (!(chg > 0.0f) || isinf(chg)) return;
  unsigned long long key = ((unsigned long long)__float_as_uint(chg) << 32) | (unsigned long long)(0xffffffffu - order);
  if (key > b.key) { b.key = key; b.bin = bin; b.default_left = dl; b.lg = lg; b.lh = lh; }
}

// A CTA covers 4 consecutive owned slots ("virtual slots") x 256 bins of one node: 512 threads, thread = 2 consecutive
// bins of one slot (lane & 3 = slot).  At one bin, the 4 slots are 32 contiguous bytes of a plane, so every load
// instruction of a warp reads 8 whole 32-byte sectors.  The int64 prefix over a slot's bins is the thread's own bins,
// a shuffle scan over the 8 lanes of the slot in the warp and a carry over the 16 warps.  The CTA count per node (32 on
// 128 slots) spreads the shallow levels over the whole GPU.
constexpr int kEvalSlots = 4;                                           // virtual slots per CTA
constexpr int kEvalBinsPerThread = 2;
constexpr int kEvalThreads = kEvalSlots * B2_BINS / kEvalBinsPerThread;  // 512
constexpr int kEvalWarps = kEvalThreads / 32;                            // a warp covers 16 consecutive bins
// Above this many nodes a level is scanned by eval_splits_wide_kernel: the CTAs of this layout are short, and at 32+
// nodes (1024+ CTAs) their fixed chain of dependent loads costs more than the wide layout's longer per-thread loop.
constexpr int kNarrowMaxNodes = 16;

__host__ __device__ __forceinline__ int eval_ctas_per_node(int n_groups, int sp, int slots) { return (n_groups * sp + slots - 1) / slots; }

// the CTA's candidate: written by the thread that holds the block maximum (thread 0 writes "none"), which fences it for
// a decide in the last CTA of the grid
__device__ __forceinline__ void write_candidate(B2SplitCand* out, unsigned long long kmax, const Best& best, int f) {
  if (kmax == 0) {
    if (threadIdx.x == 0) {
      out->loss_chg = 0.0f; out->feature = -1; out->bin = 0; out->default_left = 0; out->left_g = 0; out->left_h = 0;
      out->order = 0xffffffffu; out->is_cat = 0;
      __threadfence();
    }
  } else if (best.key == kmax) {
    out->loss_chg = __uint_as_float((uint32_t)(kmax >> 32));
    out->feature = f; out->bin = best.bin; out->default_left = best.default_left;
    out->left_g = best.lg; out->left_h = best.lh; out->order = 0xffffffffu - (uint32_t)(kmax & 0xffffffffu); out->is_cat = 0;
    __threadfence();
  }
}

// With fold_decide every CTA of a scan takes a ticket on *done after its candidate is out (CTAs past ctl->n_nodes
// included), and the CTA that completes the grid resets the counter (for the next level and every replay of a
// captured tree) and decides the level (decide.cuh).
template <int kThreads>
__device__ __forceinline__ void decide_in_last_cta(const B2DecideArgs& dec, uint32_t* done) {
  __shared__ DecideScratch<kThreads> s_dec;
  __shared__ bool s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned prev = atomicAdd(done, 1u);
    s_last = prev == gridDim.x - 1;
    if (s_last) { __threadfence(); *done = 0u; }
  }
  __syncthreads();
  if (!s_last) return;
  B2P2P none;
  memset(&none, 0, sizeof(none));
  decide_block<kThreads>(s_dec, dec, false, none);
}

// Sibling subtraction in the scan (B2SiblingSub, parent_level != nullptr): a node whose histogram slot is a sibling
// slot (>= sib_base) was never built or subtracted.  Its bins are formed in registers as parent - built, exact int64,
// with (parent slot, built slot) = triples[3 j], triples[3 j + 1] for j = slot - sib_base.  With sib_out the CTA also
// stores the whole sibling slice (every bin of every slot it covers, sampled or not), because the next level reads it
// as a parent.  level_hist is only read at built slots in this mode, sib_out only at sibling slots, so the two never
// alias.
__device__ __forceinline__ void eval_node_cta(const long long* __restrict__ level_hist, int n_groups, const B2EvalNode& nd, int node,
                                              int cta_in_node, const int32_t* __restrict__ group_first,
                                              const int32_t* __restrict__ group_size, const int32_t* __restrict__ nbins,
                                              const uint8_t* __restrict__ has_missing, const uint8_t* __restrict__ is_cat,
                                              const int32_t* __restrict__ qexp, int qbits, B2TrainParamDev p, B2SplitCand* cands,
                                              int cand_stride, int log2_shards, int shard_rank, const B2ColSample& cs,
                                              const B2NodeSeg* __restrict__ seg, const B2SiblingSub& sub) {
  __shared__ long long s_wg[kEvalWarps][kEvalSlots], s_wh[kEvalWarps][kEvalSlots];   // warp totals, then carries
  __shared__ long long s_tg[kEvalSlots], s_th[kEvalSlots];                           // sums over a slot's real bins
  __shared__ unsigned long long s_key[kEvalWarps];
  __shared__ uint8_t s_allowed[kEvalSlots];
  const int sp = B2_GROUP_SLOTS >> log2_shards;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int s = threadIdx.x & (kEvalSlots - 1), b0 = (threadIdx.x / kEvalSlots) * kEvalBinsPerThread;
  // inverse scales: 2^(e - qbits)
  p.inv_scale_g = ldexp(1.0, qexp[0] - qbits);
  p.inv_scale_h = ldexp(1.0, qexp[1] - qbits);
  const int v = cta_in_node * kEvalSlots + s;              // virtual slot: this rank owns slot s of a group if s % shards == rank
  const bool v_ok = v < n_groups * sp;
  const int group = v_ok ? v / sp : 0, sl = v_ok ? v % sp : 0;
  const int slot = (sl << log2_shards) + shard_rank;       // real slot inside the group
  const size_t slice_elems = (size_t)n_groups * 2 * B2_BINS * sp;
  const size_t in_slice = (size_t)(group * 2) * B2_BINS * sp + sl;
  const bool fused = sub.parent_level != nullptr && nd.hist_index >= sub.sib_base;   // uniform over the CTA
  const int pair = fused ? nd.hist_index - sub.sib_base : 0;
  const long long* hg = level_hist + (size_t)(fused ? sub.triples[3 * pair + 1] : nd.hist_index) * slice_elems + in_slice;
  const long long* hh = hg + (size_t)B2_BINS * sp;
  const long long* pgp = fused ? sub.parent_level + (size_t)sub.triples[3 * pair] * slice_elems + in_slice : nullptr;
  const long long* php = fused ? pgp + (size_t)B2_BINS * sp : nullptr;
  long long* sgp = (fused && sub.sib_out) ? sub.sib_out + (size_t)nd.hist_index * slice_elems + in_slice : nullptr;
  long long* shp = sgp ? sgp + (size_t)B2_BINS * sp : nullptr;
  const int f = group_first[group] + slot;
  bool active = v_ok && slot < group_size[group] && !(is_cat && is_cat[f]);
  if (active && cs.level_mask) active = cs.level_mask[f] != 0;          // colsample_bytree / bylevel
  if (cs.bynode < 1.0) {                                                // colsample_bynode: this node's own subset
    if (threadIdx.x < kEvalSlots)
      s_allowed[s] = active && b2_col_selected(cs.seed, cs.tree, B2_SCOPE_NODE(seg[node].nid), f, cs.level_mask, cs.fwq,
                                               cs.n_features, b2_sample_count(cs.bynode, cs.n_level));
    __syncthreads();
    active = active && s_allowed[s];
  }
  const int nf = active ? nbins[f] : 0;
  const bool fmiss = active ? (has_missing[f] != 0) : false;

  // the thread's bins; bins at or past nf (and inactive slots) count as zero
  long long g[kEvalBinsPerThread], h[kEvalBinsPerThread];
#pragma unroll
  for (int i = 0; i < kEvalBinsPerThread; ++i) { g[i] = 0; h[i] = 0; }
  if (fused) {
    if (v_ok && (sgp || active)) {
#pragma unroll
      for (int i = 0; i < kEvalBinsPerThread; ++i) {
        const int b = b0 + i;
        g[i] = pgp[b * sp] - hg[b * sp]; h[i] = php[b * sp] - hh[b * sp];
      }
      if (sgp) {
#pragma unroll
        for (int i = 0; i < kEvalBinsPerThread; ++i) { sgp[(b0 + i) * sp] = g[i]; shp[(b0 + i) * sp] = h[i]; }
      }
#pragma unroll
      for (int i = 0; i < kEvalBinsPerThread; ++i)
        if (b0 + i >= nf) { g[i] = 0; h[i] = 0; }
    }
  } else if (active) {
#pragma unroll
    for (int i = 0; i < kEvalBinsPerThread; ++i) {
      const int b = b0 + i;
      if (b < nf) { g[i] = hg[b * sp]; h[i] = hh[b * sp]; }
    }
  }
  // exclusive prefix of the slot's bins before b0: the thread's total, scanned over the 8 lanes of the slot in the warp
  // (lanes s, s + 4, ..., s + 28), plus the totals of the warps before
  long long tg = 0, th = 0;
#pragma unroll
  for (int i = 0; i < kEvalBinsPerThread; ++i) { tg += g[i]; th += h[i]; }
  long long ig = tg, ih = th;
#pragma unroll
  for (int o = kEvalSlots; o < 32; o <<= 1) {
    const long long ug = __shfl_up_sync(0xffffffffu, ig, o), uh = __shfl_up_sync(0xffffffffu, ih, o);
    if (lane >= o) { ig += ug; ih += uh; }
  }
  if (lane >= 32 - kEvalSlots) { s_wg[warp][s] = ig; s_wh[warp][s] = ih; }
  __syncthreads();
  if (threadIdx.x < kEvalSlots) {
    long long cg = 0, ch = 0;
#pragma unroll
    for (int w = 0; w < kEvalWarps; ++w) {
      const long long a = s_wg[w][threadIdx.x], c = s_wh[w][threadIdx.x];
      s_wg[w][threadIdx.x] = cg; s_wh[w][threadIdx.x] = ch;
      cg += a; ch += c;
    }
    s_tg[threadIdx.x] = cg; s_th[threadIdx.x] = ch;
  }
  __syncthreads();
  long long pg = s_wg[warp][s] + ig - tg, ph = s_wh[warp][s] + ih - th;
  const long long real_g = s_tg[s], real_h = s_th[s];
  const long long tot_g = nd.sum_g, tot_h = nd.sum_h;
  const double G = __dmul_rn(__ll2double_rn(tot_g), p.inv_scale_g), H = __dmul_rn(__ll2double_rn(tot_h), p.inv_scale_h);
  const double root_gain = (double)nd.root_gain;
  const bool node_has_missing = fmiss && (real_g != tot_g || real_h != tot_h);
  Best best; best.key = 0; best.bin = 0; best.default_left = 0; best.lg = 0; best.lh = 0;
#pragma unroll
  for (int i = 0; i < kEvalBinsPerThread; ++i) {
    const int b = b0 + i;
    if (b >= nf) break;
    const long long eg_excl = pg, eh_excl = ph;
    pg += g[i]; ph += h[i];
    {  // forward: left = prefix inclusive, missing -> right
      const double lh_d = __dmul_rn(__ll2double_rn(ph), p.inv_scale_h);
      if (lh_d >= p.min_child_weight) {
        const double rh_d = __dadd_rn(H, -lh_d);
        if (rh_d >= p.min_child_weight) {
          const double lg_d = __dmul_rn(__ll2double_rn(pg), p.inv_scale_g);
          const double rg_d = __dadd_rn(G, -lg_d);
          const double gain = __dadd_rn(__dadd_rn(calc_gain(lg_d, lh_d, p), calc_gain(rg_d, rh_d, p)), -root_gain);
          consider(best, __double2float_rn(gain), (uint32_t)f * 1024u + (uint32_t)b, b, 0, pg, ph);
        }
      }
    }
    if (node_has_missing) {  // backward at bin b: right' = sum of real bins >= b, missing -> left
      const long long rg_i = real_g - eg_excl, rh_i = real_h - eh_excl;
      const double rh_d = __dmul_rn(__ll2double_rn(rh_i), p.inv_scale_h);
      if (rh_d >= p.min_child_weight) {
        const double lh_d = __dadd_rn(H, -rh_d);
        if (lh_d >= p.min_child_weight) {
          const double rg_d = __dmul_rn(__ll2double_rn(rg_i), p.inv_scale_g);
          const double lg_d = __dadd_rn(G, -rg_d);
          const double gain = __dadd_rn(__dadd_rn(calc_gain(lg_d, lh_d, p), calc_gain(rg_d, rh_d, p)), -root_gain);
          consider(best, __double2float_rn(gain), (uint32_t)f * 1024u + 512u + (uint32_t)(255 - b), b - 1, 1,
                   tot_g - rg_i, tot_h - rh_i);
        }
      }
    }
  }
  // block argmax on key
  unsigned long long k = best.key;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    unsigned long long other = __shfl_xor_sync(0xffffffffu, k, o);
    k = other > k ? other : k;
  }
  if (lane == 0) s_key[warp] = k;
  __syncthreads();
  unsigned long long kmax = 0;
#pragma unroll
  for (int i = 0; i < kEvalWarps; ++i) kmax = s_key[i] > kmax ? s_key[i] : kmax;
  write_candidate(cands + (size_t)node * cand_stride + cta_in_node, kmax, best, f);
}

// Grid = upper bound of the level's nodes x eval_ctas_per_node; CTAs past ctl->n_nodes only arrive.
__global__ void __launch_bounds__(kEvalThreads, 2)
eval_splits_kernel(const long long* __restrict__ level_hist, int n_groups, const B2EvalNode* __restrict__ nodes,
                   const int32_t* __restrict__ group_first, const int32_t* __restrict__ group_size,
                   const int32_t* __restrict__ nbins, const uint8_t* __restrict__ has_missing,
                   const uint8_t* __restrict__ is_cat /* nullable: categorical features are scanned by eval_cat_splits_kernel */,
                   const int32_t* __restrict__ qexp, int qbits, B2TrainParamDev p, B2SplitCand* cands,
                   int cand_stride, const B2LevelCtl* ctl, int log2_shards, int shard_rank, B2ColSample cs,
                   const B2NodeSeg* __restrict__ seg, B2SiblingSub sub, int fold_decide, B2DecideArgs dec, uint32_t* done) {
  const int cpn = eval_ctas_per_node(n_groups, B2_GROUP_SLOTS >> log2_shards, kEvalSlots);
  const int node = blockIdx.x / cpn;
  if (!ctl || node < ctl->n_nodes)   // uniform over the CTA
    eval_node_cta(level_hist, n_groups, nodes[node], node, blockIdx.x % cpn, group_first, group_size, nbins, has_missing, is_cat,
                  qexp, qbits, p, cands, cand_stride, log2_shards, shard_rank, cs, seg, sub);
  if (fold_decide) decide_in_last_cta<kEvalThreads>(dec, done);
}

// ---- deep levels (more than kNarrowMaxNodes nodes): one CTA per (node, 32 owned slots), 1024 threads = 32 slots x
// 32 bin chunks of 8 bins; the bin scan re-reads the histogram instead of keeping the 8 bins in registers.  Its level
// is decided by decide_kernel: measured on H100, a decide in the last CTA made these levels slower than the launch it
// saves.
constexpr int kWideChunks = 32;                 // bin chunks per feature
constexpr int kWideBinsPerChunk = 256 / kWideChunks;

// Sibling subtraction in the scan (B2SiblingSub, parent_level != nullptr): a node whose histogram slot is a sibling
// slot (>= sib_base) was never built or subtracted.  Its bins are formed in registers as parent - built, exact int64,
// with (parent slot, built slot) = triples[3 j], triples[3 j + 1] for j = slot - sib_base.  With sib_out the CTA also
// stores the whole sibling slice (every bin of every slot it covers, sampled or not), because the next level reads it
// as a parent; the bin scan then re-reads the stored values.  Without sib_out (the last histogram level) nothing is
// stored and the scan subtracts again.  level_hist is only read at built slots in this mode, sib_out only at sibling
// slots, so the two never alias.
__global__ void __launch_bounds__(32 * kWideChunks)
eval_splits_wide_kernel(const long long* __restrict__ level_hist, int n_groups, const B2EvalNode* __restrict__ nodes,
                   const int32_t* __restrict__ group_first, const int32_t* __restrict__ group_size,
                   const int32_t* __restrict__ nbins, const uint8_t* __restrict__ has_missing,
                   const uint8_t* __restrict__ is_cat /* nullable: categorical features are scanned by eval_cat_splits_kernel */,
                   const int32_t* __restrict__ qexp, int qbits, B2TrainParamDev p, B2SplitCand* __restrict__ cands,
                   int cand_stride, const B2LevelCtl* __restrict__ ctl, int log2_shards, int shard_rank, B2ColSample cs,
                   const B2NodeSeg* __restrict__ seg, B2SiblingSub sub) {
  // This rank owns sp = 32 >> log2_shards slots of every group (slot s is owned by s % shards): the
  // G*sp owned "virtual slots" of a node are covered by cpn = ceil(G*sp/32) CTAs.
  const int sp = B2_GROUP_SLOTS >> log2_shards;
  const int cpn = (n_groups * sp + 31) >> 5;
  const int node = blockIdx.x / cpn, cta_in_node = blockIdx.x % cpn;
  if (ctl && node >= ctl->n_nodes) return;
  const int s = threadIdx.x & 31, q = threadIdx.x >> 5;
  __shared__ long long cs_g[kWideChunks][32], cs_h[kWideChunks][32];
  __shared__ unsigned long long wkey[kWideChunks];
  const B2EvalNode nd = nodes[node];
  // inverse scales: 2^(e - qbits)
  p.inv_scale_g = ldexp(1.0, qexp[0] - qbits);
  p.inv_scale_h = ldexp(1.0, qexp[1] - qbits);
  const int v = cta_in_node * 32 + s;                      // virtual slot
  const bool v_ok = v < n_groups * sp;
  const int group = v_ok ? v / sp : 0, sl = v_ok ? v % sp : 0;
  const int slot = (sl << log2_shards) + shard_rank;       // real slot inside the group
  const size_t slice_elems = (size_t)n_groups * 2 * B2_BINS * sp;
  const size_t in_slice = (size_t)(group * 2) * B2_BINS * sp + sl;
  const bool fused = sub.parent_level != nullptr && nd.hist_index >= sub.sib_base;   // uniform over the CTA
  const int pair = fused ? nd.hist_index - sub.sib_base : 0;
  const long long* hg = level_hist + (size_t)(fused ? sub.triples[3 * pair + 1] : nd.hist_index) * slice_elems + in_slice;
  const long long* hh = hg + (size_t)B2_BINS * sp;
  const long long* pgp = fused ? sub.parent_level + (size_t)sub.triples[3 * pair] * slice_elems + in_slice : nullptr;
  const long long* php = fused ? pgp + (size_t)B2_BINS * sp : nullptr;
  long long* sgp = (fused && sub.sib_out) ? sub.sib_out + (size_t)nd.hist_index * slice_elems + in_slice : nullptr;
  long long* shp = sgp ? sgp + (size_t)B2_BINS * sp : nullptr;
  const int f = group_first[group] + slot;
  bool active = v_ok && slot < group_size[group] && !(is_cat && is_cat[f]);
  if (active && cs.level_mask) active = cs.level_mask[f] != 0;          // colsample_bytree / bylevel
  if (cs.bynode < 1.0) {                                                // colsample_bynode: this node's own subset
    __shared__ uint8_t s_allowed[32];
    if (q == 0)
      s_allowed[s] = active && b2_col_selected(cs.seed, cs.tree, B2_SCOPE_NODE(seg[node].nid), f, cs.level_mask, cs.fwq,
                                               cs.n_features, b2_sample_count(cs.bynode, cs.n_level));
    __syncthreads();
    active = active && s_allowed[s];
  }
  const int nf = active ? nbins[f] : 0;
  const bool fmiss = active ? (has_missing[f] != 0) : false;

  long long sg = 0, sh = 0;
  if (fused) {
    if (v_ok && (sgp || active)) {
#pragma unroll
      for (int i = 0; i < kWideBinsPerChunk; ++i) {
        const int b = q * kWideBinsPerChunk + i;
        const long long g = pgp[b * sp] - hg[b * sp], h = php[b * sp] - hh[b * sp];
        if (sgp) { sgp[b * sp] = g; shp[b * sp] = h; }
        if (active && b < nf) { sg += g; sh += h; }
      }
    }
  } else if (active) {
#pragma unroll
    for (int i = 0; i < kWideBinsPerChunk; ++i) {
      int b = q * kWideBinsPerChunk + i;
      if (b < nf) { sg += hg[b * sp]; sh += hh[b * sp]; }
    }
  }
  cs_g[q][s] = sg; cs_h[q][s] = sh;
  __syncthreads();
  long long pg = 0, ph = 0, real_g = 0, real_h = 0;
#pragma unroll 8
  for (int k = 0; k < kWideChunks; ++k) {
    long long a = cs_g[k][s], b = cs_h[k][s];
    if (k < q) { pg += a; ph += b; }
    real_g += a; real_h += b;
  }
  const long long tot_g = nd.sum_g, tot_h = nd.sum_h;
  const double G = __dmul_rn(__ll2double_rn(tot_g), p.inv_scale_g), H = __dmul_rn(__ll2double_rn(tot_h), p.inv_scale_h);
  const double root_gain = (double)nd.root_gain;
  const bool node_has_missing = fmiss && (real_g != tot_g || real_h != tot_h);
  Best best; best.key = 0; best.bin = 0; best.default_left = 0; best.lg = 0; best.lh = 0;
  if (active) {
#pragma unroll 2
    for (int i = 0; i < kWideBinsPerChunk; ++i) {
      const int b = q * kWideBinsPerChunk + i;
      if (b >= nf) break;
      const long long eg_excl = pg, eh_excl = ph;
      if (!fused) { pg += hg[b * sp]; ph += hh[b * sp]; }
      else if (sgp) { pg += sgp[b * sp]; ph += shp[b * sp]; }   // stored by this thread in the first pass
      else { pg += pgp[b * sp] - hg[b * sp]; ph += php[b * sp] - hh[b * sp]; }
      {  // forward: left = prefix inclusive, missing -> right
        const double lh_d = __dmul_rn(__ll2double_rn(ph), p.inv_scale_h);
        if (lh_d >= p.min_child_weight) {
          const double rh_d = __dadd_rn(H, -lh_d);
          if (rh_d >= p.min_child_weight) {
            const double lg_d = __dmul_rn(__ll2double_rn(pg), p.inv_scale_g);
            const double rg_d = __dadd_rn(G, -lg_d);
            const double gain = __dadd_rn(__dadd_rn(calc_gain(lg_d, lh_d, p), calc_gain(rg_d, rh_d, p)), -root_gain);
            consider(best, __double2float_rn(gain), (uint32_t)f * 1024u + (uint32_t)b, b, 0, pg, ph);
          }
        }
      }
      if (node_has_missing) {  // backward at bin b: right' = sum of real bins >= b, missing -> left
        const long long rg_i = real_g - eg_excl, rh_i = real_h - eh_excl;
        const double rh_d = __dmul_rn(__ll2double_rn(rh_i), p.inv_scale_h);
        if (rh_d >= p.min_child_weight) {
          const double lh_d = __dadd_rn(H, -rh_d);
          if (lh_d >= p.min_child_weight) {
            const double rg_d = __dmul_rn(__ll2double_rn(rg_i), p.inv_scale_g);
            const double lg_d = __dadd_rn(G, -rg_d);
            const double gain = __dadd_rn(__dadd_rn(calc_gain(lg_d, lh_d, p), calc_gain(rg_d, rh_d, p)), -root_gain);
            consider(best, __double2float_rn(gain), (uint32_t)f * 1024u + 512u + (uint32_t)(255 - b), b - 1, 1,
                     tot_g - rg_i, tot_h - rh_i);
          }
        }
      }
    }
  }
  // block argmax on key
  unsigned long long k = best.key;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    unsigned long long other = __shfl_xor_sync(0xffffffffu, k, o);
    k = other > k ? other : k;
  }
  if (s == 0) wkey[q] = k;
  __syncthreads();
  unsigned long long kmax = 0;
#pragma unroll 8
  for (int i = 0; i < kWideChunks; ++i) kmax = wkey[i] > kmax ? wkey[i] : kmax;
  B2SplitCand* out = cands + (size_t)node * cand_stride + cta_in_node;
  if (kmax == 0) {
    if (threadIdx.x == 0) {
      out->loss_chg = 0.0f; out->feature = -1; out->bin = 0; out->default_left = 0; out->left_g = 0; out->left_h = 0;
      out->order = 0xffffffffu; out->is_cat = 0;
    }
  } else if (best.key == kmax) {
    out->loss_chg = __uint_as_float((uint32_t)(kmax >> 32));
    out->feature = f; out->bin = best.bin; out->default_left = best.default_left;
    out->left_g = best.lg; out->left_h = best.lh; out->order = 0xffffffffu - (uint32_t)(kmax & 0xffffffffu); out->is_cat = 0;
  }
}

// ---------------------------------------------------------------- categorical features
// XGBoost's EnumerateOneHot / EnumeratePart (src/tree/hist/evaluate_splits.h; SURVEY.md A.8): bin = category code.
// One CTA of 256 threads (thread = category) scans one categorical feature at a time; the kCatCtas CTAs of a node
// share its categorical features round-robin and each writes one candidate (with the set of categories that go
// right) behind the node's numeric candidates.  Same exact-integer sums and IEEE fp64 gain as the numeric scan.
constexpr int kCatCtas = 4;

__device__ __forceinline__ float calc_weight_f(double G, double H, const B2TrainParamDev& p) {
  return __double2float_rn(b2_calc_weight(G, H, p.min_child_weight, p.lambda, p.alpha, p.max_delta_step));
}

__global__ void __launch_bounds__(256)
eval_cat_splits_kernel(const long long* __restrict__ level_hist, int n_groups, const B2EvalNode* __restrict__ nodes,
                       const int32_t* __restrict__ cat_feats, int n_cat, const int32_t* __restrict__ feat_byte,
                       const int32_t* __restrict__ nbins, const int32_t* __restrict__ qexp, int qbits, B2TrainParamDev p,
                       B2SplitCand* __restrict__ cands, int cand_stride, int cand_offset, const B2LevelCtl* __restrict__ ctl,
                       int log2_shards, int shard_rank, B2ColSample cs, const B2NodeSeg* __restrict__ seg) {
  const int node = blockIdx.x / kCatCtas, j = blockIdx.x % kCatCtas;
  if (ctl && node >= ctl->n_nodes) return;
  typedef cub::BlockScan<long long, 256> Scan;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ float s_w[256];
  __shared__ long long s_g[256], s_h[256];
  __shared__ long long s_red[2][8];
  __shared__ unsigned long long s_wkey[8];
  __shared__ unsigned long long s_best_key;
  __shared__ uint32_t s_bits[8];
  __shared__ int s_mode, s_part;             // winner of the current feature: 0 one-hot (category s_part), 1 partition (first s_part sorted)
  __shared__ int s_skip;
  __shared__ B2SplitCand s_best;
  const int b = threadIdx.x, lane = b & 31, warp = b >> 5;
  const int sp = B2_GROUP_SLOTS >> log2_shards, shards = 1 << log2_shards;
  const size_t slice_elems = (size_t)n_groups * 2 * B2_BINS * sp;
  const B2EvalNode nd = nodes[node];
  p.inv_scale_g = ldexp(1.0, qexp[0] - qbits);
  p.inv_scale_h = ldexp(1.0, qexp[1] - qbits);
  const long long tot_g = nd.sum_g, tot_h = nd.sum_h;
  const double G = __dmul_rn(__ll2double_rn(tot_g), p.inv_scale_g), H = __dmul_rn(__ll2double_rn(tot_h), p.inv_scale_h);
  const double root_gain = (double)nd.root_gain;
  if (b == 0) s_best_key = 0;
  __syncthreads();
  for (int ci = j; ci < n_cat; ci += kCatCtas) {
    const int f = cat_feats[ci];
    const int fb = feat_byte[f], group = fb >> 5, slot = fb & 31;
    if ((slot & (shards - 1)) != shard_rank) continue;          // another rank owns this slot (uniform)
    if (cs.level_mask || cs.bynode < 1.0) {                     // column sampling (uniform decision per feature)
      if (b == 0) {
        bool ok = !cs.level_mask || cs.level_mask[f] != 0;
        if (ok && cs.bynode < 1.0)
          ok = b2_col_selected(cs.seed, cs.tree, B2_SCOPE_NODE(seg[node].nid), f, cs.level_mask, cs.fwq, cs.n_features,
                               b2_sample_count(cs.bynode, cs.n_level));
        s_skip = ok ? 0 : 1;
      }
      __syncthreads();
      const bool skip = s_skip != 0;
      __syncthreads();
      if (skip) continue;
    }
    const int sl = slot >> log2_shards;
    const long long* hg = level_hist + (size_t)nd.hist_index * slice_elems + (size_t)(group * 2) * B2_BINS * sp + sl;
    const long long* hh = hg + (size_t)B2_BINS * sp;
    const int nf = nbins[f];
    long long g = 0, h = 0;
    if (b < nf) { g = hg[b * sp]; h = hh[b * sp]; }
    // feature totals over the real categories (the rest of the node's rows are missing on this feature)
    long long rg = g, rh = h;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { rg += __shfl_xor_sync(0xffffffffu, rg, o); rh += __shfl_xor_sync(0xffffffffu, rh, o); }
    if (lane == 0) { s_red[0][warp] = rg; s_red[1][warp] = rh; }
    __syncthreads();
    long long real_g = 0, real_h = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) { real_g += s_red[0][k]; real_h += s_red[1][k]; }
    Best best; best.key = 0; best.bin = 0; best.default_left = 0; best.lg = 0; best.lh = 0;
    int my_mode = 0, my_part = 0, rank = 0;
    if (nf < p.max_cat_to_onehot) {
      // one category against the rest: first with the missing rows on the left, then on the right
      if (b < nf) {
        const long long mg = tot_g - real_g, mh = tot_h - real_h;
#pragma unroll
        for (int pass = 0; pass < 2; ++pass) {
          const long long rgi = pass ? g + mg : g, rhi = pass ? h + mh : h;
          const double rh_d = __dmul_rn(__ll2double_rn(rhi), p.inv_scale_h), lh_d = __dadd_rn(H, -rh_d);
          if (lh_d >= p.min_child_weight && rh_d >= p.min_child_weight) {
            const double rg_d = __dmul_rn(__ll2double_rn(rgi), p.inv_scale_g), lg_d = __dadd_rn(G, -rg_d);
            const double gain = __dadd_rn(__dadd_rn(calc_gain(lg_d, lh_d, p), calc_gain(rg_d, rh_d, p)), -root_gain);
            const unsigned long long before = best.key;
            consider(best, __double2float_rn(gain), (uint32_t)f * 1024u + (uint32_t)(2 * b + pass), b, pass ? 0 : 1,
                     tot_g - rgi, tot_h - rhi);
            if (best.key != before) { my_mode = 0; my_part = b; }
          }
        }
      }
    } else {
      // stable ascending sort of the categories by leaf weight (rank by counting), prefix sums in sorted order
      const float w = b < nf ? calc_weight_f(__dmul_rn(__ll2double_rn(g), p.inv_scale_g), __dmul_rn(__ll2double_rn(h), p.inv_scale_h), p)
                             : 0.0f;
      s_w[b] = w; s_g[b] = 0; s_h[b] = 0;
      __syncthreads();
      if (b < nf) {
        for (int k = 0; k < nf; ++k) { const float wk = s_w[k]; rank += (wk < w || (wk == w && k < b)) ? 1 : 0; }
        s_g[rank] = g; s_h[rank] = h;
      }
      __syncthreads();
      long long pg, ph;
      Scan(scan_tmp).InclusiveSum(s_g[b], pg);
      __syncthreads();
      Scan(scan_tmp).InclusiveSum(s_h[b], ph);
      __syncthreads();
      s_g[b] = pg; s_h[b] = ph;                                   // s_g[k] = sum of the k+1 lightest categories
      __syncthreads();
      const int n_iter = min(p.max_cat_threshold, nf) - 1;
      const int k = b;                                            // sorted position handled by this thread
      if (k < n_iter) {   // forward: the k+1 lightest categories go right, missing left
        const double rh_d = __dmul_rn(__ll2double_rn(ph), p.inv_scale_h), lh_d = __dadd_rn(H, -rh_d);
        if (lh_d >= p.min_child_weight && rh_d >= p.min_child_weight) {
          const double rg_d = __dmul_rn(__ll2double_rn(pg), p.inv_scale_g), lg_d = __dadd_rn(G, -rg_d);
          const double gain = __dadd_rn(__dadd_rn(calc_gain(lg_d, lh_d, p), calc_gain(rg_d, rh_d, p)), -root_gain);
          const unsigned long long before = best.key;
          consider(best, __double2float_rn(gain), (uint32_t)f * 1024u + (uint32_t)k, -1, 1, tot_g - pg, tot_h - ph);
          if (best.key != before) { my_mode = 1; my_part = k + 1; }
        }
      }
      if (n_iter > 0 && k >= nf - n_iter && k < nf) {   // backward: categories at sorted positions >= k go left, missing right
        const long long lgi = real_g - s_g[k - 1], lhi = real_h - s_h[k - 1];
        const double lh_d = __dmul_rn(__ll2double_rn(lhi), p.inv_scale_h), rh_d = __dadd_rn(H, -lh_d);
        if (lh_d >= p.min_child_weight && rh_d >= p.min_child_weight) {
          const double lg_d = __dmul_rn(__ll2double_rn(lgi), p.inv_scale_g), rg_d = __dadd_rn(G, -lg_d);
          const double gain = __dadd_rn(__dadd_rn(calc_gain(lg_d, lh_d, p), calc_gain(rg_d, rh_d, p)), -root_gain);
          const unsigned long long before = best.key;
          consider(best, __double2float_rn(gain), (uint32_t)f * 1024u + 512u + (uint32_t)(nf - 1 - k), -1, 0, lgi, lhi);
          if (best.key != before) { my_mode = 1; my_part = k; }
        }
      }
    }
    // block argmax of this feature, then against the running best of the CTA
    unsigned long long key = best.key;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o); key = other > key ? other : key; }
    if (lane == 0) s_wkey[warp] = key;
    __syncthreads();
    unsigned long long kmax = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) kmax = s_wkey[i] > kmax ? s_wkey[i] : kmax;
    // keys order by (loss_chg, then earlier enumeration): later features only win with a strictly larger loss_chg
    const bool better = kmax != 0 && (uint32_t)(kmax >> 32) > (uint32_t)(s_best_key >> 32);
    __syncthreads();
    if (better) {
      if (best.key == kmax) {
        s_best.loss_chg = __uint_as_float((uint32_t)(kmax >> 32)); s_best.feature = f; s_best.bin = best.bin;
        s_best.default_left = best.default_left; s_best.left_g = best.lg; s_best.left_h = best.lh;
        s_best.order = 0xffffffffu - (uint32_t)(kmax & 0xffffffffu); s_best.is_cat = 1;
        s_mode = my_mode; s_part = my_part; s_best_key = kmax;
      }
      if (b < 8) s_bits[b] = 0;
      __syncthreads();
      if (b < nf && (s_mode == 0 ? (b == s_part) : (rank < s_part))) atomicOr(&s_bits[b >> 5], 1u << (b & 31));
      __syncthreads();
    }
  }
  if (b == 0) {
    B2SplitCand* out = cands + (size_t)node * cand_stride + cand_offset + j;
    if (s_best_key == 0) {
      out->loss_chg = 0.0f; out->feature = -1; out->bin = 0; out->default_left = 0; out->left_g = 0; out->left_h = 0;
      out->order = 0xffffffffu; out->is_cat = 0;
    } else {
      *out = s_best;
#pragma unroll
      for (int i = 0; i < 8; ++i) out->cat_bits[i] = s_bits[i];
    }
  }
}

// root totals: sum of all 256 bins of slot 0 / group 0 (every row lands in exactly one bin, the
// missing sentinel included) -> nodes[0].sum_g/h and root_gain, and the root's sums in the tree table
__global__ void root_totals_kernel(const long long* __restrict__ level_hist, int n_groups, B2EvalNode* nodes,
                                   const int32_t* __restrict__ qexp, int qbits, B2TrainParamDev p, int log2_shards,
                                   long long* __restrict__ tree_sum_g, long long* __restrict__ tree_sum_h) {
  __shared__ long long sg[256], sh[256];
  const int sp = B2_GROUP_SLOTS >> log2_shards;
  const size_t slice_elems = (size_t)n_groups * 2 * B2_BINS * sp;
  // any owned slot works (padding slots too): every row lands in exactly one bin of every slot
  const long long* hg = level_hist + (size_t)nodes[0].hist_index * slice_elems;
  sg[threadIdx.x] = hg[(size_t)threadIdx.x * sp];
  sh[threadIdx.x] = hg[(size_t)(B2_BINS + threadIdx.x) * sp];
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) { sg[threadIdx.x] += sg[threadIdx.x + o]; sh[threadIdx.x] += sh[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    p.inv_scale_g = ldexp(1.0, qexp[0] - qbits);
    p.inv_scale_h = ldexp(1.0, qexp[1] - qbits);
    nodes[0].sum_g = sg[0]; nodes[0].sum_h = sh[0];
    tree_sum_g[0] = sg[0]; tree_sum_h[0] = sh[0];
    double G = __dmul_rn(__ll2double_rn(sg[0]), p.inv_scale_g), H = __dmul_rn(__ll2double_rn(sh[0]), p.inv_scale_h);
    nodes[0].root_gain = __double2float_rn(calc_gain(G, H, p));
  }
}

}  // namespace b2

extern "C" {
// candidates per node written by the scan of a level of max_nodes nodes (the layout depends on the node count)
int b2_eval_ctas_per_node(int n_groups, int log2_shards, int max_nodes) {
  return b2::eval_ctas_per_node(n_groups, B2_GROUP_SLOTS >> log2_shards, max_nodes <= b2::kNarrowMaxNodes ? b2::kEvalSlots : 32);
}
int b2_eval_narrow_max_nodes() { return b2::kNarrowMaxNodes; }
// dec != nullptr (levels of at most b2_eval_narrow_max_nodes() nodes): the last CTA decides the level, decide_kernel is
// then not launched; done = its arrival counter
int b2_launch_eval_splits(const long long* level_hist, int n_groups, const B2EvalNode* nodes, int n_nodes,
                          const int32_t* group_first, const int32_t* group_size, const int32_t* nbins,
                          const uint8_t* has_missing, const uint8_t* is_cat, const int32_t* qexp, int qbits, B2TrainParamDev p,
                          B2SplitCand* cands, int cand_stride, const B2LevelCtl* ctl, int log2_shards, int shard_rank,
                          B2ColSample cs, const B2NodeSeg* seg, B2SiblingSub sub, const B2DecideArgs* dec, uint32_t* done,
                          cudaStream_t stream) {
  if (n_nodes <= 0) return 0;   // with ctl: n_nodes is the upper bound of the level
  B2DecideArgs d;
  if (dec) d = *dec; else memset(&d, 0, sizeof(d));
  const int cpn = b2_eval_ctas_per_node(n_groups, log2_shards, n_nodes);
  if (n_nodes <= b2::kNarrowMaxNodes)
    b2::eval_splits_kernel<<<n_nodes * cpn, b2::kEvalThreads, 0, stream>>>(level_hist, n_groups, nodes, group_first, group_size,
                                                                           nbins, has_missing, is_cat, qexp, qbits, p, cands,
                                                                           cand_stride, ctl, log2_shards, shard_rank, cs, seg, sub,
                                                                           dec ? 1 : 0, d, done);
  else if (dec) return (int)cudaErrorInvalidValue;
  else
    b2::eval_splits_wide_kernel<<<n_nodes * cpn, 32 * b2::kWideChunks, 0, stream>>>(level_hist, n_groups, nodes, group_first,
                                                                                     group_size, nbins, has_missing, is_cat, qexp,
                                                                                     qbits, p, cands, cand_stride, ctl,
                                                                                     log2_shards, shard_rank, cs, seg, sub);
  return (int)cudaGetLastError();
}
int b2_cat_ctas() { return b2::kCatCtas; }
// categorical features of the level's nodes; candidates go to cands[node*cand_stride + cand_offset + (0..kCatCtas)]
int b2_launch_eval_cat_splits(const long long* level_hist, int n_groups, const B2EvalNode* nodes, int n_nodes,
                              const int32_t* cat_feats, int n_cat, const int32_t* feat_byte, const int32_t* nbins,
                              const int32_t* qexp, int qbits, B2TrainParamDev p, B2SplitCand* cands, int cand_stride,
                              int cand_offset, const B2LevelCtl* ctl, int log2_shards, int shard_rank, B2ColSample cs,
                              const B2NodeSeg* seg, cudaStream_t stream) {
  if (n_nodes <= 0 || n_cat <= 0) return 0;
  b2::eval_cat_splits_kernel<<<n_nodes * b2::kCatCtas, 256, 0, stream>>>(level_hist, n_groups, nodes, cat_feats, n_cat, feat_byte,
                                                                        nbins, qexp, qbits, p, cands, cand_stride, cand_offset,
                                                                        ctl, log2_shards, shard_rank, cs, seg);
  return (int)cudaGetLastError();
}
int b2_launch_root_totals(const long long* level_hist, int n_groups, B2EvalNode* nodes, const int32_t* qexp, int qbits,
                          B2TrainParamDev p, int log2_shards, long long* tree_sum_g, long long* tree_sum_h,
                          cudaStream_t stream) {
  b2::root_totals_kernel<<<1, 256, 0, stream>>>(level_hist, n_groups, nodes, qexp, qbits, p, log2_shards, tree_sum_g, tree_sum_h);
  return (int)cudaGetLastError();
}
}
