// split_kernel.cu -- split-gain scan over the (allreduced) level histograms.
//
// Replaces XGBoost's EvaluateSplits stage reached through xgb.train()
// (xgboost_ray/main.py:745-752; SURVEY.md 8a row a12, Appendix A.6).  One CTA per
// (node, 4 feature slots); a thread scans 4 bins of one slot (eval_node_cta).
// Prefix sums are exact int64, gains are IEEE fp64 with explicit round-to-nearest ops (no fma
// contraction), so every rank and the CPU oracle compute identical candidates.
//
// The rules every scan shares are written once below -- node totals, slot addressing, the feature filter, the gain of
// one split, the enumeration order, the arg-max and the candidate write -- and each kernel keeps only its layout:
// which thread holds which bins, and how it builds their prefixes.
#include <string.h>

#include <cub/block/block_scan.cuh>

#include "common.cuh"
#include "decide.cuh"
#include "sampling.cuh"
#include "launch.h"

namespace b2 {

__device__ __forceinline__ double calc_gain(double G, double H, const B2TrainParamDev& p) {
  return b2_calc_gain(G, H, p.min_child_weight, p.lambda, p.alpha, p.max_delta_step);
}

struct Best {
  unsigned long long key = 0;  // (loss_chg bits << 32) | ~order ; 0 = none
  int32_t bin = 0, default_left = 0;
  long long lg = 0, lh = 0;
};

__device__ __forceinline__ void consider(Best& b, float chg, uint32_t order, int bin, int dl, long long lg, long long lh) {
  if (!(chg > 0.0f) || isinf(chg)) return;
  unsigned long long key = ((unsigned long long)__float_as_uint(chg) << 32) | (unsigned long long)(0xffffffffu - order);
  if (key > b.key) { b.key = key; b.bin = bin; b.default_left = dl; b.lg = lg; b.lh = lh; }
}

// Enumeration order of feature f's candidates (consider's tie-break): its forward candidates i = 0, 1, ... come before
// its backward ones.  A numeric scan's forward candidate at bin b is i = b, its backward one i = 255 - b.
__device__ __forceinline__ uint32_t fwd_order(int f, int i) { return (uint32_t)f * 1024u + (uint32_t)i; }
__device__ __forceinline__ uint32_t bwd_order(int f, int i) { return (uint32_t)f * 1024u + 512u + (uint32_t)i; }

// A node's totals as the gain sees them.  qe: the quantisation exponents of its gradients and hessians (qexp, or
// qexp + 2 k for target k of a vector-leaf tree).
struct NodeTotals {
  double inv_g, inv_h;   // inverse scales 2^(e - qbits)
  double G, H;
  double root_gain;      // the node's own gain, subtracted from every split's
};
__device__ __forceinline__ NodeTotals node_totals(long long g, long long h, const int32_t* qe, int qbits, const B2TrainParamDev& p) {
  NodeTotals t;
  t.inv_g = ldexp(1.0, qe[0] - qbits);
  t.inv_h = ldexp(1.0, qe[1] - qbits);
  t.G = __dmul_rn(__ll2double_rn(g), t.inv_g);
  t.H = __dmul_rn(__ll2double_rn(h), t.inv_h);
  t.root_gain = calc_gain(t.G, t.H, p);
  return t;
}
// a node of the level: its gain is the fp32 one decide (root_totals_kernel at the root) stored with it
__device__ __forceinline__ NodeTotals node_totals(const B2EvalNode& nd, const int32_t* qexp, int qbits, const B2TrainParamDev& p) {
  NodeTotals t = node_totals(nd.sum_g, nd.sum_h, qexp, qbits, p);
  t.root_gain = (double)nd.root_gain;
  return t;
}

// Loss change of the split whose `known` child has the fixed-point sums (cg, ch); the other child holds the rest of
// the node.  0, which consider() never takes, when either child's hessian is below min_child_weight.  The two gains
// are always added left + right, so the result does not depend on which child the scan knows.
enum Child { kLeft, kRight };
__device__ __forceinline__ float split_gain(Child known, long long cg, long long ch, const NodeTotals& t, const B2TrainParamDev& p) {
  const double kh = __dmul_rn(__ll2double_rn(ch), t.inv_h);
  if (!(kh >= p.min_child_weight)) return 0.0f;
  const double oh = __dadd_rn(t.H, -kh);
  if (!(oh >= p.min_child_weight)) return 0.0f;
  const double kg = __dmul_rn(__ll2double_rn(cg), t.inv_g), og = __dadd_rn(t.G, -kg);
  const bool l = known == kLeft;
  const double gain = __dadd_rn(__dadd_rn(calc_gain(l ? kg : og, l ? kh : oh, p), calc_gain(l ? og : kg, l ? oh : kh, p)),
                                -t.root_gain);
  return __double2float_rn(gain);
}

// Where virtual slot v of a node lives.  This rank owns sp = 32 >> log2_shards slots of every group (slot s is owned
// by s % shards), so the node's n_groups * sp owned slots are numbered group-major: v = group * sp + s / shards.
//
// Sibling subtraction in the scan (B2SiblingSub, parent_level != nullptr): a node whose histogram slot is a sibling
// slot (>= sib_base) was never built or subtracted.  Its bins are formed in registers as parent - built, exact int64,
// with (parent slot, built slot) = triples[3 j], triples[3 j + 1] for j = slot - sib_base.  With sib_out the CTA also
// stores the whole sibling slice (every bin of every slot it covers, sampled or not), because the next level reads it
// as a parent.  level_hist is only read at built slots in this mode, sib_out only at sibling slots, so the two never
// alias.
struct SlotAddr {
  bool v_ok;                     // v < n_groups * sp
  bool fused;                    // the node's bins are parent - built (uniform over the CTA)
  int group, slot, f;            // group, real slot inside it, feature
  const long long *hg, *hh;      // g / h plane of the node's slot (fused: of the built sibling)
  const long long *pgp, *php;    // fused: the parent's
  long long *sgp, *shp;          // fused with sib_out: where the node's bins are stored
};
__device__ __forceinline__ SlotAddr slot_addr(const long long* level_hist, int v, int n_groups, int log2_shards, int shard_rank,
                                              int hist_index, const B2SiblingSub& sub, const int32_t* __restrict__ group_first) {
  const int sp = B2_GROUP_SLOTS >> log2_shards;
  SlotAddr a;
  a.v_ok = v < n_groups * sp;
  a.group = a.v_ok ? v / sp : 0;
  const int sl = a.v_ok ? v % sp : 0;
  a.slot = (sl << log2_shards) + shard_rank;
  const size_t slice_elems = (size_t)n_groups * 2 * B2_BINS * sp;
  const size_t in_slice = (size_t)(a.group * 2) * B2_BINS * sp + sl;
  a.fused = sub.parent_level != nullptr && hist_index >= sub.sib_base;
  const int pair = a.fused ? hist_index - sub.sib_base : 0;
  a.hg = level_hist + (size_t)(a.fused ? sub.triples[3 * pair + 1] : hist_index) * slice_elems + in_slice;
  a.hh = a.hg + (size_t)B2_BINS * sp;
  a.pgp = a.fused ? sub.parent_level + (size_t)sub.triples[3 * pair] * slice_elems + in_slice : nullptr;
  a.php = a.fused ? a.pgp + (size_t)B2_BINS * sp : nullptr;
  a.sgp = (a.fused && sub.sib_out) ? sub.sib_out + (size_t)hist_index * slice_elems + in_slice : nullptr;
  a.shp = a.sgp ? a.sgp + (size_t)B2_BINS * sp : nullptr;
  a.f = group_first[a.group] + a.slot;
  return a;
}

// Whether feature f may split node nid: in the level's column sample (colsample_bytree / bylevel), in the node's own
// (colsample_bynode), and in an interaction set that holds the node's path.
__device__ __forceinline__ bool feature_allowed(const B2ColSample& cs, int nid, int f) {
  if (cs.level_mask && cs.level_mask[f] == 0) return false;
  if (cs.bynode < 1.0 &&
      !b2_col_selected(cs.seed, cs.tree, B2_SCOPE_NODE(nid), f, cs.level_mask, cs.fwq, cs.n_features,
                       b2_sample_count(cs.bynode, cs.n_level)))
    return false;
  return !cs.ic.sets_of || b2_interaction_allowed(cs.ic, nid, f);
}

// active && feature_allowed for the slot s of a CTA whose threads s < kSlots hold one slot each.  Every thread applies
// the level mask itself (left to thread s alone, it costs eval_splits_wide_kernel 20 more bytes of spill stores); the
// per-node tests run once per slot, in thread s, and reach the CTA through shared memory.  The filter never changes
// v_ok, so the fused sibling subtraction still stores every slot.
template <int kSlots>
__device__ __forceinline__ bool slot_allowed(bool active, const B2ColSample& cs, int nid, int f, int s) {
  if (active && cs.level_mask) active = cs.level_mask[f] != 0;
  if (!(cs.bynode < 1.0) && !cs.ic.sets_of) return active;
  __shared__ uint8_t s_allowed[kSlots];
  if (threadIdx.x < kSlots) s_allowed[s] = active && feature_allowed(cs, nid, f);
  __syncthreads();
  return active && s_allowed[s];
}

// The largest key over the CTA's kWarps warps, in every thread (s_key: one word per warp).
template <int kWarps>
__device__ __forceinline__ unsigned long long block_max_key(unsigned long long k, unsigned long long (&s_key)[kWarps]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xffffffffu, k, o);
    k = other > k ? other : k;
  }
  if ((threadIdx.x & 31) == 0) s_key[threadIdx.x >> 5] = k;
  __syncthreads();
  unsigned long long kmax = 0;
#pragma unroll
  for (int i = 0; i < kWarps; ++i) kmax = s_key[i] > kmax ? s_key[i] : kmax;
  return kmax;
}

// the candidate of feature f whose key is the block maximum kmax
__device__ __forceinline__ void set_candidate(B2SplitCand& c, unsigned long long kmax, const Best& best, int f, int is_cat) {
  c.loss_chg = __uint_as_float((uint32_t)(kmax >> 32));
  c.feature = f; c.bin = best.bin; c.default_left = best.default_left;
  c.left_g = best.lg; c.left_h = best.lh; c.order = 0xffffffffu - (uint32_t)(kmax & 0xffffffffu); c.is_cat = is_cat;
}

// the CTA's candidate: written by the thread that holds the block maximum (thread 0 writes "none").  kFence: fenced
// for a decide in the last CTA of the grid.
template <bool kFence>
__device__ __forceinline__ void write_candidate(B2SplitCand* out, unsigned long long kmax, const Best& best, int f) {
  if (kmax == 0) {
    if (threadIdx.x == 0) {
      b2_no_candidate(*out);
      if (kFence) __threadfence();
    }
  } else if (best.key == kmax) {
    set_candidate(*out, kmax, best, f, 0);
    if (kFence) __threadfence();
  }
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

struct SlotPrefixScratch {
  long long wg[kEvalWarps][kEvalSlots], wh[kEvalWarps][kEvalSlots];   // warp totals, then carries
  long long tg[kEvalSlots], th[kEvalSlots];                           // sums over a slot's real bins
};

// In the 4-slot layout: the exclusive prefix (pg, ph) of the slot's bins before the thread's first bin, and the slot's
// sums (real_g, real_h).  The thread's total is scanned over the 8 lanes of the slot in the warp (lanes s, s + 4, ...,
// s + 28), plus the totals of the warps before.  A caller that reuses sm first waits until every thread has returned.
__device__ __forceinline__ void slot_prefix(SlotPrefixScratch& sm, const long long (&g)[kEvalBinsPerThread],
                                            const long long (&h)[kEvalBinsPerThread], long long& pg, long long& ph,
                                            long long& real_g, long long& real_h) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, s = threadIdx.x & (kEvalSlots - 1);
  long long tg = 0, th = 0;
#pragma unroll
  for (int i = 0; i < kEvalBinsPerThread; ++i) { tg += g[i]; th += h[i]; }
  long long ig = tg, ih = th;
#pragma unroll
  for (int o = kEvalSlots; o < 32; o <<= 1) {
    const long long ug = __shfl_up_sync(0xffffffffu, ig, o), uh = __shfl_up_sync(0xffffffffu, ih, o);
    if (lane >= o) { ig += ug; ih += uh; }
  }
  if (lane >= 32 - kEvalSlots) { sm.wg[warp][s] = ig; sm.wh[warp][s] = ih; }
  __syncthreads();
  if (threadIdx.x < kEvalSlots) {
    long long cg = 0, ch = 0;
#pragma unroll
    for (int w = 0; w < kEvalWarps; ++w) {
      const long long a = sm.wg[w][threadIdx.x], c = sm.wh[w][threadIdx.x];
      sm.wg[w][threadIdx.x] = cg; sm.wh[w][threadIdx.x] = ch;
      cg += a; ch += c;
    }
    sm.tg[threadIdx.x] = cg; sm.th[threadIdx.x] = ch;
  }
  __syncthreads();
  pg = sm.wg[warp][s] + ig - tg; ph = sm.wh[warp][s] + ih - th;
  real_g = sm.tg[s]; real_h = sm.th[s];
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

__device__ __forceinline__ void eval_node_cta(const long long* __restrict__ level_hist, int n_groups, const B2EvalNode& nd, int node,
                                              int cta_in_node, const int32_t* __restrict__ group_first,
                                              const int32_t* __restrict__ group_size, const int32_t* __restrict__ nbins,
                                              const uint8_t* __restrict__ has_missing, const uint8_t* __restrict__ is_cat,
                                              const int32_t* __restrict__ qexp, int qbits, const B2TrainParamDev& p,
                                              B2SplitCand* cands, int cand_stride, int log2_shards, int shard_rank,
                                              const B2ColSample& cs, const B2NodeSeg* __restrict__ seg, const B2SiblingSub& sub) {
  __shared__ SlotPrefixScratch s_pre;
  __shared__ unsigned long long s_key[kEvalWarps];
  const int sp = B2_GROUP_SLOTS >> log2_shards;
  const int s = threadIdx.x & (kEvalSlots - 1), b0 = (threadIdx.x / kEvalSlots) * kEvalBinsPerThread;
  const SlotAddr a = slot_addr(level_hist, cta_in_node * kEvalSlots + s, n_groups, log2_shards, shard_rank, nd.hist_index, sub,
                               group_first);
  const int f = a.f;
  const bool active = slot_allowed<kEvalSlots>(a.v_ok && a.slot < group_size[a.group] && !(is_cat && is_cat[f]), cs,
                                               seg[node].nid, f, s);
  const int nf = active ? nbins[f] : 0;
  const bool fmiss = active ? (has_missing[f] != 0) : false;

  // the thread's bins; bins at or past nf (and inactive slots) count as zero
  long long g[kEvalBinsPerThread], h[kEvalBinsPerThread];
#pragma unroll
  for (int i = 0; i < kEvalBinsPerThread; ++i) { g[i] = 0; h[i] = 0; }
  if (a.fused) {
    if (a.v_ok && (a.sgp || active)) {
#pragma unroll
      for (int i = 0; i < kEvalBinsPerThread; ++i) {
        const int b = b0 + i;
        g[i] = a.pgp[b * sp] - a.hg[b * sp]; h[i] = a.php[b * sp] - a.hh[b * sp];
      }
      if (a.sgp) {
#pragma unroll
        for (int i = 0; i < kEvalBinsPerThread; ++i) { a.sgp[(b0 + i) * sp] = g[i]; a.shp[(b0 + i) * sp] = h[i]; }
      }
#pragma unroll
      for (int i = 0; i < kEvalBinsPerThread; ++i)
        if (b0 + i >= nf) { g[i] = 0; h[i] = 0; }
    }
  } else if (active) {
#pragma unroll
    for (int i = 0; i < kEvalBinsPerThread; ++i) {
      const int b = b0 + i;
      if (b < nf) { g[i] = a.hg[b * sp]; h[i] = a.hh[b * sp]; }
    }
  }
  long long pg, ph, real_g, real_h;
  slot_prefix(s_pre, g, h, pg, ph, real_g, real_h);
  const NodeTotals t = node_totals(nd, qexp, qbits, p);
  const bool node_has_missing = fmiss && (real_g != nd.sum_g || real_h != nd.sum_h);
  Best best;
#pragma unroll
  for (int i = 0; i < kEvalBinsPerThread; ++i) {
    const int b = b0 + i;
    if (b >= nf) break;
    const long long eg_excl = pg, eh_excl = ph;
    pg += g[i]; ph += h[i];
    // forward: left = prefix inclusive, missing -> right
    consider(best, split_gain(kLeft, pg, ph, t, p), fwd_order(f, b), b, 0, pg, ph);
    if (node_has_missing) {  // backward at bin b: right' = sum of real bins >= b, missing -> left
      const long long rg = real_g - eg_excl, rh = real_h - eh_excl;
      consider(best, split_gain(kRight, rg, rh, t, p), bwd_order(f, 255 - b), b - 1, 1, nd.sum_g - rg, nd.sum_h - rh);
    }
  }
  write_candidate<true>(cands + (size_t)node * cand_stride + cta_in_node, block_max_key(best.key, s_key), best, f);
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
// saves.  With sibling subtraction (slot_addr) the bin scan re-reads the sibling's bins this thread stored; without
// sib_out (the last histogram level) nothing is stored and the scan subtracts again.
constexpr int kWideChunks = 32;                 // bin chunks per feature
constexpr int kWideBinsPerChunk = 256 / kWideChunks;

__global__ void __launch_bounds__(32 * kWideChunks)
eval_splits_wide_kernel(const long long* __restrict__ level_hist, int n_groups, const B2EvalNode* __restrict__ nodes,
                   const int32_t* __restrict__ group_first, const int32_t* __restrict__ group_size,
                   const int32_t* __restrict__ nbins, const uint8_t* __restrict__ has_missing,
                   const uint8_t* __restrict__ is_cat /* nullable: categorical features are scanned by eval_cat_splits_kernel */,
                   const int32_t* __restrict__ qexp, int qbits, B2TrainParamDev p, B2SplitCand* __restrict__ cands,
                   int cand_stride, const B2LevelCtl* __restrict__ ctl, int log2_shards, int shard_rank, B2ColSample cs,
                   const B2NodeSeg* __restrict__ seg, B2SiblingSub sub) {
  // the node's owned slots are covered by cpn = ceil(n_groups * sp / 32) CTAs
  const int sp = B2_GROUP_SLOTS >> log2_shards;
  const int cpn = (n_groups * sp + 31) >> 5;
  const int node = blockIdx.x / cpn, cta_in_node = blockIdx.x % cpn;
  if (ctl && node >= ctl->n_nodes) return;
  const int s = threadIdx.x & 31, q = threadIdx.x >> 5;
  __shared__ long long cs_g[kWideChunks][32], cs_h[kWideChunks][32];
  __shared__ unsigned long long s_key[kWideChunks];
  const B2EvalNode nd = nodes[node];
  const NodeTotals t = node_totals(nd, qexp, qbits, p);
  const SlotAddr a = slot_addr(level_hist, cta_in_node * 32 + s, n_groups, log2_shards, shard_rank, nd.hist_index, sub, group_first);
  const int f = a.f;
  const bool active = slot_allowed<32>(a.v_ok && a.slot < group_size[a.group] && !(is_cat && is_cat[f]), cs, seg[node].nid, f, s);
  const int nf = active ? nbins[f] : 0;
  const bool fmiss = active ? (has_missing[f] != 0) : false;

  long long sg = 0, sh = 0;
  if (a.fused) {
    if (a.v_ok && (a.sgp || active)) {
#pragma unroll
      for (int i = 0; i < kWideBinsPerChunk; ++i) {
        const int b = q * kWideBinsPerChunk + i;
        const long long g = a.pgp[b * sp] - a.hg[b * sp], h = a.php[b * sp] - a.hh[b * sp];
        if (a.sgp) { a.sgp[b * sp] = g; a.shp[b * sp] = h; }
        if (active && b < nf) { sg += g; sh += h; }
      }
    }
  } else if (active) {
#pragma unroll
    for (int i = 0; i < kWideBinsPerChunk; ++i) {
      int b = q * kWideBinsPerChunk + i;
      if (b < nf) { sg += a.hg[b * sp]; sh += a.hh[b * sp]; }
    }
  }
  cs_g[q][s] = sg; cs_h[q][s] = sh;
  __syncthreads();
  long long pg = 0, ph = 0, real_g = 0, real_h = 0;
#pragma unroll 8
  for (int k = 0; k < kWideChunks; ++k) {
    const long long cg = cs_g[k][s], ch = cs_h[k][s];
    if (k < q) { pg += cg; ph += ch; }
    real_g += cg; real_h += ch;
  }
  const bool node_has_missing = fmiss && (real_g != nd.sum_g || real_h != nd.sum_h);
  Best best;
  if (active) {
#pragma unroll 2
    for (int i = 0; i < kWideBinsPerChunk; ++i) {
      const int b = q * kWideBinsPerChunk + i;
      if (b >= nf) break;
      const long long eg_excl = pg, eh_excl = ph;
      if (!a.fused) { pg += a.hg[b * sp]; ph += a.hh[b * sp]; }
      else if (a.sgp) { pg += a.sgp[b * sp]; ph += a.shp[b * sp]; }   // stored by this thread in the first pass
      else { pg += a.pgp[b * sp] - a.hg[b * sp]; ph += a.php[b * sp] - a.hh[b * sp]; }
      // forward: left = prefix inclusive, missing -> right
      consider(best, split_gain(kLeft, pg, ph, t, p), fwd_order(f, b), b, 0, pg, ph);
      if (node_has_missing) {  // backward at bin b: right' = sum of real bins >= b, missing -> left
        const long long rg = real_g - eg_excl, rh = real_h - eh_excl;
        consider(best, split_gain(kRight, rg, rh, t, p), bwd_order(f, 255 - b), b - 1, 1, nd.sum_g - rg, nd.sum_h - rh);
      }
    }
  }
  write_candidate<false>(cands + (size_t)node * cand_stride + cta_in_node, block_max_key(best.key, s_key), best, f);
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
  const NodeTotals t = node_totals(nd, qexp, qbits, p);
  const long long tot_g = nd.sum_g, tot_h = nd.sum_h;
  if (b == 0) s_best_key = 0;
  __syncthreads();
  for (int ci = j; ci < n_cat; ci += kCatCtas) {
    const int f = cat_feats[ci];
    const int fb = feat_byte[f], group = fb >> 5, slot = fb & 31;
    if ((slot & (shards - 1)) != shard_rank) continue;          // another rank owns this slot (uniform)
    if (cs.level_mask || cs.bynode < 1.0 || cs.ic.sets_of) {    // column sampling, interaction constraints (uniform per feature)
      if (b == 0) s_skip = feature_allowed(cs, seg[node].nid, f) ? 0 : 1;
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
    Best best;
    int my_mode = 0, my_part = 0, rank = 0;
    if (nf < p.max_cat_to_onehot) {
      // one category against the rest: first with the missing rows on the left, then on the right
      if (b < nf) {
        const long long mg = tot_g - real_g, mh = tot_h - real_h;
#pragma unroll
        for (int pass = 0; pass < 2; ++pass) {
          const long long rgi = pass ? g + mg : g, rhi = pass ? h + mh : h;
          const unsigned long long before = best.key;
          consider(best, split_gain(kRight, rgi, rhi, t, p), fwd_order(f, 2 * b + pass), b, pass ? 0 : 1, tot_g - rgi, tot_h - rhi);
          if (best.key != before) { my_mode = 0; my_part = b; }
        }
      }
    } else {
      // stable ascending sort of the categories by leaf weight (rank by counting), prefix sums in sorted order
      const float w = b < nf ? calc_weight_f(__dmul_rn(__ll2double_rn(g), t.inv_g), __dmul_rn(__ll2double_rn(h), t.inv_h), p)
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
        const unsigned long long before = best.key;
        consider(best, split_gain(kRight, pg, ph, t, p), fwd_order(f, k), -1, 1, tot_g - pg, tot_h - ph);
        if (best.key != before) { my_mode = 1; my_part = k + 1; }
      }
      if (n_iter > 0 && k >= nf - n_iter && k < nf) {   // backward: categories at sorted positions >= k go left, missing right
        const long long lgi = real_g - s_g[k - 1], lhi = real_h - s_h[k - 1];
        const unsigned long long before = best.key;
        consider(best, split_gain(kLeft, lgi, lhi, t, p), bwd_order(f, nf - 1 - k), -1, 0, lgi, lhi);
        if (best.key != before) { my_mode = 1; my_part = k; }
      }
    }
    // block argmax of this feature, then against the running best of the CTA
    const unsigned long long kmax = block_max_key(best.key, s_wkey);
    // keys order by (loss_chg, then earlier enumeration): later features only win with a strictly larger loss_chg
    const bool better = kmax != 0 && (uint32_t)(kmax >> 32) > (uint32_t)(s_best_key >> 32);
    __syncthreads();
    if (better) {
      if (best.key == kmax) {
        set_candidate(s_best, kmax, best, f, 1);
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
      b2_no_candidate(*out);
    } else {
      *out = s_best;
#pragma unroll
      for (int i = 0; i < 8; ++i) out->cat_bits[i] = s_bits[i];
    }
  }
}

// Sums of the 256 bins of one slot (g plane at hg, h plane B2_BINS * sp elements on) by a CTA of 256 threads, valid in
// thread 0.  Every row lands in exactly one bin of every slot, the missing sentinel included, so any owned slot (padding
// slots too) gives the node's totals.  Only thread 0 reads the scratch after the last barrier, so a loop may call this
// again at once.
__device__ __forceinline__ void slot_sums(const long long* __restrict__ hg, int sp, long long& g, long long& h) {
  __shared__ long long sg[256], sh[256];
  sg[threadIdx.x] = hg[(size_t)threadIdx.x * sp];
  sh[threadIdx.x] = hg[(size_t)(B2_BINS + threadIdx.x) * sp];
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) { sg[threadIdx.x] += sg[threadIdx.x + o]; sh[threadIdx.x] += sh[threadIdx.x + o]; }
    __syncthreads();
  }
  g = sg[0]; h = sh[0];
}

// root totals: the sums of slot 0 / group 0 -> nodes[0].sum_g/h and root_gain, and the root's sums in the tree table
__global__ void root_totals_kernel(const long long* __restrict__ level_hist, int n_groups, B2EvalNode* nodes,
                                   const int32_t* __restrict__ qexp, int qbits, B2TrainParamDev p, int log2_shards,
                                   long long* __restrict__ tree_sum_g, long long* __restrict__ tree_sum_h) {
  const int sp = B2_GROUP_SLOTS >> log2_shards;
  const size_t slice_elems = (size_t)n_groups * 2 * B2_BINS * sp;
  long long g, h;
  slot_sums(level_hist + (size_t)nodes[0].hist_index * slice_elems, sp, g, h);
  if (threadIdx.x == 0) {
    nodes[0].sum_g = g; nodes[0].sum_h = h;
    tree_sum_g[0] = g; tree_sum_h[0] = h;
    nodes[0].root_gain = __double2float_rn(node_totals(g, h, qexp, qbits, p).root_gain);
  }
}

// ---------------------------------------------------------------- vector-leaf trees (multi_strategy=multi_output_tree)
// DESIGN.md 2 item 19.  One tree for T targets: target k has its own quantisation exponents (qexp[2k], qexp[2k + 1]) and
// its own level histograms at level_hist + k * tstride (the scalar layout, one node slot per hist_index).  vtot holds
// every node's per-target fixed-point totals [nid][T][g, h] and vgain its fp32 gain(node) = fp32(sum_k CalcGain(G_k, H_k)).
__device__ __forceinline__ double vector_gain(const long long* __restrict__ tot, int T, const int32_t* __restrict__ qexp, int qbits,
                                              const B2TrainParamDev& p) {
  double acc = 0.0;
  for (int k = 0; k < T; ++k) acc = __dadd_rn(acc, node_totals(tot[2 * k], tot[2 * k + 1], qexp + 2 * k, qbits, p).root_gain);
  return acc;
}

// The narrow layout of eval_node_cta for every level (4 slots x 256 bins per CTA, 2 bins per thread), looping over the
// targets: per target the exact int64 prefix of the thread's bins, then that target's CalcGain terms added, in ascending
// k, to one double accumulator per (bin, direction, child).  A child "has hessian" when its hessian sum is nonzero in
// some target; the two bits ride in the candidate's left_g / left_h for decide's expand test.  No min_child_weight
// filter: a target below it adds 0.  Backward candidates exist when the feature has missing values and, for some
// target, the node's sums over the real bins differ from its totals.
__global__ void __launch_bounds__(kEvalThreads, 1)
eval_splits_vector_kernel(const long long* __restrict__ level_hist, size_t tstride, int T, int n_groups,
                          const B2EvalNode* __restrict__ nodes, const long long* __restrict__ vtot, const float* __restrict__ vgain,
                          const int32_t* __restrict__ group_first, const int32_t* __restrict__ group_size,
                          const int32_t* __restrict__ nbins, const uint8_t* __restrict__ has_missing,
                          const int32_t* __restrict__ qexp, int qbits, B2TrainParamDev p, B2SplitCand* cands, int cand_stride,
                          const B2LevelCtl* __restrict__ ctl, B2ColSample cs, const B2NodeSeg* __restrict__ seg) {
  const int sp = B2_GROUP_SLOTS;
  const int cpn = eval_ctas_per_node(n_groups, sp, kEvalSlots);
  const int node = blockIdx.x / cpn, cta_in_node = blockIdx.x % cpn;
  if (node >= ctl->n_nodes) return;   // uniform over the CTA
  __shared__ SlotPrefixScratch s_pre;
  __shared__ unsigned long long s_key[kEvalWarps];
  const int s = threadIdx.x & (kEvalSlots - 1), b0 = (threadIdx.x / kEvalSlots) * kEvalBinsPerThread;
  const B2EvalNode nd = nodes[node];
  const int nid = seg[node].nid;
  const SlotAddr a = slot_addr(level_hist, cta_in_node * kEvalSlots + s, n_groups, 0, 0, nd.hist_index, B2SiblingSub{}, group_first);
  const int f = a.f;
  const bool active = slot_allowed<kEvalSlots>(a.v_ok && a.slot < group_size[a.group], cs, nid, f, s);
  const int nf = active ? nbins[f] : 0;
  const bool fmiss = active ? (has_missing[f] != 0) : false;
  const long long* tot = vtot + (size_t)nid * T * 2;
  double acc_l[kEvalBinsPerThread][2], acc_r[kEvalBinsPerThread][2];   // [bin][forward, backward]
  bool nz_l[kEvalBinsPerThread][2], nz_r[kEvalBinsPerThread][2];
#pragma unroll
  for (int i = 0; i < kEvalBinsPerThread; ++i)
#pragma unroll
    for (int d = 0; d < 2; ++d) { acc_l[i][d] = 0.0; acc_r[i][d] = 0.0; nz_l[i][d] = false; nz_r[i][d] = false; }
  bool any_missing = false;
  for (int k = 0; k < T; ++k) {
    const long long* hg = a.hg + (size_t)k * tstride;
    const long long* hh = hg + (size_t)B2_BINS * sp;
    long long g[kEvalBinsPerThread], h[kEvalBinsPerThread];
#pragma unroll
    for (int i = 0; i < kEvalBinsPerThread; ++i) {
      const int b = b0 + i;
      g[i] = 0; h[i] = 0;
      if (b < nf) { g[i] = hg[b * sp]; h[i] = hh[b * sp]; }
    }
    __syncthreads();   // the previous target's carries are read
    long long pg, ph, real_g, real_h;
    slot_prefix(s_pre, g, h, pg, ph, real_g, real_h);
    const long long tot_g = tot[2 * k], tot_h = tot[2 * k + 1];
    const NodeTotals t = node_totals(tot_g, tot_h, qexp + 2 * k, qbits, p);
    any_missing = any_missing || (fmiss && (real_g != tot_g || real_h != tot_h));
#pragma unroll
    for (int i = 0; i < kEvalBinsPerThread; ++i) {
      if (b0 + i >= nf) break;
      const long long eg_excl = pg, eh_excl = ph;
      pg += g[i]; ph += h[i];
      {  // forward: left = prefix inclusive, missing -> right
        const double lh_d = __dmul_rn(__ll2double_rn(ph), t.inv_h), rh_d = __dadd_rn(t.H, -lh_d);
        const double lg_d = __dmul_rn(__ll2double_rn(pg), t.inv_g), rg_d = __dadd_rn(t.G, -lg_d);
        acc_l[i][0] = __dadd_rn(acc_l[i][0], calc_gain(lg_d, lh_d, p));
        acc_r[i][0] = __dadd_rn(acc_r[i][0], calc_gain(rg_d, rh_d, p));
        nz_l[i][0] = nz_l[i][0] || ph != 0; nz_r[i][0] = nz_r[i][0] || (tot_h - ph) != 0;
      }
      {  // backward at bin b: right = real bins >= b, missing -> left
        const long long rg_i = real_g - eg_excl, rh_i = real_h - eh_excl;
        const double rh_d = __dmul_rn(__ll2double_rn(rh_i), t.inv_h), lh_d = __dadd_rn(t.H, -rh_d);
        const double rg_d = __dmul_rn(__ll2double_rn(rg_i), t.inv_g), lg_d = __dadd_rn(t.G, -rg_d);
        acc_l[i][1] = __dadd_rn(acc_l[i][1], calc_gain(lg_d, lh_d, p));
        acc_r[i][1] = __dadd_rn(acc_r[i][1], calc_gain(rg_d, rh_d, p));
        nz_l[i][1] = nz_l[i][1] || (tot_h - rh_i) != 0; nz_r[i][1] = nz_r[i][1] || rh_i != 0;
      }
    }
  }
  const double parent_gain = (double)vgain[nid];
  Best best;
#pragma unroll
  for (int i = 0; i < kEvalBinsPerThread; ++i) {
    const int b = b0 + i;
    if (b >= nf) break;
    consider(best, __double2float_rn(__dadd_rn(__dadd_rn(acc_l[i][0], acc_r[i][0]), -parent_gain)), fwd_order(f, b),
             b, 0, nz_l[i][0] ? 1 : 0, nz_r[i][0] ? 1 : 0);
    if (any_missing)
      consider(best, __double2float_rn(__dadd_rn(__dadd_rn(acc_l[i][1], acc_r[i][1]), -parent_gain)), bwd_order(f, 255 - b),
               b - 1, 1, nz_l[i][1] ? 1 : 0, nz_r[i][1] ? 1 : 0);
  }
  write_candidate<true>(cands + (size_t)node * cand_stride + cta_in_node, block_max_key(best.key, s_key), best, f);
}

// the root's per-target totals (all 256 bins of slot 0 / group 0 of target k) and its gain
__global__ void __launch_bounds__(256)
vector_root_totals_kernel(const long long* __restrict__ level_hist, size_t tstride, int T, int n_groups,
                          const int32_t* __restrict__ qexp, int qbits, B2TrainParamDev p, long long* __restrict__ vtot,
                          float* __restrict__ vgain) {
  for (int k = 0; k < T; ++k) {
    long long g, h;
    slot_sums(level_hist + (size_t)k * tstride, B2_GROUP_SLOTS, g, h);
    if (threadIdx.x == 0) { vtot[2 * k] = g; vtot[2 * k + 1] = h; }
  }
  if (threadIdx.x == 0) vgain[0] = __double2float_rn(vector_gain(vtot, T, qexp, qbits, p));
}

// After decide: the per-target totals of the children of split j (one CTA each), from the parent's histogram in the
// level buffer -- left = the chosen feature's bins 0..split_bin, plus its missing rows (totals minus real bins) when
// default_left; right = parent - left -- and each child's gain.  ev_nxt's sums get target 0's totals, which pick the
// child whose histogram is built (level_finalize.cuh).
__global__ void __launch_bounds__(256)
vector_child_totals_kernel(const long long* __restrict__ level_hist, size_t tstride, int T, int n_groups,
                           const B2LevelCtl* __restrict__ ctl, const B2SplitWork* __restrict__ split_work,
                           const int32_t* __restrict__ pair_parent_hist, const B2NodeSeg* __restrict__ seg_nxt,
                           const int32_t* __restrict__ tree_parent, const int32_t* __restrict__ feat_byte,
                           const int32_t* __restrict__ nbins, const int32_t* __restrict__ qexp, int qbits, B2TrainParamDev p,
                           long long* __restrict__ vtot, float* __restrict__ vgain, B2EvalNode* __restrict__ ev_nxt) {
  const int j = blockIdx.x;
  if (j >= ctl->n_split) return;
  const int sp = B2_GROUP_SLOTS;
  const size_t slice_elems = (size_t)n_groups * 2 * B2_BINS * sp;
  const B2SplitWork w = split_work[j];
  const int l = seg_nxt[2 * j].nid, r = l + 1, par = tree_parent[l];
  const int fb = feat_byte[w.feature], nf = nbins[w.feature];
  const size_t off = (size_t)pair_parent_hist[j] * slice_elems + (size_t)((fb >> 5) * 2) * B2_BINS * sp + (fb & 31);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = warp; k < T; k += blockDim.x / 32) {
    const long long* hg = level_hist + (size_t)k * tstride + off;
    const long long* hh = hg + (size_t)B2_BINS * sp;
    long long pg = 0, ph = 0, rg = 0, rh = 0;
    for (int b = lane; b < B2_BINS; b += 32) {
      if (b >= nf) break;
      const long long a = hg[b * sp], c = hh[b * sp];
      rg += a; rh += c;
      if (b <= w.split_bin) { pg += a; ph += c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      pg += __shfl_xor_sync(0xffffffffu, pg, o); ph += __shfl_xor_sync(0xffffffffu, ph, o);
      rg += __shfl_xor_sync(0xffffffffu, rg, o); rh += __shfl_xor_sync(0xffffffffu, rh, o);
    }
    if (lane == 0) {
      const long long tg = vtot[((size_t)par * T + k) * 2], th = vtot[((size_t)par * T + k) * 2 + 1];
      if (w.default_left) { pg += tg - rg; ph += th - rh; }
      vtot[((size_t)l * T + k) * 2] = pg; vtot[((size_t)l * T + k) * 2 + 1] = ph;
      vtot[((size_t)r * T + k) * 2] = tg - pg; vtot[((size_t)r * T + k) * 2 + 1] = th - ph;
    }
  }
  __syncthreads();
  if (threadIdx.x < 2) {
    const int c = threadIdx.x == 0 ? l : r;
    const long long* t = vtot + (size_t)c * T * 2;
    vgain[c] = __double2float_rn(vector_gain(t, T, qexp, qbits, p));
    ev_nxt[2 * j + threadIdx.x].sum_g = t[0]; ev_nxt[2 * j + threadIdx.x].sum_h = t[1];
  }
}

}  // namespace b2

extern "C" {
int b2_launch_eval_splits_vector(const long long* level_hist, size_t tstride, int T, int n_groups, const B2EvalNode* nodes,
                                 int max_nodes, const long long* vtot, const float* vgain, const int32_t* group_first,
                                 const int32_t* group_size, const int32_t* nbins, const uint8_t* has_missing,
                                 const int32_t* qexp, int qbits, B2TrainParamDev p, B2SplitCand* cands, int cand_stride,
                                 const B2LevelCtl* ctl, B2ColSample cs, const B2NodeSeg* seg, cudaStream_t stream) {
  if (max_nodes <= 0) return 0;
  const int cpn = b2::eval_ctas_per_node(n_groups, B2_GROUP_SLOTS, b2::kEvalSlots);
  b2::eval_splits_vector_kernel<<<max_nodes * cpn, b2::kEvalThreads, 0, stream>>>(level_hist, tstride, T, n_groups, nodes, vtot, vgain,
                                                                                 group_first, group_size, nbins, has_missing, qexp,
                                                                                 qbits, p, cands, cand_stride, ctl, cs, seg);
  return (int)cudaGetLastError();
}
// candidates per node of the vector scan (the narrow layout at every level)
int b2_eval_vector_ctas_per_node(int n_groups) { return b2::eval_ctas_per_node(n_groups, B2_GROUP_SLOTS, b2::kEvalSlots); }
int b2_launch_vector_root_totals(const long long* level_hist, size_t tstride, int T, int n_groups, const int32_t* qexp, int qbits,
                                 B2TrainParamDev p, long long* vtot, float* vgain, cudaStream_t stream) {
  b2::vector_root_totals_kernel<<<1, 256, 0, stream>>>(level_hist, tstride, T, n_groups, qexp, qbits, p, vtot, vgain);
  return (int)cudaGetLastError();
}
int b2_launch_vector_child_totals(const long long* level_hist, size_t tstride, int T, int n_groups, int max_splits,
                                  const B2LevelCtl* ctl, const B2SplitWork* split_work, const int32_t* pair_parent_hist,
                                  const B2NodeSeg* seg_nxt, const int32_t* tree_parent, const int32_t* feat_byte,
                                  const int32_t* nbins, const int32_t* qexp, int qbits, B2TrainParamDev p, long long* vtot,
                                  float* vgain, B2EvalNode* ev_nxt, cudaStream_t stream) {
  if (max_splits <= 0) return 0;
  b2::vector_child_totals_kernel<<<max_splits, 256, 0, stream>>>(level_hist, tstride, T, n_groups, ctl, split_work, pair_parent_hist,
                                                                 seg_nxt, tree_parent, feat_byte, nbins, qexp, qbits, p, vtot,
                                                                 vgain, ev_nxt);
  return (int)cudaGetLastError();
}
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
