// common.cuh -- shared declarations for the sm_90a histogram-tree engine.
//
// Layouts (DESIGN.md "Data layout in HBM"):
//   bins      uint8 [n_rows][row_stride]     row_stride = n_groups*32; group g owns bytes
//                                            [g*32, g*32+gsize[g]) of a row, rest zero padding;
//                                            bin 255 is the missing sentinel
//   bins_col  uint8 [n_features][col_stride] feature-major copy, read by the row partition (1 byte/row
//                                            from a 128-byte row would cost a whole DRAM burst per row)
//   gpair     int2  [n_rows]                 (qg, qh) fixed-point gradient / hessian
//   hist      int64 [node][group][2][256][32] plane 0 = sum qg, plane 1 = sum qh, slot = feature
//                                            within group; 128 KiB per (node, group)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define B2_GROUP_SLOTS 32
#define B2_BINS 256
#define B2_MISSING_BIN 255
#define B2_PLANE_ELEMS (B2_BINS * B2_GROUP_SLOTS)          // 8192
#define B2_GROUP_ELEMS (2 * B2_PLANE_ELEMS)                // 16384 int64 per (node, group)

// ---- 40-bit fixed-point sums (leaf values, base_score) kept as two int64 limbs: value = hi * 2^24 + lo.
// A row adds |q| <= 2^40, so one int64 holds fewer than 2^23 rows of such values; a leaf or the intercept can hold
// many more.  Every writer sums an exact int64 partial first (a bounded number of rows) and adds it as
// (t >> 24, t & (2^24 - 1)): the high limbs add up to at most 2^(71-24) and the low limbs to at most 2^55 for fewer
// than 2^31 rows, so neither wraps, and limbs of different CTAs / ranks simply add.
#define B2_LIMB_SHIFT 24
__device__ __forceinline__ void b2_atomic_add_limbs(long long* hi_lo, long long t) {
  atomicAdd(reinterpret_cast<unsigned long long*>(hi_lo), (unsigned long long)(t >> B2_LIMB_SHIFT));
  atomicAdd(reinterpret_cast<unsigned long long*>(hi_lo) + 1, (unsigned long long)(t & ((1ll << B2_LIMB_SHIFT) - 1)));
}
// the correctly rounded value of hi * 2^24 + lo: carry lo's overflow into hi (|hi| < 2^53 and 0 <= lo < 2^24 are
// then exact doubles), one rounding in the add.  Equal to __ll2double_rn(sum) whenever the sum fits in an int64.
__device__ __forceinline__ double b2_limbs_to_double(long long hi, long long lo) {
  hi += lo >> B2_LIMB_SHIFT;
  lo &= (1ll << B2_LIMB_SHIFT) - 1;
  return __dadd_rn(__dmul_rn(__ll2double_rn(hi), (double)(1ll << B2_LIMB_SHIFT)), __ll2double_rn(lo));
}

// one entry per node whose histogram is built from rows in this launch
struct B2HistWork {
  int32_t seg_begin;    // first position in ridx (or first row id when ridx == nullptr)
  int32_t seg_count;    // rows of this node on this GPU
  int32_t hist_index;   // node slot in the output level buffer
  int32_t chunk_begin;  // exclusive prefix sum of ceil(seg_count / chunk_rows)
};

// CTA plan of the histogram kernel: a CTA type owns one PAIR of feature groups (2 x 64 KiB of shared memory); its
// share of the persistent grid is proportional to the shared-atomic wavefronts the pair costs per row, because the last
// group may be NARROW (w <= 16 features, processed one lane per row in w steps instead of two lanes in 16).
#define B2_HIST_MAX_TYPES 8
struct B2HistPlan {
  int32_t n_types;
  int32_t cta_begin[B2_HIST_MAX_TYPES + 1];   // type t owns CTAs [cta_begin[t], cta_begin[t+1])
  int32_t narrow_w;                           // width of the last group if it is narrow (power of two <= 16), else 0
};

// per-split-node descriptor for the row partition kernel
struct B2SplitWork {
  int32_t seg_begin, seg_count;
  int32_t feature;        // split feature id: column of the feature-major bin copy
  int32_t split_bin;      // rows with bin <= split_bin go left
  int32_t default_left;   // direction of the missing sentinel (only if feature has missing)
  int32_t has_missing;
  int32_t chunk_begin;    // prefix of ceil(seg_count / PART_CHUNK)
  int32_t is_cat;         // categorical split: rows whose bin (= category code) has its bit set go RIGHT
  uint32_t cat_bits[8];   // bit (b & 31) of word b >> 5
};

// candidate split written by the evaluation kernel, one per (node, group)
struct B2SplitCand {
  float loss_chg;
  int32_t feature;       // global feature id, -1 = none
  int32_t bin;           // split bin (rows with bin <= bin go left; -1 possible for backward)
  int32_t default_left;
  int64_t left_g, left_h; // fixed-point sums of the left child
  uint32_t order;        // enumeration order key for tie-breaking
  int32_t is_cat;        // categorical candidate: bin = category for a one-hot split, -1 for a partition split
  uint32_t cat_bits[8];  // categories that go right
};

struct B2EvalNode {
  int64_t sum_g, sum_h;  // node totals (fixed point)
  int32_t hist_index;    // slot in level buffer
  float root_gain;
};

struct B2TreeNodeDev {
  int32_t left, right;
  int32_t feature;       // -1 leaf
  float cond;
  float value;
  int32_t default_left;
  int32_t cat_slot;      // -1 numeric split, else row of the model's category-set table ([slot][8] words)
  int32_t pad;
};

// ---- TreeSHAP path table (shap_kernel.cu; built on the host by engine.cu build_paths).  Every leaf of every tree is
// one path: element 0 is the bias (feature -1), then one element per DISTINCT feature on the root -> leaf path, the
// repeated splits on it merged: numeric splits into an interval, categorical splits into an intersected category set,
// missing values into one flag (missing follows the path only if every merged split sends it that way).
#define B2_SHAP_MAX_PATH 16            // bias + at most 14 distinct features (max_depth <= 14) + slack
#define B2_PATH_MISSING_OK 1u          // a missing value follows the path
#define B2_PATH_HAS_HI 2u              // numeric: x < hi is required
#define B2_PATH_OUTSIDE_OK 4u          // categorical: a value outside [0, 256) follows the path
struct B2PathElem {
  int32_t feature;        // -1 = bias element
  int32_t cat_slot;       // -1 numeric, else row of the path category table ([slot][8] words, categories allowed)
  float lo, hi;           // numeric: lo <= x (lo = -inf when unbounded) and, with B2_PATH_HAS_HI, x < hi
  uint32_t flags;
  uint32_t pad;
  double zero_fraction;   // prod cover(child) / cover(parent) over the merged splits; 0 when a parent has zero cover
};
struct B2PathInfo {
  int32_t elem_begin;     // first element in the element table
  int32_t len;            // elements (bias included), <= B2_SHAP_MAX_PATH
  int32_t cls;            // output group of the tree
  int32_t pad;
  double value;           // leaf value
};

// One step of the A.9 traversal on raw floats, shared by every kernel that walks a tree (predict_kernel,
// shap_kernel.cu leaf_index_kernel): x < cond -> left, missing -> default.  Categorical node (cat_slot >= 0;
// common/categorical.h Decision): category in the node's set -> right; not in the set, negative or beyond the set -> left.
__device__ __forceinline__ int b2_tree_step(const B2TreeNodeDev& nd, float v, float missing, int missing_is_nan,
                                            const uint32_t* __restrict__ cat_table) {
  const bool miss = isnan(v) || (!missing_is_nan && v == missing);
  if (miss) return nd.default_left ? nd.left : nd.right;
  if (nd.cat_slot >= 0) {
    bool in_set = false;
    if (v >= 0.0f && v < 256.0f) { const int c = (int)v; in_set = (cat_table[(size_t)nd.cat_slot * 8 + (c >> 5)] >> (c & 31)) & 1u; }
    return in_set ? nd.right : nd.left;
  }
  return v < nd.cond ? nd.left : nd.right;
}

// node id of the leaf row x reaches in the tree whose nodes start at tn
__device__ __forceinline__ int b2_tree_leaf(const B2TreeNodeDev* __restrict__ tn, const float* __restrict__ x, float missing,
                                            int missing_is_nan, const uint32_t* __restrict__ cat_table, float* leaf_value) {
  int nid = 0;
  B2TreeNodeDev nd = tn[0];
  while (nd.feature >= 0) {
    nid = b2_tree_step(nd, x[nd.feature], missing, missing_is_nan, cat_table);
    nd = tn[nid];
  }
  *leaf_value = nd.value;
  return nid;
}

// ---- device-resident control tables of the sync-free level loop (control_kernel.cu)
struct B2LevelCtl {
  int32_t n_nodes;            // nodes of this level (to evaluate / decide)
  int32_t n_split;            // nodes that expand (filled by decide)
  int32_t part_chunks;        // partition work items of this level
  int32_t hist_n_work;        // histogram build list of THIS level (filled by the previous finalize)
  int32_t hist_total_chunks;
  int32_t hist_chunk_rows;
  int32_t n_pairs;            // (parent, built, sibling) triples of this level
  int32_t leaf_base_next;     // number of leaves after this level's decide = leaf index of the next level's first node
};
struct B2NodeSeg { int32_t nid, begin, count, buf; };
struct B2LeafDev { int32_t nid, buf, begin, count; };
struct B2SegWork {  // generic chunked (segment, id) descriptor
  int32_t seg_begin, seg_count, id, chunk_begin;
  int32_t buf, pad0, pad1, pad2;
};
struct B2TreeDev {            // arrays of capacity max_nodes
  int32_t *left, *right, *parent, *feature, *split_bin, *default_left, *split_type;
  uint32_t* cat_bits;         // [max_nodes][8], written only for categorical splits
  float* loss_chg;
  long long *sum_g, *sum_h;   // fixed-point node totals
  float *leaf_weight, *leaf_value;
  int32_t* n_nodes;
};
struct B2CtlParams { double mcw, lambda, alpha, max_delta_step; float gamma, eta; };

// column sampling of one level (sampling.cuh): level_mask = features of the level's set (nullptr = all);
// bynode < 1 makes every node draw its own subset of that set on the device
struct B2ColSample {
  const uint8_t* level_mask;
  const uint32_t* fwq;      // feature weights in Q16 (nullptr = all 1.0)
  double bynode;
  int32_t n_level;          // features in the level's set
  int32_t n_features;
  uint32_t seed, tree;
};

// what the last CTA of a level's partition does once every row is placed (level_finalize.cuh)
struct B2FinalizeArgs {
  B2LevelCtl* ctl_nxt;
  B2NodeSeg* seg_nxt;
  B2EvalNode* ev_nxt;
  const int32_t* pair_parent_hist;
  B2HistWork* hist_work;
  int32_t* triples;
  long long* stat_rows;
  uint32_t* done;               // CTAs of the partition that finished; the last one resets it to 0
  int32_t max_pairs, need_hist, n_streams, window_rows, chunk_rows_override;
};

// sibling = parent - built inside the split scan (split_kernel.cu eval_splits_kernel), instead of a separate pass
struct B2SiblingSub {
  const long long* parent_level;   // nullptr: every node's slot already holds its histogram
  const int32_t* triples;          // [pair][3]: parent slot (previous level), built slot, sibling slot
  long long* sib_out;              // nullable: store the siblings here (the level buffer) for the next level's parents
  int32_t sib_base;                // first sibling slot of the level
};

// what decide does at the end of a level's split scan (decide.cuh): run by decide_kernel, or by the last CTA of
// eval_splits_kernel on one GPU
struct B2DecideArgs {
  B2LevelCtl* ctl_cur;
  B2LevelCtl* ctl_nxt;
  const B2NodeSeg* seg_cur;
  B2NodeSeg* seg_nxt;
  const B2EvalNode* ev_cur;
  B2EvalNode* ev_nxt;
  const B2SplitCand* cands;        // [cand_ranks][cand_rank_stride]: cands_per_node candidates per node
  B2SplitCand* cand_best;          // [nodes] the winner of every node (scratch)
  const B2SplitCand* local_cands;  // peer-memory exchange: this rank's own candidates
  B2TreeDev tree;
  B2SplitWork* split_work;
  int32_t* pair_parent_hist;
  B2LeafDev* leaves;
  int32_t* n_leaves;
  const uint8_t* has_missing;
  const int32_t* qexp;
  int32_t* part_counters;          // nullable: zeroed for the level's partition
  B2CtlParams p;
  int32_t cands_per_node, cand_ranks, cand_rank_stride, can_split, qbits;
};

// ---- peer-memory exchange over NVLink / NVSwitch (p2p.cuh, p2p_exchange.cu, control_kernel.cu)
// Every rank maps four regions of every peer (cudaIpc): the histogram build buffer (peers READ their owned slices out
// of it), and three tables the peers WRITE into -- split candidates, per-tree |g|,|h| maxima + leaf sums, and epoch
// flags.  An exchange "slot" is a lock-step sequence of epochs: all ranks run the same kernel sequence, so the n-th
// exchange of a slot is epoch n on every rank.  The epoch counters live in device memory and are advanced by the
// kernels themselves, which keeps the whole tree capturable in a CUDA graph.
#define B2_P2P_MAX_WORLD 8
enum { kSlotHist = 0, kSlotCand = 1, kSlotAbsmax = 2, kSlotLeaf = 3, kSlotClose = 4, kP2PSlots = 5 };
struct B2P2P {
  long long* build[B2_P2P_MAX_WORLD];      // hist_build of rank w ([shards][node_cap][slice]); own pointer for w == rank
  B2SplitCand* cands[B2_P2P_MAX_WORLD];    // candidate table of rank w ([world][cand_cap])
  long long* misc[B2_P2P_MAX_WORLD];       // misc table of rank w ([world][misc_stride] int64: [0]=absmax bits, [2..]=leaf sum limbs)
  uint32_t* flags[B2_P2P_MAX_WORLD];       // flag array of rank w ([kP2PSlots][world])
  uint32_t* epoch;                         // [kP2PSlots] local: last completed epoch of each slot
  uint32_t* done;                          // [kP2PSlots] local: CTA completion counters of multi-CTA exchange kernels
  uint32_t* err;                           // local: != 0 after a timed-out / aborted wait (1 + slot)
  const uint32_t* abort_flag;              // local: set by B2_CommAbort through a side stream
  int32_t world, rank;
  int32_t cand_cap, misc_stride;
  long long spin_limit;                    // polls (each ~0.25 us) before a wait gives up
};

struct B2TrainParamDev {
  double min_child_weight, lambda, alpha;
  double inv_scale_g, inv_scale_h;
  double max_delta_step;   // 0 = off (CalcWeight clips to +-max_delta_step, CalcGain uses the clipped weight)
  int32_t max_cat_to_onehot, max_cat_threshold;
};

// ---- CalcWeight / CalcGain / CalcGainGivenWeight (xgboost src/tree/param.h; SURVEY.md A.6, A.7) with explicit
// IEEE round-to-nearest operations: the kernels, the host code and the CPU oracle evaluate the same sequence.
#ifdef __CUDACC__
__device__ __forceinline__ double b2_thr_l1(double g, double a) {
  if (g > a) return __dadd_rn(g, -a);
  if (g < -a) return __dadd_rn(g, a);
  return 0.0;
}
__device__ __forceinline__ double b2_calc_weight(double G, double H, double mcw, double lambda, double alpha, double mds) {
  if (H < mcw || H <= 0.0) return 0.0;
  const double t = (alpha == 0.0) ? G : b2_thr_l1(G, alpha);
  double dw = __ddiv_rn(-t, __dadd_rn(H, lambda));
  if (mds != 0.0 && fabs(dw) > mds) dw = copysign(mds, dw);
  return dw;
}
__device__ __forceinline__ double b2_calc_gain(double G, double H, double mcw, double lambda, double alpha, double mds) {
  if (H < mcw || H <= 0.0) return 0.0;
  if (mds == 0.0) {
    const double t = (alpha == 0.0) ? G : b2_thr_l1(G, alpha);
    return __ddiv_rn(__dmul_rn(t, t), __dadd_rn(H, lambda));
  }
  const double w = b2_calc_weight(G, H, mcw, lambda, alpha, mds);
  const double ret = -__dadd_rn(__dmul_rn(__dmul_rn(2.0, G), w), __dmul_rn(__dadd_rn(H, lambda), __dmul_rn(w, w)));
  return alpha == 0.0 ? ret : __dadd_rn(ret, __dmul_rn(alpha, fabs(w)));
}
#endif
