// tree.cu -- growing one tree on the GPU: the level loop of scalar and vector-leaf trees, their buffers and control
// tables, the NVLink peer-memory exchange set-up, the CUDA graphs of a tree's launches, and turning a finished tree's
// read-back block into a TreeHost.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <chrono>
#include <tuple>

#include "host.h"
#include "launch.h"
#include "sampling.cuh"

namespace b2host __attribute__((visibility("hidden"))) {

int window_rows_for(int qbits) {
  // overflow-guard interval of the histogram kernel: |q| <= 2^qbits, so 2^(30-qbits) rows add less than 2^30
  // to a cell that was below 2^30 at the last check (hist_kernel.cu flush_large_cells)
  return 1 << (30 - qbits);
}

// the root's chunk size; the other levels pick theirs in finalize_level_block (level_finalize.cuh), by the same rule
int pick_chunk_rows(Booster* b, int64_t rows) {
  int c = b->p.hist_chunk_rows;
  if (c <= 0) {
    const int n_streams = std::max(1, b->ctx->num_sms * 3 / b->train->n_groups);
    const int64_t per_stream = rows / n_streams;
    int64_t target = per_stream >= 16384 ? per_stream / 4 : per_stream;
    c = 512;
    while (c < target && c < 8192) c <<= 1;
  }
  const int w = window_rows_for(b->p.qbits);
  if (c > w) c = w;   // one chunk = one int32 window
  return c;
}

// layout of the per-tree read-back block (device t_* buffers are copied verbatim into one pinned block)
struct TreeLayout {
  size_t max_nodes, i32_count, f32_count, i64_count, bytes;
  size_t off_f32, off_i64, off_qexp, off_cat;
};
TreeLayout tree_layout(int max_depth) {
  TreeLayout L;
  L.max_nodes = ((size_t)1 << (max_depth + 1));
  L.i32_count = 7 * L.max_nodes + 2;
  L.f32_count = 3 * L.max_nodes;
  L.i64_count = 2 * L.max_nodes + (size_t)max_depth + 2;
  L.off_f32 = L.i32_count * 4;
  L.off_i64 = (L.off_f32 + L.f32_count * 4 + 7) & ~(size_t)7;
  L.off_qexp = L.off_i64 + L.i64_count * 8;
  L.off_cat = L.off_qexp + 16;
  L.bytes = L.off_cat + L.max_nodes * 8 * sizeof(uint32_t);
  return L;
}
B2TreeDev tree_dev(Booster* b) {
  const TreeLayout L = tree_layout(b->ctl_depth);
  B2TreeDev t;
  int32_t* i = b->t_i32.p; const size_t m = L.max_nodes;
  t.left = i; t.right = i + m; t.parent = i + 2 * m; t.feature = i + 3 * m; t.split_bin = i + 4 * m; t.default_left = i + 5 * m;
  t.split_type = i + 6 * m;
  t.n_nodes = i + 7 * m;
  t.cat_bits = b->t_cat.p;
  t.loss_chg = b->t_f32.p; t.leaf_weight = b->t_f32.p + m; t.leaf_value = b->t_f32.p + 2 * m;
  t.sum_g = b->t_i64.p; t.sum_h = b->t_i64.p + m;
  return t;
}

// Map every peer's build buffer, candidate table, misc table and flag array (cudaIpc) for the peer-memory exchange.
// All ranks take the same decision: one failed mapping anywhere leaves every rank on NCCL.
int p2p_timeout_seconds() {
  const char* e = getenv("B2_P2P_TIMEOUT_S");
  int v = e ? atoi(e) : 60;
  return v < 1 ? 1 : v;
}
void p2p_setup(Booster* b) {
  Booster::P2PState& st = b->p2p;
  if (st.tried || b->shards <= 1) return;
  st.tried = true;
  const char* env = getenv("B2_EXCHANGE");
  if (env && (strcmp(env, "nccl") == 0 || strcmp(env, "NCCL") == 0)) return;
  Comm* c = b->comm; cudaStream_t s = b->ctx->stream; const int W = c->world;
  if (W > B2_P2P_MAX_WORLD) return;
  const size_t misc_stride = b->x_misc_stride;
  const size_t n_flags = (size_t)b2_p2p_flag_words(W), n_words = 2 * (size_t)kP2PSlots + 2;
  st.words.ensure(n_words);
  CUDA_CHECK(cudaMemsetAsync(st.flags, 0, n_flags * sizeof(uint32_t), s));
  CUDA_CHECK(cudaMemsetAsync(st.words.p, 0, n_words * sizeof(uint32_t), s));
  CUDA_CHECK(cudaMemsetAsync(st.misc, 0, (size_t)W * misc_stride * sizeof(long long), s));
  cudaIpcMemHandle_t mine; int ok = 1;
  if (cudaIpcGetMemHandle(&mine, b->xarena.p) != cudaSuccess) { ok = 0; cudaGetLastError(); memset(&mine, 0, sizeof(mine)); }
  DevBuf<uint8_t> d_mine, d_all; d_mine.ensure(sizeof(mine)); d_all.ensure(sizeof(mine) * (size_t)W);
  CUDA_CHECK(cudaMemcpyAsync(d_mine.p, &mine, sizeof(mine), cudaMemcpyHostToDevice, s));
  NCCL_CHECK(nccl()->AllGather(d_mine.p, d_all.p, sizeof(mine), kNcclUint8, c->comm, s));   // also orders the memsets before any peer store
  std::vector<cudaIpcMemHandle_t> all((size_t)W);
  CUDA_CHECK(cudaMemcpyAsync(all.data(), d_all.p, sizeof(mine) * (size_t)W, cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  memset(&st.pp, 0, sizeof(st.pp));
  st.pp.world = W; st.pp.rank = c->rank; st.pp.cand_cap = st.cand_cap; st.pp.misc_stride = (int32_t)misc_stride;
  st.pp.epoch = st.words.p; st.pp.done = st.words.p + kP2PSlots; st.pp.err = st.words.p + 2 * kP2PSlots;
  st.pp.abort_flag = c->d_abort ? c->d_abort : st.words.p + 2 * kP2PSlots + 1;
  st.pp.spin_limit = (long long)p2p_timeout_seconds() * 1000000LL;
  for (int w = 0; w < W && ok; ++w) {
    uint8_t* base = b->xarena.p;
    if (w != c->rank) {
      void* q = nullptr;
      if (cudaIpcOpenMemHandle(&q, all[w], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { ok = 0; cudaGetLastError(); break; }
      st.opened.push_back(q);
      base = (uint8_t*)q;
    }
    st.pp.build[w] = (long long*)base; st.pp.cands[w] = (B2SplitCand*)(base + b->xoff_cands);
    st.pp.misc[w] = (long long*)(base + b->xoff_misc); st.pp.flags[w] = (uint32_t*)(base + b->xoff_flags);
  }
  // agree: max over ranks of "failed"
  DevBuf<int32_t> d_ok; d_ok.ensure(1);
  int32_t neg = ok ? 0 : 1;
  CUDA_CHECK(cudaMemcpyAsync(d_ok.p, &neg, sizeof(neg), cudaMemcpyHostToDevice, s));
  allreduce(c, d_ok.p, 1, kNcclInt32, kNcclMax, s);
  CUDA_CHECK(cudaMemcpyAsync(&neg, d_ok.p, sizeof(neg), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  if (neg) {
    for (void* q : st.opened) cudaIpcCloseMemHandle(q);
    st.opened.clear();
    if (getenv("B2_EXCHANGE")) fprintf(stderr, "[b2hist] peer mapping failed on some rank; histogram exchange stays on NCCL\n");
    return;
  }
  st.enabled = true;
}

// feature-slot sharding of the histogram exchange: rank r owns slots s with s % shards == r (DESIGN.md 5)
// (vector-leaf trees: every rank scans every slot of the allreduced T-target level buffer, no sharding)
int hist_shards(const Booster* b) {
  const int world = b->comm ? b->comm->world : 1;
  return (world > 1 && world <= 32 && (32 % world) == 0 && !b->p.vector_leaf()) ? world : 1;
}

// The two level buffers hold 2^(D-1) nodes x n_groups x 128 KiB split over the shards, and a sharded exchange adds a
// build buffer of 2^(D-1) nodes x n_groups x 128 KiB: 8 GiB at max_depth 16 with one feature group, far more for a
// wide matrix.  A booster whose buffers do not fit in the device memory free now (the pool's cached blocks count as
// free) is refused when it is created, before anything is allocated for it, rather than failing in cudaMalloc partway
// through its first tree.  Vector-leaf trees have their own check (prepare_tree_buffers); update mode grows nothing.
void check_level_memory(const Booster* b) {
  if (b->p.vector_leaf() || b->p.update_mode) return;
  const int D = b->p.max_depth, G = b->train->n_groups, shards = hist_shards(b);
  const double half = (double)((size_t)1 << (D - 1)), node_bytes = (double)G * B2_GROUP_ELEMS * sizeof(long long);
  const double need = 2.0 * half * node_bytes / shards + (shards > 1 ? half * node_bytes : 0.0);
  size_t free_bytes = 0, total_bytes = 0;
  CUDA_CHECK(cudaMemGetInfo(&free_bytes, &total_bytes));
  int dev = 0; CUDA_CHECK(cudaGetDevice(&dev));
  size_t cached = 0;
  if (dev >= 0 && dev < 64) { std::lock_guard<std::mutex> lk(g_dev_pool[dev].mu); cached = g_dev_pool[dev].cached; }
  const double avail = (double)free_bytes + (double)cached;
  if (need > avail)
    fail("max_depth %d with %d feature groups needs %.1f GiB of level histograms, and %.1f GiB of device memory is free; "
         "use a smaller max_depth or fewer features", D, G, need / (double)(1ull << 30), avail / (double)(1ull << 30));
}

void ensure_ctl_tables(Booster* b) {
  const int D = b->p.max_depth; const int G = b->train->n_groups;
  if (b->ctl_depth == D) return;
  if (b->ctl_depth != 0 && b->p2p.enabled) fail("max_depth cannot change while the peer-memory exchange is mapped");
  for (auto& r : b->rb) {   // captured launch sequences hold the old table addresses
    for (auto& kv : r.graphs) Booster::destroy_graph(kv.second);
    r.graphs.clear();
  }
  b->direct_trees.clear();
  b->ctl_depth = D;
  const TreeLayout L = tree_layout(D);
  const size_t lcap = (size_t)1 << D, half = (size_t)1 << (D > 0 ? D - 1 : 0);
  b->t_block.ensure(L.bytes);
  b->t_i32.p = (int32_t*)b->t_block.p; b->t_f32.p = (float*)(b->t_block.p + L.off_f32);
  b->t_i64.p = (long long*)(b->t_block.p + L.off_i64); b->t_qexp.p = (int32_t*)(b->t_block.p + L.off_qexp);
  b->t_cat.p = (uint32_t*)(b->t_block.p + L.off_cat);
  b->d_ctl.ensure(3);
  for (int k = 0; k < 2; ++k) { b->d_seg[k].ensure(lcap); b->d_ev[k].ensure(lcap); }
  b->d_hist_work.ensure(half); b->d_split_work.ensure(half);
  b->d_counters.ensure(2 * half); b->d_triples.ensure(3 * half); b->d_pair_parent.ensure(half);
  if (!b->d_part_done.p) { b->d_part_done.ensure(1); CUDA_CHECK(cudaMemsetAsync(b->d_part_done.p, 0, sizeof(uint32_t), b->ctx->stream)); }
  if (!b->d_eval_done.p) { b->d_eval_done.ensure(1); CUDA_CHECK(cudaMemsetAsync(b->d_eval_done.p, 0, sizeof(uint32_t), b->ctx->stream)); }
  b->d_cand_best.ensure(half);
  b->hist_scratch.ensure(b2_hist_scratch_elems(bin_source(b->train), (int)half));
  b->d_leaves.ensure(L.max_nodes); b->d_seg_work.ensure(L.max_nodes);
  b->d_leaf_sums.ensure(4 * lcap); b->d_leaf_values.ensure(lcap);   // [leaf][g, h][hi, lo] limbs (common.cuh)
  if (b->ic_words > 0) b->d_ic_compat.ensure(L.max_nodes * (size_t)b->ic_words);
  b->node_elems = (size_t)G * B2_GROUP_ELEMS;
  b->shards = hist_shards(b);
  b->log2_shards = 0; while ((1 << b->log2_shards) < b->shards) b->log2_shards++;
  b->sp = B2_GROUP_SLOTS / b->shards;
  b->slice_elems = (size_t)G * 2 * B2_BINS * b->sp;
  b->cpn_num = b2_eval_ctas_per_node(G, b->log2_shards, 1);   // the most numeric candidates per node of any level
  b->cpn = b->cpn_num + (b->train->any_cat() ? b2_cat_ctas() : 0);
  if (!b->p.vector_leaf()) { b->hist[0].ensure(half * b->slice_elems); b->hist[1].ensure(half * b->slice_elems); }   // vector trees: d_vhist
  if (b->shards > 1) {
    auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
    const size_t build_bytes = up(half * b->node_elems * sizeof(long long));
    const size_t cands_bytes = up(half * b->cpn * b->shards * sizeof(B2SplitCand));
    b->x_misc_stride = 2 + 4 * lcap;                                   // even: 16-byte aligned regions
    const size_t misc_bytes = up((size_t)b->shards * b->x_misc_stride * sizeof(long long));
    const size_t flag_bytes = up((size_t)b2_p2p_flag_words(b->shards) * sizeof(uint32_t));
    b->xoff_cands = build_bytes; b->xoff_misc = b->xoff_cands + cands_bytes; b->xoff_flags = b->xoff_misc + misc_bytes;
    b->xarena.ensure(b->xoff_flags + flag_bytes);
    b->hist_build.p = (long long*)b->xarena.p;
    b->d_cands_all.p = (B2SplitCand*)(b->xarena.p + b->xoff_cands);
    b->p2p.misc = (long long*)(b->xarena.p + b->xoff_misc);
    b->p2p.flags = (uint32_t*)(b->xarena.p + b->xoff_flags);
  }
  b->d_cands.ensure(half * b->cpn);
  CUDA_CHECK(cudaMemsetAsync(b->t_i64.p, 0, L.i64_count * 8, b->ctx->stream));
  b->p2p.cand_cap = (int)(half * b->cpn);
  p2p_setup(b);
}

// Launch bookkeeping of one tree: with direct launches it is applied right away, a captured tree keeps it with its
// graph and applies it on every replay.
struct TreeStats {
  long long hist_launches = 0, kernel_launches = 0;
  double allreduce_bytes = 0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> hist_ev;
  bool capturing = false;
};
void record_hist_launch(Booster* b, TreeStats& st, cudaEvent_t& e0, cudaEvent_t& e1, bool begin) {
  if (!b->p.profile) return;
  cudaStream_t s = b->ctx->stream;
  if (begin) {
    if (st.capturing) { CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1)); }   // owned by the graph
    else { e0 = get_event(b); e1 = get_event(b); }
    // inside a capture the record becomes an event-record node that every replay executes (external event)
    CUDA_CHECK(cudaEventRecordWithFlags(e0, s, st.capturing ? cudaEventRecordExternal : cudaEventRecordDefault));
  } else {
    CUDA_CHECK(cudaEventRecordWithFlags(e1, s, st.capturing ? cudaEventRecordExternal : cudaEventRecordDefault));
    st.hist_ev.push_back({e0, e1});
  }
}

bool env_flag(const char* name, bool dflt) {
  const char* e = getenv(name);
  return e ? atoi(e) != 0 : dflt;
}

// Where the histogram kernel of a level accumulates: the reduce-scatter / peer-read build buffer when the exchange
// is sharded by feature slot (shards == world), else the level buffer itself (single GPU, or in-place allreduce).
long long* build_target(Booster* b, long long* level_buf) { return b->shards > 1 ? b->hist_build.p : level_buf; }

// Histogram exchange of the nodes built for one level + sibling subtraction (parent - built).
//   peer memory : ONE kernel reads the W partial slices out of the peers' build buffers, stores built and sibling
//   NCCL        : reduce-scatter (shards == world) or in-place allreduce, then hist_subtract_kernel
// `triples` == nullptr: the root (nothing to subtract).
void exchange_and_subtract(Booster* b, TreeStats& st, const long long* parent_level, long long* level_buf, const int32_t* triples,
                           const B2LevelCtl* ctl_nxt, int nb, int node_cap) {
  cudaStream_t s = b->ctx->stream;
  const bool multi = b->comm && b->comm->world > 1;
  if (multi && b->comm->aborted.load()) fail("communicator aborted");
  if (multi && b->p2p.enabled) {
    LAUNCH_CHECK(b2_launch_p2p_reduce_subtract(&b->p2p.pp, parent_level, level_buf, triples, ctl_nxt, nb, node_cap,
                                               (int64_t)b->slice_elems, b->ctx->num_sms, s));
    st.allreduce_bytes += (double)nb * b->node_elems * 8 * (b->shards - 1) / b->shards;
    st.kernel_launches++;
    mark_phase(b, 2);
    return;
  }
  if (multi && b->shards > 1) {
    NCCL_CHECK(nccl()->ReduceScatter(b->hist_build.p, level_buf, (size_t)nb * b->slice_elems, kNcclInt64, kNcclSum, b->comm->comm, s));
    st.allreduce_bytes += (double)nb * b->node_elems * 8 * (b->shards - 1) / b->shards;
  } else if (multi) {
    NCCL_CHECK(nccl()->AllReduce(level_buf, level_buf, (size_t)nb * b->node_elems, kNcclInt64, kNcclSum, b->comm->comm, s));
    st.allreduce_bytes += (double)nb * b->node_elems * 8;
  }
  mark_phase(b, 2);
  if (triples) {
    LAUNCH_CHECK(b2_launch_hist_subtract(parent_level, level_buf, triples, nb, (int64_t)b->slice_elems, ctl_nxt, s));
    st.kernel_launches++;
  }
  mark_phase(b, 3);
}

// reg:quantileerror buffers for up to max_leaves segments, allocated outside any capture; the histograms start zeroed
// and every scan zeroes what it read
void ensure_quantile_buffers(Booster* b, int max_leaves) {
  cudaStream_t s = b->ctx->stream;
  const size_t elems = b2_quantile_hist_elems(max_leaves);
  if (b->d_qhist.cap < elems) {
    b->d_qhist.ensure(elems);
    CUDA_CHECK(cudaMemsetAsync(b->d_qhist.p, 0, elems * sizeof(unsigned long long), s));
  }
  b->d_qsel.ensure(b2_quantile_sel_bytes(max_leaves));
  if (!b->d_one.p) {
    const int32_t one = 1;
    b->d_one.ensure(1);
    CUDA_CHECK(cudaMemcpyAsync(b->d_one.p, &one, sizeof(one), cudaMemcpyHostToDevice, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
  }
  if (b->d_alpha.cap < b->p.quantile_alpha.size()) {
    upload(b->d_alpha, b->p.quantile_alpha, s);
    CUDA_CHECK(cudaStreamSynchronize(s));
  }
}

// The alpha_k-quantile of the residuals y - margin[:, k] (margin nullable: 0) of the rows with a nonzero hessian in each
// of the *n_leaves segments given by pos (nullable: one segment), exact over all ranks (quantile_kernel.cu).  Writes
// fp32(q * eta) to leaf_value[leaf] and, with leaves, to tree_value[leaves[leaf].nid]; an empty segment is left as it is.
// qexp[1] is the exponent of the largest hessian of all ranks (the weights' fixed-point scale).
int quantile_select(Booster* b, int k, const uint16_t* pos, const float* margin, const float2* gh, const int32_t* qexp,
                    const int32_t* n_leaves, int max_leaves, float eta, const B2LeafDev* leaves, float* leaf_value,
                    float* tree_value) {
  Matrix* m = b->train; cudaStream_t s = b->ctx->stream; const int K = b->p.num_class;
  const int weighted = m->n_weight > 0 ? 1 : 0;
  const size_t elems = b2_quantile_hist_elems(max_leaves) / (weighted ? 1 : 2);
  for (int pass = 0; pass < b2_quantile_passes(); ++pass) {
    LAUNCH_CHECK(b2_launch_quantile_count(pass, pos, m->label.p, margin, K, k, gh, m->n, qexp, weighted, b->d_qsel.p,
                                          max_leaves, b->d_qhist.p, b->ctx->num_sms, s));
    allreduce(b->comm, b->d_qhist.p, elems, kNcclUint64, kNcclSum, s);   // digit counts of all ranks: exact
    LAUNCH_CHECK(b2_launch_quantile_scan(pass, n_leaves, max_leaves, weighted, b->p.quantile_alpha[k], eta, b->d_qhist.p,
                                         b->d_qsel.p, leaves, leaf_value, tree_value, s));
  }
  return 2 * b2_quantile_passes();
}

B2TrainParamDev train_params(const Params& p) {
  B2TrainParamDev dp;
  dp.min_child_weight = (double)p.min_child_weight; dp.lambda = (double)p.lambda; dp.alpha = (double)p.alpha;
  dp.inv_scale_g = dp.inv_scale_h = 1.0;
  dp.max_cat_to_onehot = p.max_cat_to_onehot; dp.max_cat_threshold = p.max_cat_threshold;
  dp.max_delta_step = (double)p.max_delta_step;
  return dp;
}

// the leaf values of the num_parallel_tree trees grown from the same gradients are scaled by eta / num_parallel_tree
B2CtlParams ctl_params(const Params& p) {
  B2CtlParams cp;
  cp.mcw = (double)p.min_child_weight; cp.lambda = (double)p.lambda; cp.alpha = (double)p.alpha;
  cp.max_delta_step = (double)p.max_delta_step; cp.gamma = p.gamma; cp.eta = p.eta / (float)p.num_parallel_tree;
  return cp;
}

// B2_BoosterSetParam changed b->p from old: the tree graphs of both round-buffer sets are stale when a value that
// train_params or ctl_params pass to the kernels by value changed (run_tree captures them again on their next use)
void tree_params_changed(Booster* b, const Params& old) {
  const Params& p = b->p;
  if (std::tie(p.eta, p.gamma, p.min_child_weight, p.lambda, p.alpha, p.max_delta_step, p.max_cat_to_onehot,
               p.max_cat_threshold) ==
      std::tie(old.eta, old.gamma, old.min_child_weight, old.lambda, old.alpha, old.max_delta_step,
               old.max_cat_to_onehot, old.max_cat_threshold))
    return;
  for (auto& r : b->rb)
    for (auto& kv : r.graphs) kv.second.stale = true;
}

// Column sampling of one tree: the tree's feature set and one nested set per level are drawn on the host (they depend
// on (seed, tree, level) only, never on the data) into d_col_masks, the per-node subsets inside the split-scan kernels.
// Returns the number of features of every level's set.
std::vector<int> draw_column_masks(Booster* b, uint32_t tree_index) {
  Matrix* m = b->train; const Params& p = b->p; const int D = p.max_depth, F = m->F;
  std::vector<int> n_level_feats(D, F);
  if (!p.use_cols()) return n_level_feats;
  const uint32_t* fwq = m->fwq.empty() ? nullptr : m->fwq.data();
  std::vector<uint8_t> mask_tree(F), masks((size_t)D * F);
  std::vector<B2ColRank> col_scratch(F);
  const int n_tree = b2_col_select((uint32_t)p.seed, tree_index, B2_SCOPE_TREE, nullptr, fwq, F,
                                   b2_sample_count((double)p.colsample_bytree, F), col_scratch.data(), mask_tree.data());
  for (int d = 0; d < D; ++d)
    n_level_feats[d] = b2_col_select((uint32_t)p.seed, tree_index, B2_SCOPE_LEVEL(d), mask_tree.data(), fwq, F,
                                     b2_sample_count((double)p.colsample_bylevel, n_tree), col_scratch.data(),
                                     masks.data() + (size_t)d * F);
  b->d_col_masks.ensure(masks.size());
  CUDA_CHECK(cudaMemcpyAsync(b->d_col_masks.p, masks.data(), masks.size(), cudaMemcpyHostToDevice, b->ctx->stream));   // pageable source: staged before return
  return n_level_feats;
}

// Fixed-point quantisation of the gradients of targets k0 .. k0 + nt - 1 for one tree, with a global scale per target
// (the |g|, |h| maxima over the ranks): the target's exponents go to d_qexp[j] and its quantised pairs to q[j] (j: the
// target's place in the tree).  Row subsampling zeroes the same rows in every target: the draw depends on
// (seed, tree, rank, row) only.
void quantise_gradients(Booster* b, TreeStats& st, int k0, int nt, uint32_t tree_index) {
  const Params& p = b->p; cudaStream_t s = b->ctx->stream; const int64_t n = b->train->n; const int sms = b->ctx->num_sms;
  const bool p2p = b->comm && b->comm->world > 1 && b->p2p.enabled;
  uint32_t* absmax = b->d_absmax.p + 2 * k0;
  for (int j = 0; j < nt; ++j) {
    float2* gh = b->gh.p + (size_t)(k0 + j) * n;
    if (p.subsample < 1.0f) {
      LAUNCH_CHECK(b2_launch_subsample(gh, n, (uint32_t)p.seed, tree_index, b->comm ? (uint32_t)b->comm->rank : 0u,
                                       (double)p.subsample, sms, s));
      st.kernel_launches++;
    }
    if (!b->absmax_fused) {   // custom objective / row sampling / many classes: |g|,|h| maxima in their own pass
      CUDA_CHECK(cudaMemsetAsync(absmax + 2 * j, 0, 2 * sizeof(uint32_t), s));
      LAUNCH_CHECK(b2_launch_absmax(gh, n, absmax + 2 * j, sms, s));
      st.kernel_launches++;
    }
  }
  if (!p2p) allreduce(b->comm, absmax, 2 * (size_t)nt, kNcclUint32, kNcclMax, s);
  for (int j = 0; j < nt; ++j) {
    int32_t* qexp = b->d_qexp.p + 2 * j;
    if (p2p) LAUNCH_CHECK(b2_launch_p2p_quant_exponent(&b->p2p.pp, absmax + 2 * j, qexp, s));
    else LAUNCH_CHECK(b2_launch_quant_exponent(absmax + 2 * j, qexp, s));
    LAUNCH_CHECK(b2_launch_quantize(b->gh.p + (size_t)(k0 + j) * n, n, qexp, p.qbits, b->q.p + (size_t)j * n, sms, s));
    st.kernel_launches += 2;
  }
}

// One histogram build into tgt from the quantised pairs q: the root (ridx == nullptr: every row, in chunks sized on the
// host; a rank without rows launches nothing) or the `nodes` nodes of ctl's work list over the ordered rows ridx.
void launch_hist(Booster* b, TreeStats& st, const int2* q, const int32_t* ridx, const B2LevelCtl* ctl, int nodes,
                 long long* tgt) {
  Matrix* m = b->train; const int64_t n = m->n;
  int root = 0, chunks = 0, chunk_rows = 0;
  if (!ridx) {
    if (n == 0) return;
    root = 1; chunk_rows = pick_chunk_rows(b, n); chunks = (int)((n + chunk_rows - 1) / chunk_rows);
  }
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  record_hist_launch(b, st, e0, e1, true);
  LAUNCH_CHECK(b2_launch_hist(bin_source(m), m->d_group_size.p, q, ridx, b->d_hist_work.p, root, chunks, chunk_rows,
                              window_rows_for(b->p.qbits), m->n_groups, tgt, b->hist_scratch.p, ctl, b->log2_shards, nodes,
                              b->ctx->num_sms, b->ctx->stream));
  record_hist_launch(b, st, e0, e1, false);
  st.hist_launches++; st.kernel_launches++;
}

void hist_build_raw(Matrix* m, const int32_t* qg, const int32_t* qh, const int32_t* ridx, int64_t n_sel, int window_rows,
                    int chunk_rows, int64_t* out, float* kernel_ms) {
  Ctx* ctx = m->ctx; cudaStream_t s = ctx->stream; const B2BinRows src = bin_source(m);
  std::vector<int2> gp((size_t)std::max<int64_t>(m->n, 1));
  for (int64_t i = 0; i < m->n; ++i) gp[i] = make_int2(qg[i], qh[i]);
  DevBuf<int2> d_gp; DevBuf<int32_t> d_ridx; DevBuf<long long> d_hist, d_scratch; DevBuf<B2HistWork> d_work;
  upload(d_gp, gp, s);
  if (ridx) upload(d_ridx, ridx, (size_t)std::max<int64_t>(n_sel, 0), s);
  const size_t node_elems = (size_t)m->n_groups * B2_GROUP_ELEMS;
  d_hist.ensure(node_elems); d_scratch.ensure(b2_hist_scratch_elems(src, 1));
  CUDA_CHECK(cudaMemsetAsync(d_hist.p, 0, node_elems * sizeof(long long), s));
  if (window_rows <= 0) window_rows = 4096;
  if (chunk_rows <= 0) chunk_rows = 2048;
  if (chunk_rows > window_rows) chunk_rows = window_rows;
  B2HistWork w{0, (int32_t)n_sel, 0, 0};
  upload(d_work, &w, 1, s);
  const int chunks = (int)((n_sel + chunk_rows - 1) / chunk_rows);
  cudaEvent_t e0, e1; CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
  CUDA_CHECK(cudaEventRecord(e0, s));
  if (n_sel > 0)
    LAUNCH_CHECK(b2_launch_hist(src, m->d_group_size.p, d_gp.p, ridx ? d_ridx.p : nullptr, d_work.p, 1, chunks, chunk_rows,
                                window_rows, m->n_groups, d_hist.p, d_scratch.p, nullptr, 0, 1, ctx->num_sms, s));
  CUDA_CHECK(cudaEventRecord(e1, s));
  std::vector<long long> h(node_elems);
  CUDA_CHECK(cudaMemcpyAsync(h.data(), d_hist.p, node_elems * sizeof(long long), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  if (kernel_ms) { float ms = 0; cudaEventElapsedTime(&ms, e0, e1); *kernel_ms = ms; }
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  for (int f = 0; f < m->F; ++f) {
    const int g = m->feat_byte[f] / B2_GROUP_SLOTS, sl = m->feat_byte[f] % B2_GROUP_SLOTS;
    for (int bb = 0; bb < 256; ++bb) {
      out[((size_t)f * 256 + bb) * 2] = h[(size_t)g * B2_GROUP_ELEMS + bb * 32 + sl];
      out[((size_t)f * 256 + bb) * 2 + 1] = h[(size_t)g * B2_GROUP_ELEMS + B2_PLANE_ELEMS + bb * 32 + sl];
    }
  }
}

// What decide does at the end of level d's split scan, with cpn candidates per node and rank
B2DecideArgs decide_args(Booster* b, const B2TreeDev& tree, const B2CtlParams& cp, int d, int cpn) {
  Matrix* m = b->train; B2LevelCtl* ctl = b->d_ctl.p;
  const int cur = d & 1, nxt = cur ^ 1;
  const bool can_split = d < b->p.max_depth;
  B2DecideArgs da;
  da.ctl_cur = ctl + cur; da.ctl_nxt = ctl + nxt; da.seg_cur = b->d_seg[cur].p; da.seg_nxt = b->d_seg[nxt].p;
  da.ev_cur = b->d_ev[cur].p; da.ev_nxt = b->d_ev[nxt].p;
  da.cands = b->d_cands.p; da.cand_best = b->d_cand_best.p; da.local_cands = b->d_cands.p;
  da.tree = tree; da.split_work = b->d_split_work.p; da.pair_parent_hist = b->d_pair_parent.p; da.leaves = b->d_leaves.p;
  da.n_leaves = tree.n_nodes + 1; da.has_missing = m->d_has_missing.p; da.qexp = b->d_qexp.p;
  da.part_counters = can_split ? b->d_counters.p : nullptr; da.p = cp;
  B2Interaction ic{nullptr, nullptr, 0};
  if (b->ic_words > 0) { ic.sets_of = b->d_ic_sets_of.p; ic.compat = b->d_ic_compat.p; ic.words = b->ic_words; }
  da.ic = ic;
  da.cands_per_node = cpn; da.cand_ranks = b->shards; da.cand_rank_stride = (1 << d) * cpn;
  da.can_split = can_split ? 1 : 0; da.qbits = b->p.qbits; da.vector_leaf = 0;
  return da;
}

// column sampling of level d's split scan: n_level features in the level's set, filtered per node by ic
B2ColSample col_sample(Booster* b, int d, int n_level, uint32_t tree_index, const B2Interaction& ic) {
  Matrix* m = b->train; const Params& p = b->p;
  B2ColSample cs;
  cs.level_mask = p.use_cols() ? b->d_col_masks.p + (size_t)d * m->F : nullptr;
  cs.fwq = m->fwq.empty() ? nullptr : m->d_fwq.p;
  cs.bynode = (double)p.colsample_bynode; cs.n_level = n_level; cs.n_features = m->F;
  cs.seed = (uint32_t)p.seed; cs.tree = p.use_cols() ? tree_index : 0u;
  cs.ic = ic;
  return cs;
}

// Rows of level d's nodes (the root's rows are the identity list) and the bound of its split work items
const int32_t* level_ridx(Booster* b, int d) { return d == 0 ? nullptr : b->ridx[d & 1].p; }
int split_work_items(Booster* b, int d) {
  const int64_t n = b->train->n; const int pchunk = b2_split_chunk_rows();
  return (int)((n + pchunk - 1) / pchunk) + (1 << d);   // chunks of all rows + nodes of the level: an upper bound
}

// Partition the rows of level d's expanding nodes into the other index list (decide zeroed the counters); the last CTA
// of the partition finalises the level: child segments, build-child choice, next histogram work list
void partition_level(Booster* b, TreeStats& st, int d) {
  Matrix* m = b->train; const Params& p = b->p; B2LevelCtl* ctl = b->d_ctl.p;
  const int cur = d & 1, nxt = cur ^ 1;
  B2FinalizeArgs fin;
  fin.ctl_nxt = ctl + nxt; fin.seg_nxt = b->d_seg[nxt].p; fin.ev_nxt = b->d_ev[nxt].p; fin.pair_parent_hist = b->d_pair_parent.p;
  fin.hist_work = b->d_hist_work.p; fin.triples = b->d_triples.p; fin.done = b->d_part_done.p;
  fin.stat_rows = b->t_i64.p + 2 * tree_layout(p.max_depth).max_nodes + d + 1;   // rows per level, after the node sums
  fin.max_pairs = 1 << d; fin.need_hist = d + 1 < p.max_depth ? 1 : 0;
  fin.n_streams = std::max(1, b->ctx->num_sms * 3 / m->n_groups); fin.window_rows = window_rows_for(p.qbits);
  fin.chunk_rows_override = p.hist_chunk_rows;
  LAUNCH_CHECK(b2_launch_partition(bin_source(m), level_ridx(b, d), b->ridx[nxt].p, b->d_split_work.p, ctl + cur,
                                   split_work_items(b, d), b->d_counters.p, m->any_cat() ? 1 : 0, fin, b->ctx->num_sms,
                                   b->ctx->stream));
  st.kernel_launches++;
}

// The children of the last split level d are leaves: no ordered index lists any more.  Leaves that stopped earlier get
// their rows' leaf index (pos) from their segments, rows of the nodes that split here are assigned in one pass
// (partition_kernel.cu); with sums, both also add gh (quantised by qexp) to the 40-bit fixed-point leaf sums.
void assign_leaves(Booster* b, TreeStats& st, int d, const float2* gh, const int32_t* qexp, long long* sums) {
  Matrix* m = b->train; B2LevelCtl* ctl = b->d_ctl.p; cudaStream_t s = b->ctx->stream; const int sms = b->ctx->num_sms;
  const int lchunk = b2_part_chunk_rows();
  const int max_leaf_chunks = (int)((m->n + lchunk - 1) / lchunk) + (1 << b->p.max_depth);
  LAUNCH_CHECK(b2_launch_leaf_sums(gh, b->ridx[0].p, b->ridx[1].p, b->d_seg_work.p, ctl + 2, max_leaf_chunks, qexp, 40, sums,
                                   b->pos.p, sms, s));
  LAUNCH_CHECK(b2_launch_final_assign(bin_source(m), level_ridx(b, d), b->d_split_work.p, ctl + (d & 1), split_work_items(b, d),
                                      gh, qexp, 40, sums, b->pos.p, m->any_cat() ? 1 : 0, sms, s));
  st.kernel_launches += 2;
}

// Grow one tree for class k from gh[k] (already on device); updates margin[:, k].  No host
// synchronisation: every data-dependent decision is taken by the control kernels, the host
// enqueues a fixed sequence and the finished tree is copied into pinned block `slot`.
// With st.capturing the stream is in capture mode: nothing here may allocate, touch pageable host memory or depend on
// host state that changes from tree to tree (run_tree decides when that holds).
void grow_tree(Booster* b, int k, int slot, TreeStats& st) {
  Matrix* m = b->train; Ctx* ctx = b->ctx; cudaStream_t s = ctx->stream; const Params& p = b->p;
  const int64_t n = m->n; const int K = p.num_class; const int G = m->n_groups; const int D = p.max_depth;
  const float2* gh = b->gh.p + (size_t)k * n;
  ensure_ctl_tables(b);
  const TreeLayout L = tree_layout(D);
  const bool multi = b->comm && b->comm->world > 1;
  const bool p2p = multi && b->p2p.enabled;
  // leaf sums from a streaming pass over (pos, gh) in row order; needs one shared-memory accumulator per leaf
  const bool leaf_stream = D <= b2_leaf_acc_max_depth();
  // sibling subtraction inside eval_splits_kernel (no hist_subtract pass).  The peer-memory exchange subtracts while it
  // reduces, and the categorical scan reads the sibling slots itself, so both keep the stored siblings.
  const bool sub_in_scan = !p2p && !m->any_cat();
  mark_phase(b, -1);
  // position of this tree in the model (sampling seed): the trees of a round still pending come before it
  const uint32_t tree_index = (uint32_t)b->trees.size() + (uint32_t)b->pending_trees + (uint32_t)slot;
  quantise_gradients(b, st, k, 1, tree_index);
  const std::vector<int> n_level_feats = draw_column_masks(b, tree_index);
  const B2TrainParamDev dp = train_params(p);
  const B2CtlParams cp = ctl_params(p);
  const B2TreeDev tree = tree_dev(b);
  int32_t* d_n_leaves = tree.n_nodes + 1;
  B2LevelCtl* ctl = b->d_ctl.p;
  const size_t lcap = (size_t)1 << D;

  LAUNCH_CHECK(b2_launch_tree_init(tree, ctl, b->d_seg[0].p, b->d_ev[0].p, d_n_leaves, (int)n, b->d_hist_work.p, s));
  CUDA_CHECK(cudaMemsetAsync(b->d_leaf_sums.p, 0, 4 * lcap * sizeof(long long), s));
  mark_phase(b, 0);
  // ---- root histogram (no gather; row count known on the host)
  const int sh = b->log2_shards;
  const int shard_rank = b->shards > 1 ? b->comm->rank : 0;
  CUDA_CHECK(cudaMemsetAsync(build_target(b, b->hist[0].p), 0, b->node_elems * sizeof(long long), s));
  launch_hist(b, st, b->q.p, nullptr, nullptr, 1, build_target(b, b->hist[0].p));
  mark_phase(b, 1);
  exchange_and_subtract(b, st, nullptr, b->hist[0].p, nullptr, nullptr, 1, 1);
  LAUNCH_CHECK(b2_launch_root_totals(b->hist[0].p, G, b->d_ev[0].p, b->d_qexp.p, p.qbits, dp, sh, tree.sum_g, tree.sum_h, s));
  st.kernel_launches += 2;
  int hb = 0;  // hist buffer holding the current level
  for (int d = 0; d <= D; ++d) {
    const int cur = d & 1, nxt = cur ^ 1;
    const int max_nodes_level = 1 << d;
    const bool can_split = d < D;
    // candidates per node of this level: the scan's CTAs per node (its layout depends on the node count) + categorical
    const int cpn_num = b2_eval_ctas_per_node(G, sh, max_nodes_level);
    const int cpn = cpn_num + (m->any_cat() ? b2_cat_ctas() : 0);
    B2DecideArgs da = decide_args(b, tree, cp, d, cpn);
    // one GPU, numeric features only, levels scanned by the narrow layout: the last CTA of the scan decides the level
    // (no decide launch)
    const bool fold_decide = can_split && !multi && !m->any_cat() && max_nodes_level <= b2_eval_narrow_max_nodes();
    if (can_split) {
      const B2ColSample cs = col_sample(b, d, n_level_feats[d], tree_index, da.ic);
      // siblings of this level: parent (previous level buffer) - built, formed in the scan; stored only when the next
      // level takes them as parents
      B2SiblingSub sub{nullptr, nullptr, nullptr, 0};
      if (sub_in_scan && d > 0) {
        sub.parent_level = b->hist[hb ^ 1].p; sub.triples = b->d_triples.p;
        sub.sib_out = d + 1 < D ? b->hist[hb].p : nullptr; sub.sib_base = max_nodes_level / 2;
      }
      LAUNCH_CHECK(b2_launch_eval_splits(b->hist[hb].p, G, b->d_ev[cur].p, max_nodes_level, m->d_group_first.p, m->d_group_size.p,
                                         m->d_nbins.p, m->d_has_missing.p, m->any_cat() ? m->d_is_cat.p : nullptr, b->d_qexp.p,
                                         p.qbits, dp, b->d_cands.p, cpn, ctl + cur, sh, shard_rank, cs, b->d_seg[cur].p, sub,
                                         fold_decide ? &da : nullptr, b->d_eval_done.p, s));
      st.kernel_launches++;
      if (m->any_cat()) {
        LAUNCH_CHECK(b2_launch_eval_cat_splits(b->hist[hb].p, G, b->d_ev[cur].p, max_nodes_level, m->d_cat_feats.p,
                                               (int)m->cat_feats.size(), m->d_feat_byte.p, m->d_nbins.p, b->d_qexp.p, p.qbits, dp,
                                               b->d_cands.p, cpn, cpn_num, ctl + cur, sh, shard_rank, cs, b->d_seg[cur].p, s));
        st.kernel_launches++;
      }
      if (p2p) {   // decide_kernel stores the candidates straight into the peers' tables and waits for theirs
        da.cands = b->d_cands_all.p;
        da.cand_rank_stride = b->p2p.cand_cap;
      } else if (b->shards > 1) {   // every rank scanned only its own slots: gather the per-node candidates
        const size_t bytes = (size_t)max_nodes_level * cpn * sizeof(B2SplitCand);
        NCCL_CHECK(nccl()->AllGather(b->d_cands.p, b->d_cands_all.p, bytes, kNcclUint8, b->comm->comm, s));
        da.cands = b->d_cands_all.p;
      }
    }
    if (!fold_decide) {
      LAUNCH_CHECK(b2_launch_decide(&da, (p2p && can_split) ? &b->p2p.pp : nullptr, s));
      st.kernel_launches++;
    }
    mark_phase(b, 4);
    if (!can_split) break;
    if (d == D - 1) {   // with leaf_stream the sums are left to leaf_accumulate_kernel after the last decide
      LAUNCH_CHECK(b2_launch_leaf_plan(b->d_leaves.p, &ctl[cur].leaf_base_next, b->d_seg_work.p, ctl + 2, s));
      assign_leaves(b, st, d, gh, b->d_qexp.p, leaf_stream ? nullptr : b->d_leaf_sums.p);
      st.kernel_launches++;
      mark_phase(b, 5);
      continue;
    }
    partition_level(b, st, d);
    mark_phase(b, 5);
    if (d + 1 < D) {
      // ---- histograms of level d+1: built children in slots [0, 2^d), siblings in [2^d, 2^(d+1))
      const int nh = hb ^ 1;
      long long* tgt = build_target(b, b->hist[nh].p);
      // (peer-memory exchange: every peer finished reading this rank's build buffer before it published the candidates
      // that the decide kernel above waited for, so the buffer can be zeroed here without another handshake)
      CUDA_CHECK(cudaMemsetAsync(tgt, 0, (size_t)max_nodes_level * b->node_elems * sizeof(long long), s));
      launch_hist(b, st, b->q.p, b->ridx[nxt].p, ctl + nxt, max_nodes_level, tgt);
      mark_phase(b, 1);
      exchange_and_subtract(b, st, b->hist[hb].p, b->hist[nh].p, sub_in_scan ? nullptr : b->d_triples.p, ctl + nxt,
                            max_nodes_level, max_nodes_level);
      hb = nh;
    }
  }
  // ---- leaves: 40-bit fixed-point leaf sums -> sum over the ranks -> weights -> margin update
  if (leaf_stream) {   // every row's leaf index is in pos: sum the leaves in row order
    LAUNCH_CHECK(b2_launch_leaf_accumulate(gh, b->pos.p, n, D, b->d_qexp.p, 40, b->d_leaf_sums.p, ctx->num_sms, s));
    st.kernel_launches++;
  }
  if (p2p) { LAUNCH_CHECK(b2_launch_p2p_leaf_sums(&b->p2p.pp, d_n_leaves, b->d_leaf_sums.p, s)); st.kernel_launches++; }
  else allreduce(b->comm, b->d_leaf_sums.p, 4 * lcap, kNcclInt64, kNcclSum, s);   // limb by limb: exact
  LAUNCH_CHECK(b2_launch_leaf_values(b->d_leaves.p, d_n_leaves, b->d_leaf_sums.p, b->d_qexp.p, 40, cp, b->d_leaf_values.p, tree, b->t_qexp.p, s));
  // reg:quantileerror: the leaf value becomes the alpha_k-quantile of the leaf's residuals at the margin before this tree
  if (b->refresh_leaves)
    st.kernel_launches += quantile_select(b, k, b->pos.p, b->margin.p, gh, b->d_qexp.p, d_n_leaves, (int)lcap, cp.eta,
                                          b->d_leaves.p, b->d_leaf_values.p, tree.leaf_value);
  LAUNCH_CHECK(b2_launch_margin_update(b->margin.p, K, k, b->pos.p, b->d_leaf_values.p, p.dart ? b->d_dart_w_new.p : nullptr, n,
                                       ctx->num_sms, s));
  st.kernel_launches += 2;
  mark_phase(b, 6);
  // ---- read the finished tree back (pinned, asynchronous; resolved when the round is drained)
  char* stg = (char*)b->rb[b->rb_cur].staging[slot];
  // one copy: the category sets (the block's tail) only when the matrix has categorical features
  CUDA_CHECK(cudaMemcpyAsync(stg, b->t_block.p, m->any_cat() ? L.bytes : L.off_cat, cudaMemcpyDeviceToHost, s));
}

// read-back block of a vector-leaf tree (d_vblock): node totals [max_nodes][T][g, h] int64, node vectors [max_nodes][T]
// float, the T exponent pairs
struct VectorLayout { size_t off_vec, off_qexp, bytes; };
VectorLayout vector_layout(int max_depth, int T) {
  const size_t mx = (size_t)1 << (max_depth + 1);
  VectorLayout V;
  V.off_vec = mx * T * 2 * sizeof(long long);
  V.off_qexp = V.off_vec + mx * T * sizeof(float);
  V.bytes = V.off_qexp + 2 * (size_t)T * sizeof(int32_t);
  return V;
}

// One vector-leaf tree for all T targets (DESIGN.md 2 item 19), one GPU.  The partition, the leaf plan, sampling and the
// tree topology are the scalar tree's; per target: the quantisation (own exponents), the level histograms (own slice of
// d_vhist, siblings by hist_subtract) and the leaf sums.  The split scan sums the targets' gains, the child-totals kernel
// keeps every node's per-target totals, and the leaves are vectors.
void grow_vector_tree(Booster* b, int slot, TreeStats& st) {
  Matrix* m = b->train; Ctx* ctx = b->ctx; cudaStream_t s = ctx->stream; const Params& p = b->p;
  const int64_t n = m->n; const int T = p.num_target; const int G = m->n_groups; const int D = p.max_depth;
  ensure_ctl_tables(b);
  const TreeLayout L = tree_layout(D);
  const VectorLayout V = vector_layout(D, T);
  const bool leaf_stream = D <= b2_leaf_acc_max_depth();
  mark_phase(b, -1);
  const uint32_t tree_index = (uint32_t)b->trees.size() + (uint32_t)b->pending_trees + (uint32_t)slot;
  const size_t lcap = (size_t)1 << D, half = (size_t)1 << (D - 1);
  const size_t tstride = half * b->slice_elems;   // one target's level buffer
  long long* vtot = (long long*)b->d_vblock.p;
  float* tree_vec = (float*)(b->d_vblock.p + V.off_vec);
  int32_t* qexp_out = (int32_t*)(b->d_vblock.p + V.off_qexp);
  float* vgain = b->t_f32.p + L.max_nodes;        // the scalar tree's leaf_weight array, unused by vector trees
  quantise_gradients(b, st, 0, T, tree_index);
  const std::vector<int> n_level_feats = draw_column_masks(b, tree_index);
  const B2TrainParamDev dp = train_params(p);
  const B2CtlParams cp = ctl_params(p);
  const bool multi = b->comm && b->comm->world > 1;
  const B2TreeDev tree = tree_dev(b);
  int32_t* d_n_leaves = tree.n_nodes + 1;
  B2LevelCtl* ctl = b->d_ctl.p;
  const size_t sums_stride = 4 * lcap;
  LAUNCH_CHECK(b2_launch_tree_init(tree, ctl, b->d_seg[0].p, b->d_ev[0].p, d_n_leaves, (int)n, b->d_hist_work.p, s));
  CUDA_CHECK(cudaMemsetAsync(b->d_vsums.p, 0, (size_t)T * sums_stride * sizeof(long long), s));
  mark_phase(b, 0);
  for (int k = 0; k < T; ++k) {   // root histograms, one per target
    long long* tgt = b->d_vhist[0].p + (size_t)k * tstride;
    CUDA_CHECK(cudaMemsetAsync(tgt, 0, b->node_elems * sizeof(long long), s));
    launch_hist(b, st, b->q.p + (size_t)k * n, nullptr, nullptr, 1, tgt);
    mark_phase(b, 1);
    exchange_and_subtract(b, st, nullptr, tgt, nullptr, nullptr, 1, 1);
  }
  LAUNCH_CHECK(b2_launch_vector_root_totals(b->d_vhist[0].p, tstride, T, G, b->d_qexp.p, p.qbits, dp, vtot, vgain, s));
  st.kernel_launches++;
  const int cpn = b2_eval_vector_ctas_per_node(G);
  int hb = 0;
  for (int d = 0; d <= D; ++d) {
    const int cur = d & 1, nxt = cur ^ 1;
    const int max_nodes_level = 1 << d;
    const bool can_split = d < D;
    B2DecideArgs da = decide_args(b, tree, cp, d, cpn);
    da.vector_leaf = 1;
    if (can_split) {
      const B2ColSample cs = col_sample(b, d, n_level_feats[d], tree_index, da.ic);
      LAUNCH_CHECK(b2_launch_eval_splits_vector(b->d_vhist[hb].p, tstride, T, G, b->d_ev[cur].p, max_nodes_level, vtot, vgain,
                                                m->d_group_first.p, m->d_group_size.p, m->d_nbins.p, m->d_has_missing.p,
                                                b->d_qexp.p, p.qbits, dp, b->d_cands.p, cpn, ctl + cur, cs, b->d_seg[cur].p, s));
      st.kernel_launches++;
    }
    LAUNCH_CHECK(b2_launch_decide(&da, nullptr, s));
    st.kernel_launches++;
    mark_phase(b, 4);
    if (!can_split) break;
    // the children's per-target totals, from this level's histograms (still in d_vhist[hb])
    LAUNCH_CHECK(b2_launch_vector_child_totals(b->d_vhist[hb].p, tstride, T, G, max_nodes_level, ctl + cur, b->d_split_work.p,
                                               b->d_pair_parent.p, b->d_seg[nxt].p, tree.parent, m->d_feat_byte.p, m->d_nbins.p,
                                               b->d_qexp.p, p.qbits, dp, vtot, vgain, b->d_ev[nxt].p, s));
    st.kernel_launches++;
    if (d == D - 1) {   // every row's leaf index (and without leaf_stream, the leaf sums of every target)
      LAUNCH_CHECK(b2_launch_leaf_plan(b->d_leaves.p, &ctl[cur].leaf_base_next, b->d_seg_work.p, ctl + 2, s));
      for (int k = 0; k < (leaf_stream ? 1 : T); ++k)
        assign_leaves(b, st, d, b->gh.p + (size_t)k * n, b->d_qexp.p + 2 * k,
                      leaf_stream ? nullptr : b->d_vsums.p + (size_t)k * sums_stride);
      st.kernel_launches++;
      mark_phase(b, 5);
      continue;
    }
    partition_level(b, st, d);
    mark_phase(b, 5);
    if (d + 1 < D) {   // per target: built children, then siblings = parent - built over the target's whole slice
      const int nh = hb ^ 1;
      for (int k = 0; k < T; ++k) {
        long long* tgt = b->d_vhist[nh].p + (size_t)k * tstride;
        CUDA_CHECK(cudaMemsetAsync(tgt, 0, (size_t)max_nodes_level * b->node_elems * sizeof(long long), s));
        launch_hist(b, st, b->q.p + (size_t)k * n, b->ridx[nxt].p, ctl + nxt, max_nodes_level, tgt);
        mark_phase(b, 1);
        exchange_and_subtract(b, st, b->d_vhist[hb].p + (size_t)k * tstride, tgt, b->d_triples.p, ctl + nxt, max_nodes_level,
                              max_nodes_level);
      }
      hb = nh;
    }
  }
  if (leaf_stream)
    for (int k = 0; k < T; ++k) {
      LAUNCH_CHECK(b2_launch_leaf_accumulate(b->gh.p + (size_t)k * n, b->pos.p, n, D, b->d_qexp.p + 2 * k, 40,
                                             b->d_vsums.p + (size_t)k * sums_stride, ctx->num_sms, s));
      st.kernel_launches++;
    }
  allreduce(b->comm, b->d_vsums.p, (size_t)T * sums_stride, kNcclInt64, kNcclSum, s);   // limb by limb: exact
  if (multi) st.allreduce_bytes += (double)T * sums_stride * sizeof(long long);
  LAUNCH_CHECK(b2_launch_vector_leaf_values(b->d_leaves.p, d_n_leaves, b->d_vsums.p, sums_stride, b->d_qexp.p, T, 40, cp,
                                            b->d_leaf_vec.p, tree_vec, qexp_out, s));
  LAUNCH_CHECK(b2_launch_margin_update_vector(b->margin.p, T, b->pos.p, b->d_leaf_vec.p, n, ctx->num_sms, s));
  st.kernel_launches += 2;
  mark_phase(b, 6);
  CUDA_CHECK(cudaMemcpyAsync(b->rb[b->rb_cur].staging[slot], b->t_block.p, L.off_cat, cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaMemcpyAsync(b->rb[b->rb_cur].vstaging, b->d_vblock.p, V.bytes, cudaMemcpyDeviceToHost, s));
}

void apply_tree_stats(Booster* b, long long hist_launches, long long kernel_launches, double allreduce_bytes,
                      const std::vector<std::pair<cudaEvent_t, cudaEvent_t>>& ev) {
  b->t.hist_launches += hist_launches; b->t.kernel_launches += kernel_launches; b->t.allreduce_bytes += allreduce_bytes;
  for (auto& pr : ev) b->rb[b->rb_cur].hist_events.push_back(pr);
}

// buffers a tree needs, allocated outside of any capture
void prepare_tree_buffers(Booster* b, int slot) {
  Matrix* m = b->train; const int64_t n = m->n;
  ensure_ctl_tables(b);
  const TreeLayout L = tree_layout(b->p.max_depth);
  const size_t rows = (size_t)std::max<int64_t>(n, 1);
  b->d_absmax.ensure(2 * (size_t)b->p.num_class); b->d_qexp.ensure(2);
  b->q.ensure(rows); b->ridx[0].ensure(rows); b->ridx[1].ensure(rows); b->pos.ensure(rows);
  if (b->refresh_leaves) ensure_quantile_buffers(b, 1 << b->p.max_depth);
  if (b->staging_bytes != L.bytes) {
    for (auto& r : b->rb) {
      for (void* h : r.staging) cudaFreeHost(h);
      r.staging.clear();
    }
    b->staging_bytes = L.bytes;
  }
  std::vector<void*>& staging = b->rb[b->rb_cur].staging;
  while ((int)staging.size() <= slot) { void* h = nullptr; CUDA_CHECK(cudaMallocHost(&h, L.bytes)); staging.push_back(h); }
  if (b->p.vector_leaf()) {
    const int T = b->p.num_target, D = b->p.max_depth;
    const size_t lcap = (size_t)1 << D, half = (size_t)1 << (D - 1);
    const size_t hist_elems = (size_t)T * half * b->slice_elems;
    // the level histograms, the quantised pairs and the leaf sums of the T targets
    const double gib = (2.0 * (double)hist_elems * sizeof(long long) + (double)rows * T * sizeof(int2) +
                        (double)T * 4 * lcap * sizeof(long long)) / (double)(1ull << 30);
    if (gib > 48.0)
      fail("multi_strategy=multi_output_tree with %d targets at max_depth %d needs %.1f GiB of per-target buffers (at most "
           "48); use fewer targets, a smaller max_depth or multi_strategy=one_output_per_tree", T, D, gib);
    b->d_vhist[0].ensure(hist_elems); b->d_vhist[1].ensure(hist_elems);
    b->d_vsums.ensure((size_t)T * 4 * lcap); b->d_leaf_vec.ensure(lcap * T);
    b->d_absmax.ensure(2 * (size_t)T); b->d_qexp.ensure(2 * (size_t)T);
    b->q.ensure(rows * T);
    const VectorLayout V = vector_layout(D, T);
    b->d_vblock.ensure(V.bytes);
    Booster::RoundBuffers& R = b->rb[b->rb_cur];
    if (R.vstaging_bytes != V.bytes) {
      if (R.vstaging) cudaFreeHost(R.vstaging);
      R.vstaging = nullptr; R.vstaging_bytes = 0;
      CUDA_CHECK(cudaMallocHost(&R.vstaging, V.bytes));
      R.vstaging_bytes = V.bytes;
    }
  }
}

// One class tree: replay its CUDA graph when the launch sequence is the same for every tree (no row / column sampling,
// fused |g|,|h| maxima, no per-phase profiling), otherwise enqueue the kernels one by one.  The first tree of a class
// slot always runs with direct launches (it allocates); the next two are captured, one graph per round parity (each
// copies into its own read-back block and records its own events), and the following ones replay them alternately.
// A stale graph (tree_params_changed) is captured again and applied to its executable graph with cudaGraphExecUpdate:
// the topology is the same, only kernel arguments differ.  It is instantiated again only when the update is refused.
void run_tree(Booster* b, int k, int slot) {
  cudaStream_t s = b->ctx->stream; const Params& p = b->p;
  prepare_tree_buffers(b, slot);
  static const bool want_graph = env_flag("B2_GRAPH", true);
  const bool eligible = want_graph && !b->graph_failed && b->absmax_fused && p.subsample >= 1.0f && !p.use_cols() &&
                        p.profile < 2 && p.num_parallel_tree == 1;
  auto direct = [&]() {
    TreeStats st;
    if (p.vector_leaf()) grow_vector_tree(b, slot, st);
    else grow_tree(b, k, slot, st);
    apply_tree_stats(b, st.hist_launches, st.kernel_launches, st.allreduce_bytes, st.hist_ev);
    b->direct_trees[k]++;
  };
  if (!eligible) { direct(); return; }
  std::map<int, Booster::TreeGraph>& graphs = b->rb[b->rb_cur].graphs;
  auto it = graphs.find(k);
  if (it == graphs.end() || it->second.stale) {
    if (it == graphs.end() && b->direct_trees[k] == 0) { direct(); return; }
    const auto t0 = std::chrono::steady_clock::now();
    TreeStats st; st.capturing = true;
    cudaGraph_t graph = nullptr; cudaGraphExec_t exec = nullptr;
    bool ok = cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
    if (ok) {
      try { if (p.vector_leaf()) grow_vector_tree(b, slot, st); else grow_tree(b, k, slot, st); }
      catch (const B2Error& e) {
        cudaStreamEndCapture(s, &graph); if (graph) cudaGraphDestroy(graph); cudaGetLastError();
        for (auto& pr : st.hist_ev) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
        throw;
      }
      ok = cudaStreamEndCapture(s, &graph) == cudaSuccess && graph != nullptr;
    }
    if (ok && it != graphs.end()) {
      cudaGraphExecUpdateResultInfo info;
      if (cudaGraphExecUpdate(it->second.exec, graph, &info) == cudaSuccess) {
        exec = it->second.exec;
        it->second.exec = nullptr;   // moved to the new entry; the old one keeps only its events
        b->t.graph_updates++;
      } else {
        cudaGetLastError();
        b->t.graph_reinstantiations++;
      }
    }
    if (ok && !exec) ok = cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess;
    if (graph) cudaGraphDestroy(graph);
    if (it != graphs.end()) {
      Booster::destroy_graph(it->second);
      graphs.erase(it);
      b->t.graph_update_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
    if (!ok) {
      cudaGetLastError();
      for (auto& pr : st.hist_ev) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
      b->graph_failed = true;
      fprintf(stderr, "[b2hist] CUDA graph capture of the tree failed; continuing with direct launches\n");
      direct();
      return;
    }
    Booster::TreeGraph g;
    g.exec = exec; g.hist_ev = st.hist_ev; g.hist_launches = st.hist_launches; g.kernel_launches = st.kernel_launches;
    g.allreduce_bytes = st.allreduce_bytes;
    it = graphs.emplace(k, std::move(g)).first;
  }
  CUDA_CHECK(cudaGraphLaunch(it->second.exec, s));
  apply_tree_stats(b, it->second.hist_launches, it->second.kernel_launches, it->second.allreduce_bytes, it->second.hist_ev);
}

// after the round's stop event: turn read-back block `block` into a host tree (A.7 bookkeeping)
void materialize_tree(Booster* b, const void* block) {
  Matrix* m = b->train; const Params& p = b->p;
  const TreeLayout L = tree_layout(p.max_depth);
  const char* st = (const char*)block;
  const int32_t* i32 = (const int32_t*)st; const size_t mx = L.max_nodes;
  const float* f32 = (const float*)(st + L.off_f32);
  const long long* i64 = (const long long*)(st + L.off_i64);
  const int32_t* qexp = (const int32_t*)(st + L.off_qexp);
  const int nn = i32[7 * mx];
  const uint32_t* cat = (const uint32_t*)(st + L.off_cat);
  if (nn < 1 || (size_t)nn > mx) fail("corrupt tree read-back (n_nodes=%d)", nn);
  const double inv_sg = ldexp(1.0, qexp[0] - p.qbits), inv_sh = ldexp(1.0, qexp[1] - p.qbits);
  TreeHost t;
  for (int i = 0; i < nn; ++i) {
    t.add(i32[2 * mx + i]);
    t.left[i] = i32[i]; t.right[i] = i32[mx + i]; t.feature[i] = i32[3 * mx + i];
    const double G = (double)i64[i] * inv_sg, H = (double)i64[mx + i] * inv_sh;
    t.sum_hess[i] = H;
    if (t.feature[i] >= 0) {
      const int f = t.feature[i], bin = i32[4 * mx + i];
      t.split_bin[i] = bin; t.default_left[i] = (uint8_t)i32[5 * mx + i]; t.loss_chg[i] = f32[i];
      if (m->any_cat() && i32[6 * mx + i]) {
        // categorical split: one-hot keeps the category as split condition, a partition split stores NaN (RegTree::ExpandCategorical)
        t.split_type[i] = 1; t.any_cat = true;
        for (int w8 = 0; w8 < 8; ++w8) t.cat_bits[(size_t)i * 8 + w8] = cat[(size_t)i * 8 + w8];
        t.cond[i] = bin >= 0 ? (float)bin : NAN;
      } else
      t.cond[i] = bin < 0 ? m->min_vals[f] : m->cut_vals[m->cut_ptrs[f] + bin];
      t.base_weight[i] = h_calc_weight(p, G, H);
      t.value[i] = t.base_weight[i];
    } else {
      t.base_weight[i] = f32[mx + i];
      t.value[i] = f32[2 * mx + i];
    }
  }
  // histogram rows of this tree for the roofline accounting: root + built children per level
  const long long* level_rows = i64 + 2 * mx;
  long long rows = m->n; int launches_nonempty = m->n > 0 ? 1 : 0;
  for (int d = 1; d < p.max_depth; ++d) { rows += level_rows[d]; if (level_rows[d] > 0) launches_nonempty++; }
  long long gathered = rows - m->n;
  int built_nodes = 0;
  for (int i = 0; i < nn; ++i) if (t.feature[i] >= 0) built_nodes++;   // one built child per split (+ root)
  b->t.hist_rows += rows;
  b->t.hist_bytes += (double)rows * (m->F + 8) + (double)gathered * 4 + (double)(built_nodes + 1) * m->F * 256.0 * 16.0;
  b->trees.push_back(std::move(t));
}

// a vector-leaf tree from its read-back blocks (grow_vector_tree): the scalar block's topology, splits and loss_chg, and
// the vector block's per-target node totals (sum_hess = sum over the targets of H_k; an internal node's vector holds
// fp32(fp32(w_k) * eta) of its own sums) and leaf vectors
void materialize_vector_tree(Booster* b, const void* block, const void* vblock) {
  Matrix* m = b->train; const Params& p = b->p; const int T = p.num_target;
  const TreeLayout L = tree_layout(p.max_depth);
  const VectorLayout V = vector_layout(p.max_depth, T);
  const char* st = (const char*)block;
  const int32_t* i32 = (const int32_t*)st; const size_t mx = L.max_nodes;
  const float* f32 = (const float*)(st + L.off_f32);
  const long long* vtot = (const long long*)vblock;
  const float* vec = (const float*)((const char*)vblock + V.off_vec);
  const int32_t* qexp = (const int32_t*)((const char*)vblock + V.off_qexp);
  const int nn = i32[7 * mx];
  if (nn < 1 || (size_t)nn > mx) fail("corrupt tree read-back (n_nodes=%d)", nn);
  TreeHost t;
  t.leaf_vec.assign((size_t)nn * T, 0.0f);
  for (int i = 0; i < nn; ++i) {
    t.add(i32[2 * mx + i]);
    t.left[i] = i32[i]; t.right[i] = i32[mx + i]; t.feature[i] = i32[3 * mx + i];
    double H_sum = 0.0;
    for (int k = 0; k < T; ++k) {
      const double G = (double)vtot[((size_t)i * T + k) * 2] * ldexp(1.0, qexp[2 * k] - p.qbits);
      const double H = (double)vtot[((size_t)i * T + k) * 2 + 1] * ldexp(1.0, qexp[2 * k + 1] - p.qbits);
      H_sum += H;
      t.leaf_vec[(size_t)i * T + k] = t.feature[i] >= 0 ? h_calc_weight(p, G, H) * p.eta : vec[(size_t)i * T + k];
    }
    t.sum_hess[i] = H_sum;
    if (t.feature[i] >= 0) {
      const int f = t.feature[i], bin = i32[4 * mx + i];
      t.split_bin[i] = bin; t.default_left[i] = (uint8_t)i32[5 * mx + i]; t.loss_chg[i] = f32[i];
      t.cond[i] = bin < 0 ? m->min_vals[f] : m->cut_vals[m->cut_ptrs[f] + bin];
    }
  }
  const long long* level_rows = (const long long*)(st + L.off_i64) + 2 * mx;
  long long rows = m->n;
  for (int d = 1; d < p.max_depth; ++d) rows += level_rows[d];
  b->t.hist_rows += rows * T;
  b->trees.push_back(std::move(t));
}

// B2_BoosterAddTree: a tree from outside the engine is walked by the prediction kernels, the TreeSHAP path builder and
// the refresh updater, which follow split children until they reach a leaf.  So every split's children are nodes of
// the tree and no split is reached twice from the root (no cycle, no shared subtree); nodes the root does not reach
// (xgboost's deleted nodes) are never walked.  A model keeps the multi_strategy it was trained with.
void check_tree(const Booster* b, const TreeHost& t) {
  const size_t ti = b->trees.size();
  const int n = t.size(), T = b->p.num_target;
  if (n < 1) fail("tree %zu has no nodes", ti);
  for (int i = 0; i < n; ++i) {
    if (t.feature[i] < 0) {
      if (t.split_type[i]) fail("tree %zu node %d is a leaf with split_type %d (categorical)", ti, i, t.split_type[i]);
      continue;
    }
    if (t.feature[i] >= b->n_features)
      fail("tree %zu node %d splits on feature %d; the model has %d features", ti, i, t.feature[i], b->n_features);
    for (int c : {t.left[i], t.right[i]})
      if (c < 0 || c >= n) fail("tree %zu node %d has child %d outside [0, %d)", ti, i, c, n);
  }
  std::vector<uint8_t> seen(n, 0);
  std::vector<int> stack{0};
  while (!stack.empty()) {
    const int i = stack.back(); stack.pop_back();
    if (t.feature[i] < 0) continue;
    if (seen[i]) fail("tree %zu node %d splits and is reached twice from the root", ti, i);
    seen[i] = 1;
    stack.push_back(t.left[i]); stack.push_back(t.right[i]);
  }
  if (!b->p.vector_leaf() && !t.leaf_vec.empty())
    fail("tree %zu is a vector-leaf tree (multi_strategy=multi_output_tree); this booster grows single-output trees "
         "(multi_strategy=one_output_per_tree, %d target(s)): a model keeps the strategy it was trained with", ti, T);
  if (b->p.vector_leaf() && t.leaf_vec.empty())
    fail("tree %zu is a single-output tree (multi_strategy=one_output_per_tree); this booster grows vector-leaf trees "
         "(multi_strategy=multi_output_tree): a model keeps the strategy it was trained with", ti);
  if (b->p.vector_leaf() && t.leaf_vec.size() != (size_t)n * T)
    fail("tree %zu has a leaf vector of %zu values; it needs %lld (%d nodes x %d targets)", ti, t.leaf_vec.size(),
         (long long)n * T, n, T);
}

void sync_device_trees(Booster* b) {
  if (b->d_trees_synced == (int)b->trees.size()) return;
  if (b->p.vector_leaf()) {   // [model nodes][T], in the order of d_nodes
    b->h_leaf_table.clear();
    for (auto& t : b->trees) b->h_leaf_table.insert(b->h_leaf_table.end(), t.leaf_vec.begin(), t.leaf_vec.end());
    upload(b->d_leaf_table, b->h_leaf_table, b->ctx->stream);
  }
  b->h_nodes.clear(); b->h_tree_offset.clear(); b->h_cat_table.clear();
  for (auto& t : b->trees) {
    b->h_tree_offset.push_back((int32_t)b->h_nodes.size());
    for (int i = 0; i < t.size(); ++i) {
      int32_t cat_slot = -1;
      if (t.feature[i] >= 0 && t.split_type[i]) {
        cat_slot = (int32_t)(b->h_cat_table.size() / 8);
        b->h_cat_table.insert(b->h_cat_table.end(), t.cat_bits.begin() + (size_t)i * 8, t.cat_bits.begin() + (size_t)i * 8 + 8);
      }
      // pad: the split bin, read by the DART margin rebuild on the bin matrix (dart_kernel.cu)
      b->h_nodes.push_back(B2TreeNodeDev{t.left[i], t.right[i], t.feature[i], t.cond[i], t.value[i], (int32_t)t.default_left[i],
                                         cat_slot, t.split_bin[i]});
    }
  }
  cudaStream_t s = b->ctx->stream;
  upload(b->d_nodes, b->h_nodes, s); upload(b->d_tree_offset, b->h_tree_offset, s); upload(b->d_cat_table, b->h_cat_table, s);
  CUDA_CHECK(cudaStreamSynchronize(s));
  b->d_trees_synced = (int)b->trees.size();
}

}  // namespace b2host
