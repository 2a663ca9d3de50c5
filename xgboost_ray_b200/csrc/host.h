// host.h -- what the host files of libb2hist.so share: errors, the device context and memory, the communicator,
// Matrix, Params and Booster, and the functions one host file calls in another.
//
// One process drives one GPU (one Ray actor per GPU in the reference, xgboost_ray/main.py:862-892); row-sharded data
// parallel, model replicated, per-level histogram allreduce (SURVEY.md 8e).  Mirrors, for the hot path only, what
// `xgboost` does underneath xgboost_ray/main.py:745-752:
//   gradient -> [per class tree] quantise -> root hist -> allreduce -> eval -> partition ->
//   smaller-child hist -> allreduce -> sibling subtraction -> ... -> leaf sums -> margin update.
//
// device.cu   device context, memory pool, pinned upload pipeline, NCCL
// matrix.cu   matrix construction, registry and interleaved NVLink ingest, cuts, binning
// params.cu   parameter parsing, the objective table (kObjectives), metric names
// tree.cu     growing one tree (scalar or vector-leaf) and reading it back
// round.cu    booster setup and a boosting round: label checks, gradients, base_score, DART, refresh, the round pipeline
// predict.cu  model caches, TreeSHAP paths, prediction, contributions, leaf indices, evaluation margins, eval metrics
// engine.cu   the C ABI (include/b2hist.h): handle lookups, then one call into the files above
//
// Everything is in namespace b2host, and every file opens it with hidden visibility, so the library exports no symbol
// of the host layer: only the C ABI of engine.cu reaches it.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <string>
#include <utility>
#include <vector>

#include "../../include/b2hist.h"
#include "common.cuh"
#include "launch.h"

namespace b2host __attribute__((visibility("hidden"))) {

// ---------------------------------------------------------------- errors
struct B2Error { std::string msg; };
[[noreturn]] void fail(const char* fmt, ...);
#define CUDA_CHECK(expr)                                                                       \
  do {                                                                                         \
    cudaError_t e_ = (expr);                                                                   \
    if (e_ != cudaSuccess) fail("CUDA error %s at %s:%d: %s", cudaGetErrorName(e_), __FILE__, __LINE__, cudaGetErrorString(e_)); \
  } while (0)
#define LAUNCH_CHECK(expr)                                                                     \
  do {                                                                                         \
    int e_ = (expr);                                                                           \
    if (e_ != 0) fail("kernel launch failed (%s) at %s:%d", cudaGetErrorString((cudaError_t)e_), __FILE__, __LINE__); \
  } while (0)

// ---------------------------------------------------------------- device context
struct Ctx {
  int device = -1;
  cudaStream_t stream = nullptr;
  int num_sms = 0;
};

Ctx* get_ctx(int device);

// Device memory goes through a small caching pool: matrices and boosters allocate and free the same few large blocks
// over and over (every DMatrix, every sketch), cudaFree synchronises the device, and once a peer's buffers are mapped
// for the NVLink exchange every cudaMalloc also has to be mapped into the peers (measured: the second quantisation of
// a bench run took 0.28 s with peer mappings against 0.06 s without).  Freed blocks are kept per device and handed out
// again when their size fits (<= 25 % + 1 MiB slack); the cache is bounded by B2_POOL_MAX_GB (default 24, under a third
// of an 80 GB H100) and emptied when an allocation fails.
struct DevPool {
  std::mutex mu;
  std::multimap<size_t, void*> free_blocks;
  size_t cached = 0;
};

extern DevPool g_dev_pool[64];
void pool_trim(DevPool& pool, size_t keep);   // caller holds pool.mu
void* pool_alloc(size_t bytes, size_t* got, int* dev_out);
void pool_free(void* p, size_t bytes, int dev);

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;          // elements the caller may use
  size_t block_bytes = 0;  // size of the pooled block behind p
  int dev = 0;
  void ensure(size_t n) {
    if (n <= cap) return;
    release();
    size_t got = 0;
    p = (T*)pool_alloc(n * sizeof(T), &got, &dev);
    block_bytes = got;
    cap = n;
  }
  void release() { if (p) pool_free(p, block_bytes, dev); p = nullptr; cap = 0; block_bytes = 0; }
  ~DevBuf() { release(); }
};

// ---------------------------------------------------------------- host -> device ingest
// Where the rows of an upload come from: this process (src) or ANOTHER process' memory (pid / remote_addr), row by row
// `row_stride` bytes apart -- the driver's matrix read with process_vm_readv straight into the pinned staging slices, so
// a shard never exists as a second host copy (matrix.py:471-484 puts every shard into the object store instead).
struct UploadSource {
  const void* src = nullptr;      // local, contiguous
  long long pid = 0;              // != 0: remote
  uint64_t remote_addr = 0;       // address of row 0 in process `pid`
  size_t row_bytes = 0, row_stride = 0;
};

void upload_pipelined(Ctx* ctx, void* dst, const UploadSource& u, size_t bytes);
void upload_pipelined(Ctx* ctx, void* dst, const void* src, size_t bytes);

// ---------------------------------------------------------------- NCCL (dlopen'ed)
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { kNcclSum = 0, kNcclMax = 2, kNcclMin = 3 };   // ncclRedOp_t
enum { kNcclUint8 = 1, kNcclInt32 = 2, kNcclUint32 = 3, kNcclInt64 = 4, kNcclUint64 = 5, kNcclFloat32 = 7, kNcclFloat64 = 8 };

struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*ReduceScatter)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*CommAbort)(ncclComm_t) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};

NcclApi* nccl();

#define NCCL_CHECK(expr)                                                                              \
  do {                                                                                                \
    int r_ = (expr);                                                                                  \
    if (r_ != 0) fail("NCCL error %d (%s) at %s:%d", r_, nccl()->GetErrorString(r_), __FILE__, __LINE__); \
  } while (0)

struct Comm {
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1, device = 0;
  std::atomic<bool> aborted{false};
  uint32_t* d_abort = nullptr;        // device word polled by the peer-memory waits (p2p.cuh); set by B2_CommAbort
  cudaStream_t abort_stream = nullptr;
};

void allreduce(Comm* c, void* buf, size_t count, int dtype, int op, cudaStream_t s);

// ---------------------------------------------------------------- handles
enum HandleKind { kComm = 1, kMatrix = 2, kBooster = 3 };
struct HandleBase { int kind; };
template <typename T>
T* from_handle(B2Handle h, int kind, const char* what) {
  if (!h) fail("null %s handle", what);
  HandleBase* b = reinterpret_cast<HandleBase*>(h);
  if (b->kind != kind) fail("handle is not a %s", what);
  return reinterpret_cast<T*>(h);
}

// The bins of a quantised matrix in their layout, dense or CSR (DESIGN.md 2 item 26).  Defined in matrix.cu, the one
// place that knows the layout: the launchers get the bins through bin_source.
struct MatrixBins;

struct Matrix : HandleBase {
  Matrix();
  ~Matrix();
  uint64_t margin_version = 0;   // bumped when base_margin changes (cached evaluation margins start from it)
  uint64_t uid = 0;       // unique for the life of the process; 0 = not registered (stack temporaries)
  Ctx* ctx = nullptr;
  int64_t n = 0;
  int F = 0;
  float missing = NAN;
  DevBuf<float> raw;     // [n][F], optional
  // CSR raw values instead of raw (B2_MatrixCreateFromCSR): row i stores entries [indptr[i], indptr[i+1]) of indices /
  // values, columns strictly increasing; an entry a row does not store is missing.  Kernels get raw rows through
  // raw_source, raw_rows or for_raw_tiles, never from these buffers directly.
  bool csr = false;
  int64_t nnz = 0;
  DevBuf<int64_t> csr_indptr; DevBuf<int32_t> csr_indices; DevBuf<float> csr_values;
  bool has_raw = false;  // raw, or the CSR buffers, are on the device
  int bin_layout = B2_BIN_LAYOUT_AUTO;   // the requested B2_BIN_LAYOUT_* (B2_MatrixSetBinLayout)
  std::unique_ptr<MatrixBins> qbins;
  bool quantized = false;
  int n_groups = 0, row_stride = 0, max_bin = 0;
  std::vector<int32_t> group_first, group_size, feat_byte;
  std::vector<int32_t> cut_ptrs;
  std::vector<float> cut_vals, min_vals;
  std::vector<uint8_t> has_missing;
  std::vector<int32_t> nbins;
  std::vector<uint8_t> is_cat;        // [F] 1 = categorical feature (B2_MatrixSetFeatureTypes); empty = all numeric
  std::vector<int32_t> cat_feats;     // ids of the categorical features
  DevBuf<int32_t> d_group_first, d_group_size, d_feat_byte, d_cut_ptrs, d_nbins, d_cat_feats;
  DevBuf<float> d_cut_vals;
  DevBuf<uint8_t> d_has_missing, d_is_cat;
  bool any_cat() const { return !cat_feats.empty(); }
  DevBuf<float> label, weight, base_margin;   // label [n][n_targets] row-major
  int64_t n_label = 0, n_weight = 0, n_base_margin = 0;
  int n_targets = 1;                    // label columns (B2_MatrixSetLabel); > 1: multi-target regression / multi-label
  bool has_labels(int T) const { return n_targets == T && n_label == n * T; }
  DevBuf<float> lower, upper;          // survival label bounds (label_lower_bound / label_upper_bound), read by survival:aft
  int64_t n_lower = 0, n_upper = 0;
  bool has_bounds() const { return n_lower == n && n_upper == n; }
  // query groups (B2_MatrixSetGroups): group g is rows [qgroup_ptr[g], qgroup_ptr[g+1]); read by the rank objectives and
  // the ndcg / map / pre metrics.  rank_version changes with the groups and the labels (the 1/IDCG cache key)
  std::vector<int64_t> h_qgroup_ptr;
  DevBuf<int64_t> qgroup_ptr;
  int64_t n_qgroups = 0, max_qgroup = 0;
  uint64_t rank_version = 0;
  bool has_qgroups() const { return n_qgroups > 0; }
  std::vector<uint32_t> fwq;         // feature_weights in Q16 (empty = all 1.0)
  DevBuf<uint32_t> d_fwq;
};

template <typename T>
void upload(DevBuf<T>& d, const T* h, size_t n, cudaStream_t s) {
  d.ensure(n ? n : 1);
  if (n) CUDA_CHECK(cudaMemcpyAsync(d.p, h, n * sizeof(T), cudaMemcpyHostToDevice, s));
}
template <typename T>
void upload(DevBuf<T>& d, const std::vector<T>& h, cudaStream_t s) { upload(d, h.data(), h.size(), s); }

// ---- matrix lifecycle (matrix.cu).  new_matrix refuses a bad shape or more rows than int32 ids; the caller sets ctx
std::unique_ptr<Matrix> new_matrix(int64_t n, int F, float missing);
B2Handle register_matrix(std::unique_ptr<Matrix> m);   // gives m its uid; the handle is released by free_matrix
void free_matrix(Matrix* m);
bool matrix_alive(uint64_t uid);
void upload_raw(Matrix* m, const UploadSource& u);    // raw: the n x F values of u
// B2_MatrixCreateFromProcessInterleaved: rows r = rank (mod world) of a remote matrix, exchanged over NVLink when it can
B2Handle ingest_interleaved(Comm* c, int64_t pid, uint64_t remote_addr, int64_t n_total_rows, int n_cols, int shard_rank,
                            float missing, int device);

// ---- raw rows (matrix.cu): the one place that knows whether a matrix holds its raw values dense or as CSR
constexpr size_t kRawTileBytes = (size_t)256 << 20;   // largest dense tile densified from a CSR matrix
// rows of one raw tile: all rows of a dense matrix; for CSR floor(kRawTileBytes / (4 F)) rounded down to a multiple of
// 128 (at least 128), so every tile starts on the 128-row alignment of bins_col's column stride
int64_t raw_tile_rows(const Matrix* m);
// dense float rows [r0, r0 + rows) x [0, F): a pointer into raw, or `tile` filled from the CSR (rows <= raw_tile_rows)
const float* raw_rows(Matrix* m, int64_t r0, int64_t rows, DevBuf<float>& tile);
// every row's raw values for the tree walks, which read a CSR matrix's stored entries directly (no dense tile)
B2RawRows raw_source(const Matrix* m);
// fn(X, r0, rows) over consecutive raw tiles of at most max_rows rows covering every row (once with rows = 0 for an
// empty matrix).  Uncapped, a dense matrix is one call with X = raw: the kernels run as on a plain dense matrix.
template <typename Fn>
void for_raw_tiles(Matrix* m, Fn fn, int64_t max_rows = INT64_MAX) {
  DevBuf<float> tile;
  const int64_t step = std::min(raw_tile_rows(m), max_rows);
  int64_t r0 = 0;
  do {
    const int64_t rows = std::min<int64_t>(step, m->n - r0);
    fn(raw_rows(m, r0, rows, tile), r0, rows);
    r0 += step;
  } while (r0 < m->n);
}
// uploads the CSR arrays and checks them; a matrix in the CSR bin layout kept indptr and indices, so only its values
void upload_csr(Matrix* m, const int64_t* indptr, const int32_t* indices, const float* values);
size_t matrix_device_bytes(const Matrix* m);

// ---- bins (matrix.cu): the one place that knows whether a quantised matrix holds its bins dense or as CSR
B2BinRows bin_source(const Matrix* m);             // fails on a matrix that is not quantised
void bins_to_host(const Matrix* m, uint8_t* out);  // out [n][F]: every cell's bin (an absent CSR entry: the missing bin)
// a matrix quantised from host bins, without cuts (the histogram entries B2_HistBuildRaw*): bins [n][F] for a dense
// matrix, one bin per stored entry [nnz] for a CSR one whose indptr / indices are uploaded (upload_csr)
void upload_bins(Matrix* m, const uint8_t* bins);

// B2_MatrixSlice: a new unquantised matrix of parent rows rows[0..n) (host array), gathered on the device
B2Handle slice_matrix(Matrix* parent, const int64_t* rows, int64_t n);

void setup_groups(Matrix* m);
// bytes of the two dense bin copies (bins and bins_col) of an n x F matrix, as bin_matrix allocates them
size_t dense_bin_bytes(int64_t n, int F);
// cuts (sketched, or borrowed ones checked against the categorical codes), the bin matrix, raw released unless keep_raw
void quantize_matrix(Matrix* m, Comm* comm, int max_bin, bool borrowed_cuts, bool keep_raw);

// ---------------------------------------------------------------- booster
constexpr int kMaxTargets = 4096;   // label columns of one matrix (as many trees per round as num_parallel_tree allows)
struct Params {
  int objective = kObjSquaredError;
  int objective_index = 0;   // its row of params.cu kObjectives (objective_row)
  std::string objective_name = "reg:squarederror";
  int num_class = 1;
  // label columns of a multi-target model (outputs per row; num_class then equals it).  Given as num_target when a model
  // is loaded, otherwise taken from the train matrix when the booster is created (set_targets)
  int num_target = 1;
  bool num_target_set = false;
  int num_parallel_tree = 1;   // trees grown per class and round from the SAME gradients (random forests); leaf values are scaled by eta / n
  int max_depth = 6;
  float eta = 0.3f, gamma = 0.0f, min_child_weight = 1.0f, lambda = 1.0f, alpha = 0.0f, base_score = 0.5f;
  int qbits = 18;
  int hist_chunk_rows = 0;  // 0 = auto
  int profile = 1;
  int num_feature = 0;
  int device = 0;
  int max_cat_to_onehot = 4, max_cat_threshold = 64;   // xgboost defaults (src/tree/param.h)
  float scale_pos_weight = 1.0f, max_delta_step = 0.0f;
  bool max_delta_step_set = false;             // false: count:poisson uses 0.7 (xgboost's Learner::ConfigureObjective)
  float huber_slope = 1.0f;                    // reg:pseudohubererror delta (also the mphe metric's)
  float tweedie_variance_power = 1.5f;         // reg:tweedie rho in [1, 2)
  int aft_dist = kAftNormal;                   // survival:aft distribution (B2AftDist)
  float aft_sigma = 1.0f;                      // survival:aft scale sigma > 0
  int rank_k = 32;                             // lambdarank_num_pair_per_sample (topk pairs: the first k model positions)
  bool ndcg_exp_gain = true;                   // ndcg gain 2^y - 1 (true) or y (rank:ndcg and the ndcg metrics)
  float subsample = 1.0f, colsample_bytree = 1.0f, colsample_bylevel = 1.0f, colsample_bynode = 1.0f;
  int seed = 0;
  bool base_score_set = false;   // false: estimated from the labels before the first tree (xgboost >= 2.0, A.3)
  // interaction_constraints: feature sets S_1 .. S_C (a tree path with two or more features stays inside one set);
  // empty = no constraints.  Text form "0,1;2,3,4": sets separated by ';', features by ','.
  std::vector<std::vector<int64_t>> interaction_sets;
  // booster=dart (Dart in xgboost's gbtree.cc): trees dropped at random each round, per-tree weights
  bool dart = false;
  double rate_drop = 0.0, skip_drop = 0.0;
  bool dart_weighted = false;       // sample_type: uniform (false) / weighted
  bool dart_forest = false;         // normalize_type: tree (false) / forest
  bool one_drop = false;
  // reg:quantileerror: one output (and one tree per round) per alpha
  std::vector<float> quantile_alpha{0.5f};
  bool num_class_set = false;
  // multi_strategy: 0 one_output_per_tree (one tree per target and round), 1 multi_output_tree (one vector-leaf tree per
  // round for all targets, DESIGN.md 2 item 19; only with T > 1 targets, ignored otherwise)
  int multi_strategy = 0;
  // process_type=update with updater=refresh (DESIGN.md 2 item 20): the rounds refresh the trees of an existing model
  // instead of growing new ones; refresh_leaf = false keeps their leaf values
  bool update_mode = false, refresh_leaf = true;
  std::string updater;
  bool use_cols() const { return colsample_bytree < 1.0f || colsample_bylevel < 1.0f || colsample_bynode < 1.0f; }
  bool vector_leaf() const { return multi_strategy == 1 && num_target > 1; }
};

// What an objective is on the host: one row of params.cu kObjectives per accepted name (DESIGN.md 4.4)
enum ObjLink { kLinkIdentity, kLinkSigmoid, kLinkExp, kLinkSoftmax };
enum ObjGrad { kGradScalar, kGradSoftprob, kGradAft, kGradRank, kGradQuantile };
enum ObjLabels { kLabelsDomain, kLabelsBounds, kLabelsRank };
enum ObjIntercept { kInterceptStump, kInterceptQuantile, kInterceptFixed, kInterceptNone };
struct Objective {
  const char* name;
  B2Objective id;
  ObjLink link;
  ObjGrad grad;
  float Params::*param;   // the gradient kernel's parameter, nullptr: none
  bool multi_target, checks_finite;
  ObjLabels labels;
  ObjIntercept intercept;
  const char* label_rule = nullptr;   // kLabelsDomain: fail() format taking the objective's name and num_class
};
const Objective& objective_row(const Params& p);

// An eval_metric name (params.cu kMetrics); the family picks eval_metric's rules, launch and finish
enum MetricFamily { kEvalElementwise, kEvalClass, kEvalAuc, kEvalAft, kEvalQuantile, kEvalRank };
struct Metric { const char* name; B2Metric id; MetricFamily family; bool multi_target; };

struct TreeHost {
  std::vector<int32_t> left, right, parent, feature, split_bin;
  std::vector<float> cond, value, base_weight, loss_chg;
  std::vector<double> sum_hess;
  std::vector<uint8_t> default_left;
  std::vector<uint8_t> split_type;        // 1 = categorical split
  std::vector<uint32_t> cat_bits;         // [n][8] categories that go right (all zero for numeric nodes)
  // vector-leaf tree: [n][T] -- a leaf's values, an internal node's eta-scaled weights (empty for a scalar tree)
  std::vector<float> leaf_vec;
  bool any_cat = false;
  int add(int par) {
    int id = (int)left.size();
    left.push_back(-1); right.push_back(-1); parent.push_back(par); feature.push_back(-1); split_bin.push_back(-1);
    cond.push_back(0.f); value.push_back(0.f); base_weight.push_back(0.f); loss_chg.push_back(0.f); sum_hess.push_back(0.0);
    default_left.push_back(0); split_type.push_back(0); cat_bits.insert(cat_bits.end(), 8, 0u);
    return id;
  }
  int size() const { return (int)left.size(); }
};


struct Timers {
  double hist_ms = 0, round_ms = 0;
  double shap_ms = 0;   // kernel time of pred_contribs / pred_interactions (CUDA events around the SHAP kernels)
  long long shap_rows = 0;
  double refresh_ms = 0;   // update mode: refresh_kernel time (CUDA events around every launch)
  long long refresh_launches = 0;
  // B2_BoosterSetParam changed a value the tree graphs bake in: host time of re-capturing a tree and applying it to its
  // graph (cudaGraphExecUpdate), and how often the update was refused and the graph instantiated again instead
  double graph_update_ms = 0;
  long long graph_updates = 0, graph_reinstantiations = 0;
  double phase_ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // profile=2: quant, hist, allreduce, subtract, eval+decide, partition+finalize, leaf, other
  long long hist_launches = 0, hist_rows = 0, kernel_launches = 0, rounds = 0;
  double hist_bytes = 0, allreduce_bytes = 0;
  void reset() { *this = Timers(); }
};

struct EvalCache { DevBuf<float> margin; int n_trees_applied = 0; int64_t n = 0; uint64_t margin_version = 0; uint64_t weights_version = 0; };

// per-group descending order of a row vector (rank_kernel.cu b2_rank_order): keys_sorted / rows hold, for every model
// position, the sort key (the value) and the row.  The buffers are pooled and kept, so a booster sorts its train margins
// every round without allocating.
struct RankOrder {
  DevBuf<int32_t> iota, rows; DevBuf<uint32_t> keys, keys_sorted; DevBuf<uint8_t> temp;
  int64_t n = -1, groups = -1; size_t temp_bytes = 0;
  void run(Matrix* m, const float* v, int num_sms, cudaStream_t s) {
    if (n != m->n || groups != m->n_qgroups) {
      const size_t rows_cap = (size_t)std::max<int64_t>(m->n, 1);
      iota.ensure(rows_cap); rows.ensure(rows_cap); keys.ensure(rows_cap); keys_sorted.ensure(rows_cap);
      temp_bytes = b2_rank_order_temp_bytes(m->n, m->n_qgroups);
      temp.ensure(std::max<size_t>(temp_bytes, 1));
      LAUNCH_CHECK(b2_launch_rank_iota(iota.p, m->n, num_sms, s));
      n = m->n; groups = m->n_qgroups;
    }
    LAUNCH_CHECK(b2_rank_order(v, m->n, m->qgroup_ptr.p, m->n_qgroups, iota.p, keys.p, keys_sorted.p, rows.p, temp.p,
                               temp_bytes, num_sms, s));
  }
};

struct Booster : HandleBase {
  Ctx* ctx = nullptr;
  Params p;
  Matrix* train = nullptr;
  int n_features = 0;
  Comm* comm = nullptr;
  std::vector<TreeHost> trees;
  std::atomic<bool> cancel{false};
  // device model cache for prediction
  // d_trees_synced / paths_synced: the number of trees a cache was built from, -1 = stale (trees_edited)
  DevBuf<B2TreeNodeDev> d_nodes; DevBuf<int32_t> d_tree_offset; int d_trees_synced = 0;
  std::vector<B2TreeNodeDev> h_nodes; std::vector<int32_t> h_tree_offset;
  DevBuf<uint32_t> d_cat_table; std::vector<uint32_t> h_cat_table;   // [categorical nodes][8]
  // TreeSHAP path table (build_paths), rebuilt when the tree set changes
  DevBuf<B2PathElem> d_path_elems; DevBuf<B2PathInfo> d_paths; DevBuf<uint32_t> d_path_cats;
  std::vector<int32_t> tree_path_offset;   // [trees + 1]: paths of tree t are [offset[t], offset[t+1])
  std::vector<double> tree_expected;       // [trees] cover-weighted mean of the leaves (the tree's SHAP bias)
  int paths_synced = -1;
  // training state
  bool margin_ready = false;
  DevBuf<float> margin;          // [n][K]
  DevBuf<float2> gh;             // [K][n]
  DevBuf<float2> gh_round;       // copy of the round's gradients (num_parallel_tree > 1 with row sampling)
  DevBuf<int2> q;                // [n]
  DevBuf<int32_t> ridx[2];
  DevBuf<long long> hist[2];
  DevBuf<long long> hist_scratch;  // b2_hist_scratch_elems of a level's histogram build (launch_hist)
  // Everything a peer maps lives in ONE allocation (one cudaIpc handle per peer instead of four): the build buffer, the
  // candidate table, the misc table and the flag words are views into it
  template <typename T> struct View { T* p = nullptr; };
  DevBuf<uint8_t> xarena;
  size_t xoff_cands = 0, xoff_misc = 0, xoff_flags = 0, x_misc_stride = 0;
  View<long long> hist_build;       // reduce-scatter send buffer [shards][node_cap][slice] (only when shards > 1)
  View<B2SplitCand> d_cands_all;    // candidates of all ranks [shards][nodes][cpn]
  int shards = 1, log2_shards = 0, sp = 32, cpn = 1;   // cpn = most candidates per node of a level (numeric CTAs + categorical CTAs)
  int cpn_num = 1;
  View<uint32_t> t_cat;                    // [max_nodes][8] category sets of the tree being grown (in t_block)
  DevBuf<uint8_t> d_col_masks;             // [max_depth][F] level feature sets of the tree being grown (column sampling)
  // interaction constraints (B2Interaction): set membership of every feature, fixed for the booster, and the sets
  // compatible with each node's path in the tree being grown (written by decide)
  DevBuf<unsigned long long> d_ic_sets_of, d_ic_compat;
  int ic_words = 0;                        // 0 = no constraints
  // NVLink peer-memory exchange (p2p.cuh, p2p_exchange.cu): on when every rank mapped its peers; B2_EXCHANGE=nccl keeps NCCL
  struct P2PState {
    bool enabled = false, tried = false;
    B2P2P pp;
    DevBuf<uint32_t> words;               // [kP2PSlots] epoch, [kP2PSlots] done, err, local abort stand-in (never mapped by peers)
    uint32_t* flags = nullptr;            // views into Booster::xarena
    long long* misc = nullptr;            // [world][misc_stride]
    std::vector<void*> opened;
    int cand_cap = 0;
  } p2p;
  // CUDA graphs of the per-tree launch sequence, one per class tree of a round (grow_tree is sync-free and its
  // arguments are the same for every tree, so the sequence is captured once and replayed; B2_BoosterSetParam marks them
  // stale when it changes an argument, and run_tree captures the sequence again and updates the graph in place)
  struct TreeGraph {
    cudaGraphExec_t exec = nullptr;
    bool stale = false;                    // B2_BoosterSetParam changed a kernel argument baked into it (run_tree)
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> hist_ev;   // owned; recorded by the graph (external event nodes)
    long long hist_launches = 0, kernel_launches = 0;
    double allreduce_bytes = 0;
  };
  // Everything a round writes on the host side while it runs: the pinned read-back blocks of its trees, its timing
  // events and the tree graphs whose copy and event-record nodes point at them.  Two sets alternate by round parity, so
  // that round r+1 is enqueued while round r's blocks and events are still unread (boost_round, drain_round).
  struct RoundBuffers {
    std::vector<void*> staging;            // pinned host copies of finished trees, one per class tree of a round
    std::map<int, TreeGraph> graphs;       // per class slot
    std::vector<cudaEvent_t> ev_pool; size_t ev_used = 0;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> hist_events;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> refresh_events;   // update mode: around every refresh_kernel
    std::vector<std::pair<int, cudaEvent_t>> phase_marks;   // (phase that ENDS at this event)
    cudaEvent_t start = nullptr, stop = nullptr;
    uint32_t* h_p2p_err = nullptr;         // pinned copy of the peer-memory error word, written at the end of the round
    std::vector<float> dart_w;             // DART: the weights once this round is committed (trees before it + its own)
    bool dart_dropped = false;             // the round changed weights of earlier trees
    void* vstaging = nullptr;              // vector-leaf tree: pinned copy of the round's d_vblock
    size_t vstaging_bytes = 0;
    bool refresh = false;                  // update mode: the round refreshed the trees to_update[rsrc[slot]]
    std::vector<void*> rstaging;           // pinned copies of their read-back blocks (refresh_nodes_kernel)
    std::vector<int> rsrc;
  };
  RoundBuffers rb[2];
  int rb_cur = 0;                          // parity of the next round to enqueue
  int pending_trees = 0;                   // trees of the enqueued round not drained yet (in rb[rb_cur ^ 1]); 0 = none
  bool pending_check_finite = false;       // that round's gradient kernel reports non-finite pairs into h_grad_err
  std::map<int, int> direct_trees;         // trees grown with direct launches per class slot (the first one allocates)
  bool graph_failed = false;
  bool absmax_fused = false;               // this round's gradient kernel already produced d_absmax[k]
  bool labels_checked = false;             // the train labels are inside the objective's domain (check_labels)
  bool gh_ready = false;                   // gh holds the gradient pairs of a round (B2_BoosterGetGradients)
  DevBuf<uint32_t> d_grad_err;             // set by the gradient kernel when a gradient pair is not finite
  uint32_t* h_grad_err = nullptr;          // pinned copy, written at the end of the round's stream work
  DevBuf<uint16_t> pos;                    // [n] leaf index of every row (final_assign / leaf_sums -> margin_update)
  size_t slice_elems = 0;
  size_t node_elems = 0;
  DevBuf<uint32_t> d_absmax; DevBuf<int32_t> d_qexp;
  // device-resident control tables of the sync-free level loop (control_kernel.cu)
  int ctl_depth = 0;                       // max_depth the tables are sized for
  // the tree being grown, laid out as its pinned read-back block (TreeLayout) so that one copy brings it back
  DevBuf<uint8_t> t_block;
  View<int32_t> t_i32;                     // 7 int32 arrays [max_nodes] + n_nodes + n_leaves
  View<float> t_f32;                       // loss_chg, leaf_weight, leaf_value [max_nodes]
  View<long long> t_i64;                   // sum_g, sum_h [max_nodes] + level_rows [max_depth+1]
  View<int32_t> t_qexp;                    // the tree's quantisation exponents (written by leaf_values_kernel)
  DevBuf<B2LevelCtl> d_ctl;                // [0],[1] level ping-pong, [2] leaf pass
  DevBuf<B2NodeSeg> d_seg[2]; DevBuf<B2EvalNode> d_ev[2];
  DevBuf<B2HistWork> d_hist_work; DevBuf<B2SplitWork> d_split_work; DevBuf<B2SegWork> d_seg_work;
  DevBuf<B2SplitCand> d_cands; DevBuf<int32_t> d_counters, d_triples, d_pair_parent;
  DevBuf<uint32_t> d_part_done;            // CTAs of a partition that finished (zero between launches: the last resets it)
  DevBuf<uint32_t> d_eval_done;            // CTAs of a split scan that finished when it decides the level (same rule)
  DevBuf<B2SplitCand> d_cand_best;         // [nodes of a level] decide's winner of every node
  DevBuf<B2LeafDev> d_leaves;
  DevBuf<long long> d_leaf_sums; DevBuf<float> d_leaf_values; DevBuf<double> d_metric;
  size_t staging_bytes = 0;                // bytes of every block in rb[].staging
  DevBuf<float> d_custom_g, d_custom_h;
  std::map<uint64_t, EvalCache*> eval_cache;   // keyed by Matrix::uid
  // learning to rank: the train margins' order (every round), the discount table ln2 / log(r + 2) (grown to the largest
  // group seen), 1/IDCG of the train groups (keyed by matrix, its rank_version, k and the gain) and the stage of the
  // groups larger than the gradient kernel's shared-memory stage (with rank:map also its hit prefixes A and counts R)
  RankOrder rank_order;
  DevBuf<double> rank_disc; int64_t rank_disc_len = 0;
  DevBuf<double> rank_inv_idcg; uint64_t idcg_uid = 0, idcg_version = 0; int idcg_k = -1, idcg_gain = -1;
  DevBuf<float> rank_scratch_m, rank_scratch_y; DevBuf<double> rank_scratch_p;
  DevBuf<double> rank_scratch_a; DevBuf<int32_t> rank_scratch_r;
  // DART: the weight of every committed tree (empty for gbtree).  weights_version changes whenever weights of existing
  // trees change (a round that dropped trees, B2_BoosterSetTreeWeights): margins cached from the old weights are stale.
  std::vector<float> tree_w;
  uint64_t weights_version = 0;
  DevBuf<float> d_tree_w; uint64_t d_tree_w_version = ~0ull; size_t d_tree_w_count = 0;   // device copy for prediction
  int paths_weights_version = -1;
  // The next round's drop decision, taken before its gradients (dart_prepare): r = its round number, dropped[t] for the
  // T trees before it, w_after = the weights once it is committed (T old + its new trees).  With drops, dart_drop holds
  // its drop margin (the gradients' margin) and dart_prefix the full-margin prefix under the new weights.
  struct DartNext {
    int64_t r = -1;
    std::vector<uint8_t> dropped;
    std::vector<float> w_after;
    int n_dropped = 0;
  } dart_next;
  DevBuf<float> dart_drop, dart_prefix, d_dart_w_old, d_dart_w_full, d_dart_w_new;
  DevBuf<uint8_t> d_dart_dropped;
  // reg:quantileerror: the alphas on the device, and the leaf refresh's digit histograms (zero between passes) and
  // per-leaf selection state (quantile_kernel.cu).  refresh_leaves: the round being enqueued refreshes its leaves (a
  // custom objective's rounds keep their Newton leaves).
  DevBuf<float> d_alpha;
  DevBuf<unsigned long long> d_qhist; DevBuf<uint8_t> d_qsel; DevBuf<int32_t> d_one;
  bool refresh_leaves = false;
  // vector-leaf trees (grow_vector_tree): T-target level histograms [2][T][half][slice], 40-bit leaf sums [T][leaf][4],
  // leaf values [leaf][T], and the read-back block d_vblock (VectorLayout: node totals, node vectors, exponents)
  DevBuf<long long> d_vhist[2], d_vsums;
  DevBuf<float> d_leaf_vec;
  DevBuf<uint8_t> d_vblock;
  DevBuf<float> d_leaf_table; std::vector<float> h_leaf_table;   // prediction: [model nodes][T]
  // update mode (refresh_round): the trees added before the first round are moved out of the model into to_update, and
  // their device copy is built once (nodes with the compact leaf index in pad, category sets, node ids by depth)
  struct RefreshTree { int32_t node_off, n_nodes, n_leaves, order_off, level_off, n_levels; size_t block_bytes; };
  std::vector<TreeHost> to_update;
  std::vector<RefreshTree> rtrees;
  bool update_started = false;
  DevBuf<B2TreeNodeDev> d_rnodes; DevBuf<uint32_t> d_rcats; DevBuf<int32_t> d_rorder, d_rlevels;
  DevBuf<long long> d_rsums, d_rlimbs; DevBuf<float> d_rleaf; DevBuf<uint8_t> d_rblock;
  size_t rstaging_bytes = 0;               // bytes of every block in rb[].rstaging (the largest tree's)
  // profiling
  Timers t;
  // the one teardown of a tree graph: its executable graph and the events its nodes record
  static void destroy_graph(TreeGraph& g) {
    if (g.exec) cudaGraphExecDestroy(g.exec);
    for (auto& pr : g.hist_ev) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
    g.exec = nullptr; g.hist_ev.clear();
  }
  ~Booster() {
    // (a pending round is not drained: the stream synchronisation below waits for it and its trees are dropped)
    for (auto& r : rb)
      for (auto& kv : r.graphs) destroy_graph(kv.second);
    // No barrier with the peers here: a peer touches this rank's arena only inside the exchange kernels of a round, and
    // every one of those accesses happens-before a flag that this rank waited for before ITS round completed -- once the
    // last round is synchronised the arena is quiescent.  (A barrier in the destructor made a rank whose peer keeps its
    // Booster alive -- the rank that returns the model -- spin until the peer-wait timeout: 23 s per train() call.)
    if (ctx) cudaStreamSynchronize(ctx->stream);
    for (void* q : p2p.opened) cudaIpcCloseMemHandle(q);
    for (auto& r : rb) {
      for (auto e : r.ev_pool) cudaEventDestroy(e);
      if (r.start) cudaEventDestroy(r.start);
      if (r.stop) cudaEventDestroy(r.stop);
      for (void* h : r.staging) cudaFreeHost(h);
      if (r.h_p2p_err) cudaFreeHost(r.h_p2p_err);
      if (r.vstaging) cudaFreeHost(r.vstaging);
      for (void* h : r.rstaging) cudaFreeHost(h);
    }
    for (auto& kv : eval_cache) delete kv.second;
    if (h_grad_err) cudaFreeHost(h_grad_err);
  }
};

// ---------------------------------------------------------------- params.cu
void set_targets(Params* p, int T);
void parse_params(const char* text, Params* p, int* max_bin_out);
Params changed_params(const Params& live, const char* text);
float base_margin_value(const Params& p);
float h_calc_weight(const Params& p, double G, double H);
const Metric& metric_id(const char* name, const Params& p, float* param, int* minus);

// ---------------------------------------------------------------- tree.cu
void check_level_memory(const Booster* b);
void ensure_quantile_buffers(Booster* b, int max_leaves);
int quantile_select(Booster* b, int k, const uint16_t* pos, const float* margin, const float2* gh, const int32_t* qexp,
                    const int32_t* n_leaves, int max_leaves, float eta, const B2LeafDev* leaves, float* leaf_value,
                    float* tree_value);
B2CtlParams ctl_params(const Params& p);
void tree_params_changed(Booster* b, const Params& old);
void run_tree(Booster* b, int k, int slot);
void materialize_tree(Booster* b, const void* block);
void materialize_vector_tree(Booster* b, const void* block, const void* vblock);
void sync_device_trees(Booster* b);
// B2_BoosterAddTree: fails unless tree t can be appended to b's model (every walk from the root ends at a leaf, the
// split features exist, the leaf vector fits b's kind of tree); names the tree, the node and the value
void check_tree(const Booster* b, const TreeHost& t);
// B2_HistBuildRaw*: one histogram of m's rows ridx[0..n_sel) (nullptr: rows 0..n_sel) from the pairs (qg, qh) into out
// [F][256][2]; chunk_rows <= 0 and window_rows <= 0 take 2048 and 4096, chunk_rows is capped at window_rows
void hist_build_raw(Matrix* m, const int32_t* qg, const int32_t* qh, const int32_t* ridx, int64_t n_sel, int window_rows,
                    int chunk_rows, int64_t* out, float* kernel_ms);

// ---------------------------------------------------------------- round.cu
cudaEvent_t get_event(Booster* b);
void mark_phase(Booster* b, int phase);
void init_margin(Booster* b, float* margin, Matrix* m);
void ensure_rank_disc(Booster* b, int64_t len);
void drain_round(Booster* b);
void ensure_train_margin(Booster* b);
void dart_prepare(Booster* b);
Booster* new_booster(const char* params, Matrix* m, Comm* comm);
void set_booster_params(Booster* b, const char* params);
void boost_round(Booster* b, const float* custom_g, const float* custom_h, int64_t len);

// ---------------------------------------------------------------- predict.cu
// an existing tree changed: every cache derived from b->trees is stale (-1, never a tree count; appends are incremental)
void trees_edited(Booster* b);
void build_paths(Booster* b);
void predict_trees(Booster* b, Matrix* m, int tree_begin, int tree_end, float* out);
float* eval_margin(Booster* b, Matrix* m);
double eval_metric(Booster* b, Matrix* m, const char* name);
// B2_BoosterPredict, B2_BoosterPredictContribs, B2_BoosterPredictLeaf: tree_end <= 0 means every tree
void predict(Booster* b, Matrix* m, bool output_margin, int tree_begin, int tree_end, float* out, int64_t out_len);
void predict_contribs(Booster* b, Matrix* m, int tree_begin, int tree_end, bool interactions, float* out, int64_t out_len);
void predict_leaf(Booster* b, Matrix* m, int tree_begin, int tree_end, float* out, int64_t out_len);

}  // namespace b2host
