/*
 * b2hist.h -- C ABI of libb2hist.so: the H100-native (sm_90a) histogram-tree training engine.
 *
 * This is the drop-in boundary for the hot path that the reference (ray-project/xgboost_ray)
 * delegates to the third-party `xgboost` package.  Each entry point names the reference call
 * site(s) it replaces (paths relative to /root/reference).  The reference is pure Python, so the
 * binding a maintainer adds is a ctypes stub (INTEGRATION.md); xgboost_ray_b200/engine.py is it.
 *
 * Conventions (modelled on XGBoost's C API): every function returns 0 on success, -1 on failure
 * with the message available from B2_GetLastError(); handles are opaque; all pointers are HOST
 * pointers unless a parameter says otherwise; the caller owns input buffers (the engine copies)
 * and output buffers (caller-allocated).  Calls may be made from any thread (the engine sets the
 * CUDA device per call; the reference runs training on a non-main thread, main.py:774-776).
 * There is no CPU fallback: without a CUDA device every compute entry point fails.
 */
#ifndef B2HIST_H_
#define B2HIST_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef uint64_t B2Handle;

const char* B2_GetLastError(void);
int B2_GetVersion(void);
int B2_DeviceCount(int* out);
/* Check the params text of B2_BoosterCreate without a device: the same parsing and every rule about which parameters go
 * together.  The rules that need the label width apply when the text gives num_target=<T>; what needs the train matrix
 * itself (feature count, categorical features) does not.  A broken rule fails with B2_BoosterCreate's message. */
int B2_CheckParams(const char* params);

/* ---- communicator: replaces the Rabit bridge.
 * xgboost_ray/main.py:256-283 (_start_rabit_tracker -> rabit_args env) becomes B2_GetUniqueId on
 * the driver; xgboost_ray/main.py:308-324 + use site :724 (_RabitContext.__enter__/__exit__ ->
 * xgboost.collective.init/finalize) become B2_CommCreate / B2_CommFree on each actor;
 * B2_CommAbort is what the stop path (main.py:777-781) calls so a blocked collective returns;
 * xgboost_ray/session.py:68-75 (get_rabit_rank) becomes B2_CommRank. */
int B2_GetUniqueId(uint8_t out[128]);
int B2_CommCreate(const uint8_t uid[128], int rank, int world, int device, B2Handle* out);
int B2_CommRank(B2Handle comm, int* rank, int* world);
/* host-side allreduce of a few doubles over the communicator (xgb.collective.allreduce; xgboost averages custom
 * metric values over the workers with it, python-package callback.py _allreduce_metric).  op: 0 sum, 1 max, 2 min.
 * comm == 0 or a single-process communicator: identity. */
int B2_CommAllReduce(B2Handle comm, double* inout, int32_t n, int32_t op);
int B2_CommAbort(B2Handle comm);
int B2_CommFree(B2Handle comm);

/* ---- matrix: replaces xgb.DMatrix / xgb.QuantileDMatrix / xgb.DeviceQuantileDMatrix construction
 * in RayXGBoostActor._get_dmatrix, xgboost_ray/main.py:379-445 (sites :386, :418, :437, set_info
 * :439-442, get_label().size :727). */
int B2_MatrixCreateFromDense(const float* data, int64_t n_rows, int32_t n_cols, float missing, int device,
                             B2Handle* out);
/* A shard that arrives as several row blocks (the reference's RayDataIter hands xgb.DeviceQuantileDMatrix one block
 * per Ray object / file, xgboost_ray/matrix.py:127-196, main.py:387-418): allocate the device matrix once, then
 * upload each block at its row offset -- no host-side concatenation (matrix.py:65-67). */
int B2_MatrixCreate(int64_t n_rows, int32_t n_cols, float missing, int device, B2Handle* out);
/* A scipy.sparse matrix (xgb.DMatrix(csr), reached through xgboost_ray/main.py:437): row i stores entries
 * [indptr[i], indptr[i+1]) of indices / values; an entry a row does not store is missing, a stored one follows the
 * dense rules (NaN or `missing` is missing).  indptr is only read.  The arrays are checked on the device: indptr[0] = 0,
 * indptr non-decreasing, indptr[n_rows] = nnz, every column in [0, n_cols) and strictly increasing within its row; the
 * first row that breaks a rule fails the call and is named.  The device keeps the CSR (8 (n_rows + 1) + 8 nnz bytes),
 * never an n_rows x n_cols float copy: the kernels that read raw rows get them densified tile by tile.  Bins, cuts,
 * models and predictions equal those of the dense matrix with NaN in every absent cell. */
int B2_MatrixCreateFromCSR(int64_t* indptr, const int32_t* indices, const float* values, int64_t n_rows, int32_t n_cols,
                           int64_t nnz, float missing, int device, B2Handle* out);
int B2_MatrixSetRows(B2Handle m, int64_t row_begin, const float* data, int64_t n_rows);
/* The shard lives in ANOTHER process (the driver that holds the user's matrix): rows of n_cols floats, remote_row_stride
 * bytes apart starting at remote_addr in process `pid`, are read with process_vm_readv straight into the pinned upload
 * buffers -- the hand-off the reference does through the Ray object store (ray.put per shard, xgboost_ray/matrix.py:
 * 471-484, fetched in main.py:654-670) without ever materialising the shard on the host a second time.  Needs ptrace
 * permission on `pid` (same user; the driver allows its actors with prctl(PR_SET_PTRACER)); fails with a message
 * otherwise and the caller falls back to the shared-memory file hand-off. */
int B2_MatrixCreateFromProcess(int64_t pid, uint64_t remote_addr, int64_t remote_row_stride_bytes, int64_t n_rows,
                               int32_t n_cols, float missing, int device, B2Handle* out);
/* INTERLEAVED sharding (RayShardingMode.INTERLEAVED, xgboost_ray/matrix.py:71-87 / _get_sharding_indices :989-1003: rank r
 * owns rows r, r+W, r+2W, ...) of a matrix that lives in process `pid`, n_total_rows x n_cols floats, C-contiguous at
 * remote_addr.  A strided shard costs every rank a read of the WHOLE matrix span on the host (W-fold amplification), so
 * this COLLECTIVE call (every rank of `comm`, shard_rank == its rank) has rank w read one contiguous 1/W block, stages it
 * in HBM, and a gather kernel pulls the rows each rank owns out of the peers' staged blocks over NVLink (cudaIpc-mapped
 * peer memory).  Result: the same device matrix B2_MatrixCreateFromProcess builds from the strided shard. */
int B2_MatrixCreateFromProcessInterleaved(int64_t pid, uint64_t remote_addr, int64_t n_total_rows, int32_t n_cols,
                                          int32_t shard_rank, B2Handle comm, float missing, int device, B2Handle* out);
/* field: "label" | "weight" | "base_margin" (len n_rows, or n_rows*num_class for base_margin) |
 * "label_lower_bound" | "label_upper_bound" (len n_rows, 0 clears): the survival bounds of each row, read by
 * survival:aft only (lower == upper: exact time; upper = +inf: right-censored; lower = 0: left-censored) */
int B2_MatrixSetFloatInfo(B2Handle m, const char* field, const float* values, int64_t len);
/* label of T = n_targets columns, row-major [rows][T] (xgboost's 2-D label: multi-target regression, multi-label
 * classification; xgboost_ray's list of label columns, matrix.py:308-313, 405-416).  rows must equal the matrix's rows,
 * 1 <= T <= 4096; T = 1 is the same as B2_MatrixSetFloatInfo("label").  T > 1 is refused on a matrix with query
 * groups or survival bounds.  A booster trained on the matrix grows T trees per round, one per column. */
int B2_MatrixSetLabel(B2Handle m, const float* values, int64_t rows, int32_t n_targets);
/* query groups of a ranking matrix (xgb.DMatrix(qid=...) / set_group; the reference sorts rows by qid and ships qid per
 * shard, xgboost_ray/matrix.py:70-100, 300-304, 483, 689 and main.py:371, 399, 431): group g is the next group_sizes[g]
 * rows.  Every size is >= 1 and the sizes sum to the row count; the engine builds the int64 row offsets itself.
 * n_groups = 0 clears the groups.  Read by rank:pairwise / rank:ndcg and the ndcg / map / pre metrics. */
int B2_MatrixSetGroups(B2Handle m, const int32_t* group_sizes, int64_t n_groups);
/* feature types: is_cat[f] != 0 marks feature f categorical (xgb.DMatrix(feature_types=[...'c'...],
 * enable_categorical=True), forwarded by _get_dmatrix, xgboost_ray/main.py:365-376 / matrix.py:159,193).  Must be
 * called before B2_MatrixQuantize.  A categorical value is its category code: an integer in [0, 255]
 * ([0, 254] when the feature has missing values); its bin is the code, its cuts are 0..max code. */
int B2_MatrixSetFeatureTypes(B2Handle m, const uint8_t* is_cat, int32_t len);
int B2_MatrixGetFeatureTypes(B2Handle m, uint8_t* is_cat /*[n_cols]*/);
int B2_MatrixNumRow(B2Handle m, int64_t* out);
int B2_MatrixNumCol(B2Handle m, int32_t* out);
/* GPU quantile sketch (global over `comm`, 0 = single process) + binning into the device uint8
 * matrix.  ref != 0 reuses the cuts of an already quantised matrix; a category code of this matrix
 * that those cuts do not know is then an error (checked over `comm`).  keep_raw == 0 frees the
 * device copy of the float data afterwards (it is needed again only for Predict on this matrix). */
int B2_MatrixQuantize(B2Handle m, B2Handle comm, int32_t max_bin, B2Handle ref, int32_t keep_raw);
/* Quantise with GIVEN cut points (no sketch): a restart after an actor failure continues with the
 * cuts of the first attempt even when the world size changed, so old and new trees split on the same bins
 * (xgboost_ray/elastic.py:19-178, main.py:1644-1713; SURVEY.md 5 "freeze cuts from attempt 0").  A category code
 * the cuts do not know is an error; `comm` (0 = single process) only makes that check global. */
int B2_MatrixQuantizeWithCuts(B2Handle m, B2Handle comm, const int32_t* ptrs /*[F+1]*/, const float* vals,
                              const float* mins /*[F]*/, const uint8_t* has_missing /*[F]*/, int32_t max_bin,
                              int32_t keep_raw);
/* re-upload the float data of a matrix whose device copy was freed (same shape) */
int B2_MatrixEnsureRaw(B2Handle m, const float* data);
/* the same for a matrix created with B2_MatrixCreateFromCSR: re-upload (and check) its CSR arrays (xgboost_ray/main.py:437) */
int B2_MatrixEnsureRawCSR(B2Handle m, int64_t* indptr, const int32_t* indices, const float* values);
/* xgboost's DMatrix.slice(rindex): a new matrix of rows rows[0..n_rows) of m, in that order (duplicates allowed), built
 * on m's device from m's device data: raw values (dense, or CSR kept as CSR), the label ([rows][T]), weight, base_margin
 * ([rows][K]) and label bounds gathered, missing, the feature types and feature_weights copied.  The slice is not quantised
 * and has no query groups: it is sketched with its own cuts like a matrix built from those rows.  m needs its raw data on
 * the device (B2_MatrixEnsureRaw / EnsureRawCSR) and is not changed.  n_rows >= 1, every index in [0, m's rows); rows is
 * only read. */
int B2_MatrixSlice(B2Handle m, int64_t* rows, int64_t n_rows, B2Handle* out);
/* device bytes the matrix owns: the capacities of its raw (dense or CSR), bin and info buffers (xgboost_ray/main.py:437) */
int B2_MatrixDeviceBytes(B2Handle m, int64_t* out);
int B2_MatrixCutsSize(B2Handle m, int32_t* total_cuts);
int B2_MatrixGetCuts(B2Handle m, int32_t* ptrs /*[F+1]*/, float* vals /*[total]*/, float* mins /*[F]*/,
                     uint8_t* has_missing /*[F]*/);
/* dense (n_rows, n_cols) bins; a matrix with the CSR bin layout is densified on the device (absent entries: 255) */
int B2_MatrixGetBins(B2Handle m, uint8_t* out /*[n_rows*n_cols] dense row-major*/);
/* bin layout, set before B2_MatrixQuantize.  DENSE: two n_rows x n_cols byte copies of the bins (row- and
 * feature-major).  CSR (a matrix created with B2_MatrixCreateFromCSR only): one bin per stored entry, aligned with the
 * CSR's indices, which stay on the device with indptr; training reads them instead (DESIGN.md 2 item 26), and the
 * model is byte-identical to the dense layout's.  AUTO (the default): CSR for a CSR matrix whose two dense copies would
 * take more than half of the device's memory, otherwise DENSE.  A slice takes the layout of its parent. */
enum { B2_BIN_LAYOUT_AUTO = 0, B2_BIN_LAYOUT_DENSE = 1, B2_BIN_LAYOUT_CSR = 2 };
int B2_MatrixSetBinLayout(B2Handle m, int32_t layout);
int B2_MatrixFree(B2Handle m);

/* ---- booster: replaces xgb.train(...) at xgboost_ray/main.py:745-752 (one UpdateOneIter per
 * boosting round of its loop; callbacks stay in Python) and model.predict(...) at main.py:804.
 * params: newline-separated "key=value" lines using XGBoost parameter names (objective, num_class,
 * max_depth, eta, gamma, min_child_weight, lambda, alpha, max_bin, base_score, hist_qbits,
 * eval_metric).  train must be quantised.  comm may be 0. */
int B2_BoosterCreate(const char* params, B2Handle train, B2Handle comm, B2Handle* out);
/* Change parameters between boosting rounds (xgboost's Booster.set_param during training, e.g. a learning-rate schedule):
 * the same "key=value" lines as B2_BoosterCreate.  eta / learning_rate, gamma / min_split_loss, min_child_weight,
 * lambda / reg_lambda, alpha / reg_alpha, max_delta_step, subsample, colsample_bytree / bylevel / bynode,
 * max_cat_to_onehot and max_cat_threshold take effect from the next round, each checked by its B2_BoosterCreate rule.
 * Any other key the engine knows may only repeat its value (a new one fails, naming the key); unknown keys are ignored.
 * Either every key is applied or, on failure, none.  A round still in flight is finished with the old values first. */
int B2_BoosterSetParam(B2Handle b, const char* params);
int B2_BoosterUpdateOneIter(B2Handle b, int32_t iter);
/* custom objective (xgb.train(obj=...), tests/test_xgboost_api.py:77-102): grad/hess [n_rows*num_class] */
int B2_BoosterBoostOneIter(B2Handle b, const float* grad, const float* hess, int64_t len);
/* update mode (params process_type=update, updater=refresh, refresh_leaf; xgb.train(xgb_model=...) of xgboost's
 * TreeRefresher): the trees added with B2_BoosterAddTree before the first round are the trees to update (the root
 * must reach each of their nodes, and each has at most 65,536 leaves), and the model starts empty.  Call r (0-based) takes round r of them (num_class x num_parallel_tree
 * trees), computes the gradients at the margin of base_score / base_margin plus the rounds already refreshed, re-fits
 * every node's sum_hess, base_weight and loss_chg (and with refresh_leaf the leaf values) on the raw rows of the train
 * matrix, and appends the refreshed trees.  grad / hess == NULL: the objective's gradients, else a custom objective's
 * [n_rows*num_class].  Fails past the model's last round.  B2_BoosterUpdateOneIter / BoostOneIter fail in update mode. */
int B2_BoosterRefreshOneIter(B2Handle b, const float* grad, const float* hess, int64_t len);
/* diagnostic: the fp32 gradient pairs of the last round on the train matrix, class-major ([num_class][n_rows]),
 * as the trees of that round saw them (after the weight, before quantisation).  len = n_rows * num_class. */
int B2_BoosterGetGradients(B2Handle b, float* grad, float* hess, int64_t len);
/* metric value of `m` (the train matrix or a matrix with raw data) under the current model, reduced
 * over comm like xgboost's (sum, wsum) allreduce.  metric: rmse|logloss|error|mlogloss|merror|...|aft-nloglik|
 * interval-regression-accuracy (the last two need survival:aft and the label bounds of `m`) | ndcg[@k][-] |
 * map[@k][-] | pre[@k][-] (need the query groups of `m`: per-group values, (sum, group count) reduced over comm) */
int B2_BoosterEvalSet(B2Handle b, B2Handle m, const char* metric, double* out);
/* out [n_rows*num_class].  tree_end == 0 means all trees.  training == margin cache of train set. */
int B2_BoosterPredict(B2Handle b, B2Handle m, int32_t output_margin, int32_t tree_begin, int32_t tree_end,
                      float* out, int64_t out_len);
/* model.predict(local_data, pred_contribs=True / pred_interactions=True) at main.py:804: exact path-dependent TreeSHAP
 * (xgboost's RegTree::CalculateContributions, cover = the node's sum_hess) in margin space over trees
 * [tree_begin, tree_end) (tree_end == 0: all).  interactions == 0: out [n_rows][num_class][F+1], column F is the bias
 * (the row's base margin plus the cover-weighted mean leaf of every tree in range); interactions != 0:
 * out [n_rows][num_class][F+1][F+1] SHAP interaction values (rows sum to the contributions).  Same checks as
 * B2_BoosterPredict; bit-identical from call to call and for any row sharding. */
int B2_BoosterPredictContribs(B2Handle b, B2Handle m, int32_t tree_begin, int32_t tree_end, int32_t interactions,
                              float* out, int64_t out_len);
/* model.predict(local_data, pred_leaf=True) at main.py:804: out [n_rows][tree_end - tree_begin] = node id (as in the
 * model JSON / get_dump) of the leaf each row reaches in each tree of the range (tree_end == 0: all trees). */
int B2_BoosterPredictLeaf(B2Handle b, B2Handle m, int32_t tree_begin, int32_t tree_end, float* out, int64_t out_len);
/* copy of the training-set margin cache.  full = 0: what the next round's gradient is taken at (booster=dart: that
 * round's drop margin, whose drops B2_BoosterBoostOneIter then keeps); full = 1: the margin of the whole model (the
 * same for gbtree), what predict and the metrics see, without a traversal of the model. */
int B2_BoosterGetTrainMargin(B2Handle b, int32_t full, float* out, int64_t out_len);
/* (re)initialise the training margin cache from base_margin/base_score plus all current trees
 * (continuation from xgb_model=, main.py:1211-1220); needs the raw data of the train matrix */
int B2_BoosterResetTrainMargin(B2Handle b);
/* base_score of the model (probability space for binary:logistic).  When the params carried no base_score it is
 * estimated from the labels of all workers before the first tree (xgboost >= 2.0 behaviour, SURVEY.md A.3);
 * is_final = 0 until that has happened. */
int B2_BoosterGetBaseScore(B2Handle b, float* out, int32_t* is_final);
/* label columns of the model (1 unless it is multi-target): fixed by the train matrix when the booster is created, or by
 * num_target=<T> in params (a loaded model; a train matrix must then have T columns) */
int B2_BoosterNumTargets(B2Handle b, int32_t* out);
int B2_BoosterNumTrees(B2Handle b, int32_t* out);
/* One tree of n_nodes nodes, every array [n_nodes] unless noted.  Node i splits when split_feature[i] >= 0 (rows with
 * x < split_cond, or missing with default_left, go to left[i], the others to right[i]); otherwise it is a leaf of
 * leaf value value[i].  Node 0 is the root; parent[i] is -1 for it.  Categorical part (model JSON split_type /
 * categories*, SURVEY.md 8f row f1): split_type[i] = 1 for a categorical split; cat_bits[i*8 + (c >> 5)] bit (c & 31)
 * set = category c goes RIGHT.  Vector-leaf tree (multi_strategy=multi_output_tree, T = num_target > 1):
 * leaf_vector[i*T + k] is node i's value of target k -- a leaf's leaf value, an internal node's eta-scaled weight
 * (model JSON base_weights) -- and leaf_vector_len = n_nodes * T.  A single-output tree has leaf_vector NULL (or
 * leaf_vector_len 0). */
typedef struct B2Tree {
  int32_t n_nodes;
  int32_t* left;
  int32_t* right;
  int32_t* parent;
  int32_t* split_feature;
  int32_t* split_bin;
  float* split_cond;
  uint8_t* default_left;
  float* value;
  float* base_weight;
  float* loss_chg;
  double* sum_hess;
  uint8_t* split_type;
  uint32_t* cat_bits;     /* [n_nodes * 8] */
  float* leaf_vector;     /* [leaf_vector_len] */
  int64_t leaf_vector_len;
} B2Tree;
int B2_BoosterTreeNumNodes(B2Handle b, int32_t tree, int32_t* out);
/* Fill the caller's arrays with tree `tree`: t->n_nodes must be its node count (B2_BoosterTreeNumNodes), every array
 * is written, and leaf_vector_len must be the tree's leaf vector length (0 for a single-output tree). */
int B2_BoosterGetTree(B2Handle b, int32_t tree, B2Tree* t);
/* Append a whole tree to the model; the arrays are only read.  split_bin, base_weight, loss_chg and sum_hess may be
 * NULL (-1, 0, 0, 0); split_type and cat_bits may be NULL (no categorical split); a leaf vector is given exactly on a
 * booster created with multi_strategy=multi_output_tree.  The tree is refused, naming the tree, the node and the
 * value, when it has no nodes, a split child outside [0, n_nodes), a split node reached twice from the root (a cycle
 * or a shared subtree), a split feature outside the booster's features, a categorical split_type on a leaf, or a leaf
 * vector that does not fit the booster's kind of tree.  Nodes the root does not reach (xgboost's deleted nodes) are
 * allowed. */
int B2_BoosterAddTree(B2Handle b, const B2Tree* t);
/* booster=dart: the weight of every tree in model order (model JSON gradient_booster.weight_drop); tree t adds
 * fl(w[t] * leaf) to the margin.  Get on a gbtree booster returns 1 for every tree.  Set (after the trees were added
 * with B2_BoosterAddTree; a tree added to a dart booster starts at weight 1) needs finite weights >= 0 and one per
 * tree, and makes the train margin rebuild from the new weights. */
int B2_BoosterGetTreeWeights(B2Handle b, float* out, int64_t len);
int B2_BoosterSetTreeWeights(B2Handle b, const float* w, int64_t len);
/* JSON object with accumulated device timings / counters of the hot path (since last reset):
 * hist_ms, hist_launches, hist_rows, hist_bytes, kernel_launches, round_ms, allreduce_bytes ..., and in update mode
 * refresh_ms / refresh_launches: the time and count of refresh_kernel launches (B2_BoosterRefreshOneIter), and
 * graph_update_ms / graph_updates / graph_reinstantiations: the host time of re-capturing a tree whose graph a
 * B2_BoosterSetParam change made stale, the updates of its graph in place, and the updates refused (instantiated anew) */
int B2_BoosterGetTimers(B2Handle b, int32_t reset, char* out, int64_t out_cap);
int B2_BoosterCancel(B2Handle b);
int B2_BoosterFree(B2Handle b);

/* ---- kernel-level entry used by the parity tests and the roofline probe: histogram of `n_sel`
 * rows (ridx, or all rows when ridx == NULL) of a dense uint8 matrix; out [n_cols][256][2] int64.
 * window_rows bounds the rows a CTA accumulates in int32 before flushing. */
int B2_HistBuildRaw(const uint8_t* bins, int64_t n_rows, int32_t n_cols, const int32_t* qg, const int32_t* qh,
                    const int32_t* ridx, int64_t n_sel, int32_t window_rows, int32_t chunk_rows, int device,
                    int64_t* out, float* kernel_ms /* may be NULL */);
/* the same histogram from the CSR bin layout: row i stores bins[indptr[i] .. indptr[i+1]) of the columns in indices
 * (increasing within a row); an absent entry has bin 255.  Rows as for B2_HistBuildRaw; chunk_rows <= 0: 2048. */
int B2_HistBuildRawCSR(int64_t* indptr, const int32_t* indices, const uint8_t* bins, int64_t n_rows, int32_t n_cols,
                       const int32_t* qg, const int32_t* qh, const int32_t* ridx, int64_t n_sel, int32_t chunk_rows,
                       int device, int64_t* out, float* kernel_ms /* may be NULL */);

/* ---- kernel-level entry used by the parity tests: the training path's fixed-point quantisation of n gradient pairs
 * (max |g|, |h| -> frexp exponents -> q = rint(v * 2^(qbits - e))).  out_q [n][2] int32 (qg, qh), out_exp [2]. */
int B2_QuantizeRaw(const float* g, const float* h, int64_t n, int32_t qbits, int device, int32_t* out_q,
                   int32_t* out_exp);

#ifdef __cplusplus
}
#endif
#endif /* B2HIST_H_ */
