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
/* process-wide engine options (the environment variables of the same name in upper case with a B2_ prefix are their
 * defaults): "hist_narrow" = "0" | "1" -- feature-group layout of matrices quantised from now on (DESIGN.md 4.1). */
int B2_SetOption(const char* key, const char* value);
int B2_DeviceCount(int* out);

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
 * matrix.  ref != 0 reuses the cuts of an already quantised matrix.  keep_raw == 0 frees the
 * device copy of the float data afterwards (it is needed again only for Predict on this matrix). */
int B2_MatrixQuantize(B2Handle m, B2Handle comm, int32_t max_bin, B2Handle ref, int32_t keep_raw);
/* Quantise with GIVEN cut points (no sketch, no communication): a restart after an actor failure continues with the
 * cuts of the first attempt even when the world size changed, so old and new trees split on the same bins
 * (xgboost_ray/elastic.py:19-178, main.py:1644-1713; SURVEY.md 5 "freeze cuts from attempt 0"). */
int B2_MatrixQuantizeWithCuts(B2Handle m, const int32_t* ptrs /*[F+1]*/, const float* vals, const float* mins /*[F]*/,
                              const uint8_t* has_missing /*[F]*/, int32_t max_bin, int32_t keep_raw);
/* re-upload the float data of a matrix whose device copy was freed (same shape) */
int B2_MatrixEnsureRaw(B2Handle m, const float* data);
int B2_MatrixCutsSize(B2Handle m, int32_t* total_cuts);
int B2_MatrixGetCuts(B2Handle m, int32_t* ptrs /*[F+1]*/, float* vals /*[total]*/, float* mins /*[F]*/,
                     uint8_t* has_missing /*[F]*/);
int B2_MatrixGetBins(B2Handle m, uint8_t* out /*[n_rows*n_cols] dense row-major*/);
int B2_MatrixFree(B2Handle m);

/* ---- booster: replaces xgb.train(...) at xgboost_ray/main.py:745-752 (one UpdateOneIter per
 * boosting round of its loop; callbacks stay in Python) and model.predict(...) at main.py:804.
 * params: newline-separated "key=value" lines using XGBoost parameter names (objective, num_class,
 * max_depth, eta, gamma, min_child_weight, lambda, alpha, max_bin, base_score, hist_qbits,
 * eval_metric).  train must be quantised.  comm may be 0. */
int B2_BoosterCreate(const char* params, B2Handle train, B2Handle comm, B2Handle* out);
int B2_BoosterUpdateOneIter(B2Handle b, int32_t iter);
/* custom objective (xgb.train(obj=...), tests/test_xgboost_api.py:77-102): grad/hess [n_rows*num_class] */
int B2_BoosterBoostOneIter(B2Handle b, const float* grad, const float* hess, int64_t len);
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
/* copy of the training-set margin cache (what the next round's gradient is taken at) */
int B2_BoosterGetTrainMargin(B2Handle b, float* out, int64_t out_len);
/* (re)initialise the training margin cache from base_margin/base_score plus all current trees
 * (continuation from xgb_model=, main.py:1211-1220); needs the raw data of the train matrix */
int B2_BoosterResetTrainMargin(B2Handle b);
/* base_score of the model (probability space for binary:logistic).  When the params carried no base_score it is
 * estimated from the labels of all workers before the first tree (xgboost >= 2.0 behaviour, SURVEY.md A.3);
 * is_final = 0 until that has happened. */
int B2_BoosterGetBaseScore(B2Handle b, float* out, int32_t* is_final);
int B2_BoosterNumTrees(B2Handle b, int32_t* out);
int B2_BoosterTreeNumNodes(B2Handle b, int32_t tree, int32_t* out);
int B2_BoosterGetTree(B2Handle b, int32_t tree, int32_t* left, int32_t* right, int32_t* parent,
                      int32_t* split_feature, int32_t* split_bin, float* split_cond, uint8_t* default_left,
                      float* value, float* base_weight, float* loss_chg, double* sum_hess);
int B2_BoosterAddTree(B2Handle b, int32_t n_nodes, const int32_t* left, const int32_t* right,
                      const int32_t* parent, const int32_t* split_feature, const int32_t* split_bin,
                      const float* split_cond, const uint8_t* default_left, const float* value,
                      const float* base_weight, const float* loss_chg, const double* sum_hess);
/* categorical part of a tree (model JSON fields split_type / categories*, SURVEY.md 8f row f1): split_type[i] = 1
 * for a categorical split; cat_bits[i*8 + (c >> 5)] bit (c & 31) set = category c goes RIGHT.  Set* is called
 * after B2_BoosterAddTree when a model with categorical splits is loaded. */
int B2_BoosterGetTreeCategories(B2Handle b, int32_t tree, uint8_t* split_type /*[n]*/, uint32_t* cat_bits /*[n*8]*/);
int B2_BoosterSetTreeCategories(B2Handle b, int32_t tree, const uint8_t* split_type, const uint32_t* cat_bits);
/* JSON object with accumulated device timings / counters of the hot path (since last reset):
 * hist_ms, hist_launches, hist_rows, hist_bytes, kernel_launches, round_ms, allreduce_bytes ... */
int B2_BoosterGetTimers(B2Handle b, int32_t reset, char* out, int64_t out_cap);
int B2_BoosterCancel(B2Handle b);
int B2_BoosterFree(B2Handle b);

/* ---- kernel-level entry used by the parity tests and the roofline probe: histogram of `n_sel`
 * rows (ridx, or all rows when ridx == NULL) of a dense uint8 matrix; out [n_cols][256][2] int64.
 * window_rows bounds the rows a CTA accumulates in int32 before flushing. */
int B2_HistBuildRaw(const uint8_t* bins, int64_t n_rows, int32_t n_cols, const int32_t* qg, const int32_t* qh,
                    const int32_t* ridx, int64_t n_sel, int32_t window_rows, int32_t chunk_rows, int device,
                    int64_t* out, float* kernel_ms /* may be NULL */);

#ifdef __cplusplus
}
#endif
#endif /* B2HIST_H_ */
