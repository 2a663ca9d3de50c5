// launch.h -- the C entry points the kernel files define for the host (engine.cu), and the ids passed through them.
//
// engine.cu and every file that defines one of these functions include this header.  A definition whose parameter list
// differs from its declaration here is then a compile error (two "C" functions of one name) instead of a kernel that
// reads shifted arguments at run time.  A launcher enqueues on the given stream and returns a cudaError_t as int.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "common.cuh"

// objective ids (Params::objective, from the objective name in engine.cu parse_params)
enum B2Objective {
  kObjSquaredError = 0, kObjLogistic = 1, kObjSoftprob = 2, kObjRegLogistic = 3, kObjLogitRaw = 4, kObjSquaredLog = 5,
  kObjPseudoHuber = 6, kObjPoisson = 7, kObjGamma = 8, kObjTweedie = 9, kObjAft = 10, kObjRankPairwise = 11,
  kObjRankNdcg = 12, kObjQuantile = 13, kObjRankMap = 14
};

// eval_metric ids (engine.cu metric_id).  Kernels test some of them as ranges, so the order is part of the meaning.
enum B2Metric {
  kMetricRmse = 0, kMetricLogloss = 1, kMetricError = 2, kMetricMlogloss = 3, kMetricMerror = 4, kMetricMae = 5,
  kMetricAuc = 6, kMetricRmsle = 7, kMetricMape = 8, kMetricMphe = 9, kMetricPoissonNloglik = 10,
  kMetricGammaNloglik = 11, kMetricGammaDeviance = 12, kMetricTweedieNloglik = 13, kMetricAftNloglik = 14,
  kMetricIntervalAccuracy = 15, kMetricNdcg = 16, kMetricMap = 17, kMetricPre = 18, kMetricQuantile = 19,
  kMetricAucPr = 20
};

// pair weight of the LambdaMART gradient: 1, |delta NDCG| or |delta AP|
enum B2RankMode { kRankPairwise = 0, kRankNdcg = 1, kRankMap = 2 };

// survival:aft distribution of the noise term (aft_loss_distribution)
enum B2AftDist { kAftNormal = 0, kAftLogistic = 1, kAftExtreme = 2 };

extern "C" {

// hist_kernel.cu (the CSR bin layout's build in hist_csr_kernel.cu).  n_work / total_chunks / chunk_rows are read from
// ctl when it is given.  window_rows is read by the dense build only, group_size [n_groups] by the CSR build only.
// scratch: b2_hist_scratch_elems(src, node_cap) int64 of device memory, zeroed by the launch
size_t b2_hist_scratch_elems(B2BinRows src, int node_cap);
int b2_launch_hist(B2BinRows src, const int32_t* group_size, const int2* gpair, const int32_t* ridx, const B2HistWork* work,
                   int n_work, int total_chunks, int chunk_rows, int window_rows, int n_groups, long long* hist,
                   long long* scratch, const B2LevelCtl* ctl, int log2_shards, int node_cap, int num_sms, cudaStream_t stream);
int b2_launch_hist_subtract(const long long* parent_level, long long* level, const int32_t* triples, int n_pairs,
                            int64_t node_elems, const B2LevelCtl* ctl, cudaStream_t stream);

// split_kernel.cu
int b2_eval_ctas_per_node(int n_groups, int log2_shards, int max_nodes);
int b2_eval_narrow_max_nodes();
int b2_launch_eval_splits(const long long* level_hist, int n_groups, const B2EvalNode* nodes, int n_nodes,
                          const int32_t* group_first, const int32_t* group_size, const int32_t* nbins,
                          const uint8_t* has_missing, const uint8_t* is_cat, const int32_t* qexp, int qbits, B2TrainParamDev p,
                          B2SplitCand* cands, int cand_stride, const B2LevelCtl* ctl, int log2_shards, int shard_rank,
                          B2ColSample cs, const B2NodeSeg* seg, B2SiblingSub sub, const B2DecideArgs* dec, uint32_t* done,
                          cudaStream_t stream);
int b2_cat_ctas();
int b2_launch_eval_cat_splits(const long long* level_hist, int n_groups, const B2EvalNode* nodes, int n_nodes,
                              const int32_t* cat_feats, int n_cat, const int32_t* feat_byte, const int32_t* nbins,
                              const int32_t* qexp, int qbits, B2TrainParamDev p, B2SplitCand* cands, int cand_stride,
                              int cand_offset, const B2LevelCtl* ctl, int log2_shards, int shard_rank, B2ColSample cs,
                              const B2NodeSeg* seg, cudaStream_t stream);
int b2_launch_root_totals(const long long* level_hist, int n_groups, B2EvalNode* nodes, const int32_t* qexp, int qbits,
                          B2TrainParamDev p, int log2_shards, long long* tree_sum_g, long long* tree_sum_h,
                          cudaStream_t stream);
int b2_eval_vector_ctas_per_node(int n_groups);
int b2_launch_eval_splits_vector(const long long* level_hist, size_t tstride, int T, int n_groups, const B2EvalNode* nodes,
                                 int max_nodes, const long long* vtot, const float* vgain, const int32_t* group_first,
                                 const int32_t* group_size, const int32_t* nbins, const uint8_t* has_missing,
                                 const int32_t* qexp, int qbits, B2TrainParamDev p, B2SplitCand* cands, int cand_stride,
                                 const B2LevelCtl* ctl, B2ColSample cs, const B2NodeSeg* seg, cudaStream_t stream);
int b2_launch_vector_root_totals(const long long* level_hist, size_t tstride, int T, int n_groups, const int32_t* qexp, int qbits,
                                 B2TrainParamDev p, long long* vtot, float* vgain, cudaStream_t stream);
int b2_launch_vector_child_totals(const long long* level_hist, size_t tstride, int T, int n_groups, int max_splits,
                                  const B2LevelCtl* ctl, const B2SplitWork* split_work, const int32_t* pair_parent_hist,
                                  const B2NodeSeg* seg_nxt, const int32_t* tree_parent, const int32_t* feat_byte,
                                  const int32_t* nbins, const int32_t* qexp, int qbits, B2TrainParamDev p, long long* vtot,
                                  float* vgain, B2EvalNode* ev_nxt, cudaStream_t stream);

// control_kernel.cu
int b2_launch_decide(const B2DecideArgs* a, const B2P2P* p2p, cudaStream_t s);
int b2_launch_leaf_plan(const B2LeafDev* leaves, const int32_t* n_leaves, B2SegWork* work, B2LevelCtl* leaf_ctl, cudaStream_t s);
int b2_launch_leaf_values(const B2LeafDev* leaves, const int32_t* n_leaves, const long long* sums, const int32_t* qexp,
                          int leaf_bits, B2CtlParams p, float* leaf_value, B2TreeDev tree, int32_t* qexp_out, cudaStream_t s);
int b2_launch_vector_leaf_values(const B2LeafDev* leaves, const int32_t* n_leaves, const long long* sums, size_t sums_stride,
                                 const int32_t* qexp, int T, int leaf_bits, B2CtlParams p, float* leaf_vec, float* tree_vec,
                                 int32_t* qexp_out, cudaStream_t s);
int b2_launch_tree_init(B2TreeDev tree, B2LevelCtl* ctl0, B2NodeSeg* seg0, B2EvalNode* ev0, int32_t* n_leaves, int n_rows,
                        B2HistWork* hist_work0, cudaStream_t s);

// partition_kernel.cu
int b2_part_chunk_rows();
int b2_split_chunk_rows();
// partition and final assign read a row's bin of the split feature from bins_col, or in the CSR layout from the row's
// stored entries (b2_csr_bin)
int b2_launch_partition(B2BinRows src, const int32_t* ridx_in, int32_t* ridx_out, const B2SplitWork* work,
                        const B2LevelCtl* ctl, int max_chunks, int32_t* counters, int any_categorical, B2FinalizeArgs fin,
                        int num_sms, cudaStream_t stream);
int b2_launch_leaf_sums(const float2* gh, const int32_t* ridx0, const int32_t* ridx1, const B2SegWork* work,
                        const B2LevelCtl* ctl, int max_chunks, const int32_t* qexp, int leaf_bits, long long* sums,
                        uint16_t* pos, int num_sms, cudaStream_t stream);
int b2_launch_final_assign(B2BinRows src, const int32_t* ridx_in, const B2SplitWork* work, const B2LevelCtl* ctl,
                           int max_chunks, const float2* gh, const int32_t* qexp, int leaf_bits, long long* sums, uint16_t* pos,
                           int any_categorical, int num_sms, cudaStream_t stream);
int b2_leaf_acc_max_depth();
int b2_launch_leaf_accumulate(const float2* gh, const uint16_t* pos, int64_t n, int max_depth, const int32_t* qexp, int leaf_bits,
                              long long* sums, int num_sms, cudaStream_t stream);
int b2_launch_margin_update(float* margin, int K, int k, const uint16_t* pos, const float* leaf_value, const float* weight,
                            int64_t n, int num_sms, cudaStream_t stream);
int b2_launch_margin_update_vector(float* margin, int T, const uint16_t* pos, const float* leaf_vec, int64_t n, int num_sms,
                                   cudaStream_t stream);

// p2p_exchange.cu
int b2_p2p_flag_words(int world);
int b2_launch_p2p_reduce_subtract(const B2P2P* pp, const long long* parent_level, long long* level, const int32_t* triples,
                                  const B2LevelCtl* ctl, int max_pairs, int node_cap, int64_t slice_elems, int num_sms,
                                  cudaStream_t s);
int b2_launch_p2p_quant_exponent(const B2P2P* pp, const uint32_t* absmax, int32_t* qexp, cudaStream_t s);
int b2_launch_p2p_leaf_sums(const B2P2P* pp, const int32_t* n_leaves, long long* sums, cudaStream_t s);
int b2_launch_gather_interleaved_rows(const B2RowBlocks* blocks, float* out, int num_sms, cudaStream_t s);

// objective_kernel.cu
int b2_gradient_fused_max_classes();
int b2_launch_gradient(int objective, int K, const float* margin, const float* label, const float* weight, int64_t n,
                       float scale_pos_weight, float obj_param, float2* gh, uint32_t* absmax, uint32_t* err, int num_sms,
                       cudaStream_t s);
int b2_launch_gradient_multi_target(int objective, int T, const float* margin, const float* label, const float* weight,
                                    int64_t n, float scale_pos_weight, float obj_param, float2* gh, uint32_t* absmax,
                                    uint32_t* err, int num_sms, cudaStream_t s);
// The metric launchers (metric, metric_multi_target, aft_metric, quantile_metric) write out[0..1] = (sum w v, sum w)
// in a fixed order, so the same model and matrix give the same bits on every call on one GPU model: each CTA's sums go
// to partial, b2_metric_partial_doubles(num_sms) doubles of device scratch, and b2_launch_metric_sum adds the first g
// pairs of it in CTA order.  n <= 0 launches nothing and leaves out as it is.
size_t b2_metric_partial_doubles(int num_sms);
int b2_launch_metric_sum(const double* partial, int g, double* out, cudaStream_t s);
int b2_launch_metric_multi_target(int objective, int metric, int T, float metric_param, const float* margin,
                                  const float* label, const float* weight, int64_t n, double* partial, double* out,
                                  int num_sms, cudaStream_t s);
int b2_launch_gradient_aft(int dist, double sigma, const float* margin, const float* lower, const float* upper,
                           const float* weight, int64_t n, float2* gh, uint32_t* absmax, uint32_t* err, int num_sms,
                           cudaStream_t s);
int b2_launch_aft_bounds_check(const float* lower, const float* upper, int64_t n, uint32_t* bad, int num_sms, cudaStream_t s);
int b2_launch_aft_metric(int dist, int metric, double sigma, const float* margin, const float* lower, const float* upper,
                         const float* weight, int64_t n, double* partial, double* out, int num_sms, cudaStream_t s);
int b2_launch_label_check(int objective, int K, const float* label, int64_t n, uint32_t* bad, int num_sms, cudaStream_t s);
int b2_launch_subsample(float2* gh, int64_t n, uint32_t seed, uint32_t tree, uint32_t rank, double subsample, int num_sms,
                        cudaStream_t s);
int b2_launch_sum_fixed(const float2* gh, int64_t n, const int32_t* qexp, int bits, long long* out, int num_sms, cudaStream_t s);
int b2_launch_pack_custom(const float* g, const float* h, int K, int64_t n, float2* gh, int num_sms, cudaStream_t s);
int b2_launch_absmax(const float2* gh, int64_t n, uint32_t* absmax, int num_sms, cudaStream_t s);
int b2_launch_quant_exponent(const uint32_t* absmax, int32_t* qexp, cudaStream_t s);
int b2_launch_quantize(const float2* gh, int64_t n, const int32_t* qexp, int qbits, int2* q, int num_sms, cudaStream_t s);
// out[2] += the rows of mlogloss / merror whose label is not a class index
int b2_launch_metric(int objective, int metric, int K, float metric_param, const float* margin, const float* label,
                     const float* weight, int64_t n, double* partial, double* out, int num_sms, cudaStream_t s);
int b2_launch_predict(B2RawRows src, int64_t n, int F, float missing, const B2TreeNodeDev* nodes, const int32_t* tree_offset,
                      const uint32_t* cat_table, int tree_begin, int tree_end, int K, int npt, const float* weights, float* out,
                      int num_sms, cudaStream_t s);
int b2_launch_predict_vector(B2RawRows src, int64_t n, int F, float missing, const B2TreeNodeDev* nodes,
                             const int32_t* tree_offset, const float* leaf_vec, int tree_begin, int tree_end, int T, float* out,
                             int num_sms, cudaStream_t s);
int b2_launch_fill(float* out, int64_t n, float v, int num_sms, cudaStream_t s);
int b2_launch_transform(int objective, int K, float* m, int64_t n, int num_sms, cudaStream_t s);

// quantile_kernel.cu (sel: the per-leaf selection state, b2_quantile_sel_bytes(max_leaves) bytes)
size_t b2_quantile_hist_elems(int max_leaves);
size_t b2_quantile_sel_bytes(int max_leaves);
int b2_quantile_passes();
int b2_launch_gradient_quantile(int K, const float* alpha, const float* margin, const float* label, const float* weight,
                                int64_t n, float2* gh, uint32_t* absmax, int num_sms, cudaStream_t s);
int b2_launch_quantile_metric(int K, const float* alpha, const float* margin, const float* label, const float* weight,
                              int64_t n, double* partial, double* out, int num_sms, cudaStream_t s);
int b2_launch_quantile_count(int pass, const uint16_t* pos, const float* label, const float* margin, int K, int k,
                             const float2* gh, int64_t n, const int32_t* qexp, int weighted, const void* sel,
                             int max_leaves, unsigned long long* hist, int num_sms, cudaStream_t s);
int b2_launch_quantile_scan(int pass, const int32_t* n_leaves, int max_leaves, int weighted, float alpha, float eta,
                            unsigned long long* hist, void* sel, const B2LeafDev* leaves, float* leaf_value,
                            float* tree_value, cudaStream_t s);

// dart_kernel.cu
int b2_launch_dart_margins(B2BinRows src, int64_t n, const uint8_t* has_missing, const B2TreeNodeDev* nodes,
                           const int32_t* tree_offset, const uint32_t* cat_table, int T, int K, int npt, const float* w_drop,
                           const uint8_t* dropped, const float* w_full, float* drop, float* full, int num_sms, cudaStream_t s);

// shap_kernel.cu
size_t b2_shap_contribs_smem(int K, int F, int warps);
int b2_launch_shap_contribs(const float* X, int64_t row0, int64_t rows, int F, float missing, const B2PathElem* elems,
                            const B2PathInfo* paths, int p_begin, int p_end, const uint32_t* cat_table, int K,
                            const double* bias_k, const float* base_margin, float base_value, double* gacc, int warps,
                            size_t smem, float* out, int num_sms, cudaStream_t s);
int b2_launch_shap_interactions(const float* X, int64_t row0, int64_t rows, int F, float missing, const B2PathElem* elems,
                                const B2PathInfo* paths, int p_begin, int p_end, const uint32_t* cat_table, int K,
                                const double* bias_k, const float* base_margin, float base_value, double* gacc, float* out,
                                int num_sms, cudaStream_t s);
int b2_launch_leaf_index(B2RawRows src, int64_t row0, int64_t rows, int F, float missing, const B2TreeNodeDev* nodes,
                         const int32_t* tree_offset, const uint32_t* cat_table, int tree_begin, int tree_end, float* out,
                         int num_sms, cudaStream_t s);

// rank_kernel.cu (temp: CUB scratch of b2_rank_order_temp_bytes bytes)
int b2_rank_stage_rows();
size_t b2_rank_order_temp_bytes(int64_t n, int64_t n_groups);
int b2_launch_rank_iota(int32_t* idx, int64_t n, int num_sms, cudaStream_t s);
int b2_rank_order(const float* v, int64_t n, const int64_t* gptr, int64_t n_groups, const int32_t* iota, uint32_t* keys,
                  uint32_t* keys_out, int32_t* rows_out, void* temp, size_t temp_bytes, int num_sms, cudaStream_t s);
int b2_launch_rank_disc(double* disc, int64_t len, int num_sms, cudaStream_t s);
int b2_launch_rank_inv_idcg(const int64_t* gptr, int64_t n_groups, const uint32_t* lkeys, const double* disc, int k,
                            int exp_gain, double* inv_idcg, int num_sms, cudaStream_t s);
int b2_launch_rank_label_check(const float* label, int64_t n, int exp_gain, int binary, uint32_t* bad, int num_sms,
                               cudaStream_t s);
int b2_launch_lambdarank_gradient(int mode, const int64_t* gptr, int64_t n_groups, int64_t max_group, const uint32_t* skeys,
                                  const int32_t* srow, const float* label, const double* inv_idcg, const double* disc, int k,
                                  int exp_gain, float* scratch_m, float* scratch_y, double* scratch_p, double* scratch_a,
                                  int32_t* scratch_r, float2* gh, uint32_t* absmax, uint32_t* err, int num_sms, cudaStream_t s);
int b2_launch_rank_metric(int metric, int k, int minus, int exp_gain, const int64_t* gptr, int64_t n_groups, const int32_t* prow,
                          const float* label, const uint32_t* lkeys, const double* disc, double* vals, double* out, int num_sms,
                          cudaStream_t s);

// auc_kernel.cu (temp: scratch of b2_auc_temp_bytes bytes)
size_t b2_auc_temp_bytes(int64_t n);
int b2_auc(int pr, int K, const float* pred, const float* label, const float* weight, int64_t n, void* temp,
           size_t temp_bytes, double* out, int num_sms, cudaStream_t s);

// sketch.cu (temp: CUB scratch of b2_sort_temp_bytes bytes)
int b2_extract_batch();
int b2_launch_extract_keys(const float* X, int64_t n, int F, int f0, int nf, float missing, uint32_t* keys, int64_t n_padded,
                           int num_sms, cudaStream_t s);
size_t b2_sort_temp_bytes(int64_t n);
int b2_launch_weight_absmax(const float* w, int64_t n, uint32_t* absmax, int num_sms, cudaStream_t s);
int b2_launch_weight_quantize(const float* w, int64_t n, int64_t n_padded, const uint32_t* absmax, int32_t* wq, int num_sms,
                              cudaStream_t s);
int b2_sketch_column(const uint32_t* keys_in, const int32_t* wq_in, uint32_t* keys_sorted, int32_t* wq_sorted, long long* wpre,
                     int64_t n_total, long long n_global, void* temp, size_t temp_bytes, int32_t* flags, int32_t* idx,
                     float* uval, long long* rmin, int32_t* m_scratch, long long* n_valid_scratch, int max_bin,
                     float* cut_out, int32_t* n_cut_out, float* min_out, int32_t* has_missing_out, int num_sms,
                     cudaStream_t s);
size_t b2_sketch_batch_temp_bytes(int64_t n);
int b2_sketch_batch(const uint64_t* keys_in, const int32_t* wq_in, uint64_t* keys_sorted, int32_t* wq_sorted, long long* wpre,
                    int64_t n_sort, const int64_t* seg, const int64_t* h_seg, int f0, int nf, const uint8_t* is_cat, int world,
                    int rank, long long n_global, void* temp, size_t temp_bytes, int32_t* flags, int32_t* idx, float* uval,
                    long long* rmin, int max_bin, float* cuts, int32_t* n_cuts, float* mins, int32_t* has_missing, int num_sms,
                    cudaStream_t s);
int b2_launch_bin(const float* X, int64_t n, int F, float missing, const int32_t* cut_ptrs, const float* cut_vals,
                  const int32_t* feat_byte, const uint8_t* is_cat, int row_stride, uint8_t* bins, uint8_t* bins_col,
                  int64_t col_stride, int num_sms, cudaStream_t s);
// ebins [nnz] = the bin of every stored entry of a CSR matrix, by the rule of b2_launch_bin
int b2_launch_bin_csr(const int32_t* indices, const float* values, int64_t nnz, float missing, const int32_t* cut_ptrs,
                      const float* cut_vals, const uint8_t* is_cat, uint8_t* ebins, int num_sms, cudaStream_t s);
int b2_launch_cat_stats(const float* X, int64_t n, int F, float missing, const int32_t* cat_feats, int n_cat, int32_t* stats,
                        int num_sms, cudaStream_t s);

// sparse_kernel.cu (CSR raw values: indptr [n+1], indices / values [nnz])
int b2_launch_csr_validate(const int64_t* indptr, const int32_t* indices, int64_t n, int F, int64_t nnz, unsigned long long* bad,
                           int num_sms, cudaStream_t s);
int b2_launch_csr_densify(const int64_t* indptr, const int32_t* indices, const float* values, int64_t r0, int64_t rows, int F,
                          float* out, int num_sms, cudaStream_t s);
// out [n][F] = the dense bins of a CSR-layout matrix (absent entries: the missing sentinel)
int b2_launch_csr_bins_densify(const int64_t* indptr, const int32_t* indices, const uint8_t* ebins, int64_t n, int F,
                               uint8_t* out, int num_sms, cudaStream_t s);
// counts [F] (zeroed) += valid stored entries per numeric feature; keys / wq_out of features [f0, f0 + nf) at cursor [nf]
int b2_launch_csr_column_counts(const int32_t* indices, const float* values, int64_t nnz, float missing, const uint8_t* is_cat,
                                unsigned long long* counts, int num_sms, cudaStream_t s);
int b2_launch_csr_sketch_keys(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int f0, int nf,
                              float missing, const uint8_t* is_cat, const int32_t* wq, unsigned int* cursor, uint64_t* keys,
                              int32_t* wq_out, int num_sms, cudaStream_t s);
// stats as b2_launch_cat_stats, from the stored entries of an n-row matrix (stored: n_cat scratch)
int b2_launch_csr_cat_stats(const int32_t* indices, const float* values, int64_t nnz, int64_t n, float missing, const int32_t* cat_of,
                            int n_cat, unsigned long long* stored, int32_t* stats, int num_sms, cudaStream_t s);

// slice_kernel.cu (B2_MatrixSlice: rows[0..n) of a parent matrix, in that order, duplicates allowed; every row index is
// in range, checked by the caller)
// dst [n][width] = src [rows[i]][width]: dense raw values and the per-row side arrays
int b2_launch_gather_rows(const float* src, int64_t width, const int64_t* rows, int64_t n, float* dst, int num_sms,
                          cudaStream_t s);
size_t b2_csr_slice_temp_bytes(int64_t n);
// out_indptr [n+1] of the slice (lengths: n scratch int64, temp: b2_csr_slice_temp_bytes(n) bytes of CUB scratch)
int b2_launch_csr_slice_indptr(const int64_t* indptr, const int64_t* rows, int64_t n, int64_t* lengths, int64_t* out_indptr,
                               void* temp, size_t temp_bytes, int num_sms, cudaStream_t s);
int b2_launch_csr_slice_entries(const int64_t* indptr, const int32_t* indices, const float* values, const int64_t* rows,
                                int64_t n, const int64_t* out_indptr, int32_t* out_indices, float* out_values, int num_sms,
                                cudaStream_t s);

// refresh_kernel.cu
int b2_launch_refresh(B2RawRows src, int64_t n, int F, float missing, const B2TreeNodeDev* nodes, int n_nodes,
                      const uint32_t* cat_table, int n_leaves, const float2* gh, const int32_t* qexp, int leaf_bits,
                      uint16_t* pos, long long* sums, int num_sms, cudaStream_t stream);
int b2_launch_refresh_nodes(const B2TreeNodeDev* nodes, int n_nodes, const int32_t* order, const int32_t* level_ptr, int n_levels,
                            const long long* sums, const int32_t* qexp, int leaf_bits, B2CtlParams p, int refresh_leaf,
                            long long* limbs, unsigned char* block, float* leaf_table, cudaStream_t stream);

}  // extern "C"
