// predict.cu -- prediction on the device model: the TreeSHAP path table, margins of a range of trees, the cached
// evaluation margins of a matrix, and the eval metrics over the workers.
#include <math.h>

#include "host.h"
#include "launch.h"

namespace b2host __attribute__((visibility("hidden"))) {

void trees_edited(Booster* b) {
  b->d_trees_synced = -1; b->paths_synced = -1; b->margin_ready = false;
  for (auto& kv : b->eval_cache) if (kv.second) kv.second->n_trees_applied = 0, kv.second->n = -1;
}

// ---- TreeSHAP path table (common.cuh B2PathElem / B2PathInfo; shap_kernel.cu).  Walks every tree root -> leaf; on the
// way each split is merged into the element of its feature (appended the first time the feature is seen): the interval
// of a numeric feature narrows, the category set of a categorical feature is intersected with the side taken (keeping
// predict_kernel's rule that a category outside [0, 256) goes left), the missing flag is AND-ed with "the default
// direction is the side taken", and zero_fraction is multiplied by cover(child) / cover(parent) (0 for a zero-cover
// parent, never NaN).  The tree's expected value, sum over leaves of value * prod zero_fraction, is its SHAP bias.
struct PathBuildElem {
  int32_t feature; bool is_cat; float lo, hi; uint32_t flags; uint32_t bits[8]; double z;
};
void walk_paths(const TreeHost& t, int nid, std::vector<PathBuildElem>& path, int tree, int cls, Booster* b,
                std::vector<B2PathElem>& elems, std::vector<B2PathInfo>& infos, std::vector<uint32_t>& cats, double* expected) {
  if (t.feature[nid] < 0) {
    if (path.size() + 1 > B2_SHAP_MAX_PATH)
      fail("tree %d has a leaf below %d distinct features; TreeSHAP supports at most %d distinct features on a path", tree,
           (int)path.size(), B2_SHAP_MAX_PATH - 1);
    B2PathInfo pi{(int32_t)elems.size(), (int32_t)path.size() + 1, cls, 0, (double)t.value[nid]};
    elems.push_back(B2PathElem{-1, -1, 0.f, 0.f, 0u, 0u, 1.0});
    double zprod = 1.0;
    for (const PathBuildElem& e : path) {
      int32_t slot = -1;
      if (e.is_cat) { slot = (int32_t)(cats.size() / 8); cats.insert(cats.end(), e.bits, e.bits + 8); }
      elems.push_back(B2PathElem{e.feature, slot, e.lo, e.hi, e.flags, 0u, e.z});
      zprod *= e.z;
    }
    *expected += (double)t.value[nid] * zprod;
    infos.push_back(pi);
    return;
  }
  const int f = t.feature[nid];
  const bool is_cat = t.split_type[nid] != 0;
  const double cover = t.sum_hess[nid];
  for (int side = 0; side < 2; ++side) {
    const int child = side == 0 ? t.left[nid] : t.right[nid];
    const bool left = side == 0;
    std::vector<PathBuildElem> next = path;
    PathBuildElem* e = nullptr;
    for (auto& x : next) if (x.feature == f) e = &x;
    if (!e) {
      PathBuildElem ne;
      ne.feature = f; ne.is_cat = is_cat; ne.lo = -INFINITY; ne.hi = INFINITY;
      ne.flags = B2_PATH_MISSING_OK | B2_PATH_OUTSIDE_OK; ne.z = 1.0;
      for (int w = 0; w < 8; ++w) ne.bits[w] = 0xffffffffu;
      next.push_back(ne); e = &next.back();
    }
    e->z *= cover > 0.0 ? t.sum_hess[child] / cover : 0.0;
    if ((t.default_left[nid] != 0) != left) e->flags &= ~B2_PATH_MISSING_OK;
    if (is_cat) {
      e->is_cat = true;
      for (int w = 0; w < 8; ++w) e->bits[w] &= left ? ~t.cat_bits[(size_t)nid * 8 + w] : t.cat_bits[(size_t)nid * 8 + w];
      if (!left) e->flags &= ~B2_PATH_OUTSIDE_OK;
    } else if (left) {
      if (!(e->flags & B2_PATH_HAS_HI) || t.cond[nid] < e->hi) e->hi = t.cond[nid];
      e->flags |= B2_PATH_HAS_HI;
    } else if (t.cond[nid] > e->lo) {
      e->lo = t.cond[nid];
    }
    walk_paths(t, child, next, tree, cls, b, elems, infos, cats, expected);
  }
}

void build_paths(Booster* b) {
  if (b->paths_synced == (int)b->trees.size() && b->paths_weights_version == (int)b->weights_version) return;
  std::vector<B2PathElem> elems; std::vector<B2PathInfo> infos; std::vector<uint32_t> cats;
  b->tree_path_offset.assign(1, 0); b->tree_expected.clear();
  const int K = b->p.num_class, npt = std::max(1, b->p.num_parallel_tree);
  for (int t = 0; t < (int)b->trees.size(); ++t) {
    std::vector<PathBuildElem> path;
    double expected = 0.0;
    const int32_t first = (int32_t)infos.size();
    walk_paths(b->trees[t], 0, path, t, (t / npt) % K, b, elems, infos, cats, &expected);
    if (b->p.dart) {   // DART: the tree's leaves count with its weight
      const double w = (double)b->tree_w[t];
      for (size_t i = first; i < infos.size(); ++i) infos[i].value *= w;
      expected *= w;
    }
    b->tree_path_offset.push_back((int32_t)infos.size());
    b->tree_expected.push_back(expected);
  }
  cudaStream_t s = b->ctx->stream;
  upload(b->d_path_elems, elems, s); upload(b->d_paths, infos, s); upload(b->d_path_cats, cats, s);
  CUDA_CHECK(cudaStreamSynchronize(s));
  b->paths_synced = (int)b->trees.size();
  b->paths_weights_version = (int)b->weights_version;
}

// DART: the tree weights on the device (nullptr for gbtree: the kernels then add the plain leaf values)
const float* device_weights(Booster* b) {
  if (!b->p.dart) return nullptr;
  if (b->d_tree_w_version != b->weights_version || b->d_tree_w_count != b->tree_w.size()) {
    upload(b->d_tree_w, b->tree_w, b->ctx->stream);   // pageable source: staged before return
    b->d_tree_w_version = b->weights_version; b->d_tree_w_count = b->tree_w.size();
  }
  return b->d_tree_w.p;
}

// out += the trees [tree_begin, tree_end) on the raw rows of m
void predict_trees(Booster* b, Matrix* m, int tree_begin, int tree_end, float* out) {
  sync_device_trees(b);
  const float* w = b->p.vector_leaf() ? nullptr : device_weights(b);
  const B2RawRows src = raw_source(m);
  if (b->p.vector_leaf())
    LAUNCH_CHECK(b2_launch_predict_vector(src, m->n, m->F, m->missing, b->d_nodes.p, b->d_tree_offset.p, b->d_leaf_table.p,
                                          tree_begin, tree_end, b->p.num_target, out, b->ctx->num_sms, b->ctx->stream));
  else
    LAUNCH_CHECK(b2_launch_predict(src, m->n, m->F, m->missing, b->d_nodes.p, b->d_tree_offset.p, b->d_cat_table.p, tree_begin,
                                   tree_end, b->p.num_class, b->p.num_parallel_tree, w, out, b->ctx->num_sms, b->ctx->stream));
}

// margin of matrix m under the current model (cached per matrix, only new trees are applied)
float* eval_margin(Booster* b, Matrix* m) {
  if (b->train && m == b->train) { ensure_train_margin(b); return b->margin.p; }
  if (!m->has_raw) fail("evaluation / prediction matrix has no raw data on the device");
  if (m->F != b->n_features) fail("feature count mismatch: matrix has %d, model has %d", m->F, b->n_features);
  // drop the cached margins of matrices that were freed since the last call
  for (auto it = b->eval_cache.begin(); it != b->eval_cache.end();) {
    if (!matrix_alive(it->first)) { delete it->second; it = b->eval_cache.erase(it); } else ++it;
  }
  if (!m->uid) fail("evaluation matrix is not a registered matrix handle");
  EvalCache*& c = b->eval_cache[m->uid];
  const int K = b->p.num_class;
  if (!c || c->n != m->n || c->margin_version != m->margin_version || c->weights_version != b->weights_version) {
    delete c; c = new EvalCache(); c->n = m->n; c->margin_version = m->margin_version; c->weights_version = b->weights_version;
    c->margin.ensure((size_t)std::max<int64_t>(m->n * K, 1));
    init_margin(b, c->margin.p, m);
    c->n_trees_applied = 0;
  }
  const int nt = (int)b->trees.size();
  if (c->n_trees_applied < nt) {
    predict_trees(b, m, c->n_trees_applied, nt, c->margin.p);
    c->n_trees_applied = nt;
  }
  return c->margin.p;
}

// the first n doubles of b->d_metric summed over the workers, on the host (synchronises the stream)
static std::vector<double> metric_sums(Booster* b, size_t n, cudaStream_t s) {
  allreduce(b->comm, b->d_metric.p, n, kNcclFloat64, kNcclSum, s);
  std::vector<double> h(n);
  CUDA_CHECK(cudaMemcpyAsync(h.data(), b->d_metric.p, n * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  return h;
}

// eval_metric `name` on matrix m over every worker; the class, quantile and multi-target rules come after the margin
double eval_metric(Booster* b, Matrix* m, const char* name) {
  const Params& p = b->p; cudaStream_t s = b->ctx->stream; const int sms = b->ctx->num_sms, K = p.num_class;
  float mparam; int minus;
  const Metric& mt = metric_id(name, p, &mparam, &minus);
  const ObjGrad grad = objective_row(p).grad;
  const char* obj = p.objective_name.c_str();
  const bool rank = mt.family == kEvalRank, auc = mt.family == kEvalAuc, aft = mt.family == kEvalAft;
  if (rank && K > 1) fail("metric '%s' needs a single-output objective", name);
  if (rank && !m->has_qgroups()) fail("metric '%s' needs query groups (qid) on the evaluation matrix", name);
  // xgboost computes a per-group ranking AUC on a matrix with groups; this engine's auc / aucpr are binary or one-vs-rest
  if (auc && m->has_qgroups())
    fail("metric '%s' on a matrix with query groups (per-group ranking AUC) is not supported; use ndcg or map", name);
  if (auc && p.num_target > 1)
    fail("metric '%s' is not supported for a multi-target model (%d targets); use rmse, mae, logloss or error", name,
         p.num_target);
  if (auc && K > 1 && grad != kGradSoftprob)
    fail("metric '%s' needs one output per row or a multi:softprob / multi:softmax model; objective '%s' has %d outputs",
         name, obj, K);
  if (aft && grad != kGradAft) fail("metric '%s' does not fit objective '%s'", name, obj);
  if (aft && !m->has_bounds()) fail("metric '%s' needs label_lower_bound and label_upper_bound on the evaluation matrix", name);
  if (!aft && m->n_label > 0 && m->n_targets != p.num_target)
    fail("metric '%s': the evaluation matrix's label has %d columns, the model has %d targets", name, m->n_targets,
         p.num_target);
  if (!aft && !m->has_labels(p.num_target)) fail("evaluation matrix has no labels");
  float* margin = eval_margin(b, m);
  if (!auc && (mt.family == kEvalClass) != (grad == kGradSoftprob)) fail("metric '%s' does not fit objective '%s'", name, obj);
  if (mt.family == kEvalQuantile && grad != kGradQuantile)
    fail("metric 'quantile' needs objective reg:quantileerror (it reads quantile_alpha)");
  if (p.num_target > 1 && !mt.multi_target)
    fail("metric '%s' is not supported for a multi-target model (supported: rmse, rmsle, mae, mape, mphe, logloss, error)",
         name);
  const float* w = m->n_weight ? m->weight.p : nullptr;
  // d_metric: the AUC triples, or the aft, quantile and elementwise sums followed by their per-CTA partials
  b->d_metric.ensure(std::max(3 * (size_t)K + 1, 3 + b2_metric_partial_doubles(sms)));
  CUDA_CHECK(cudaMemsetAsync(b->d_metric.p, 0, 3 * sizeof(double), s));
  double* partial = b->d_metric.p + 3;
  DevBuf<float> pred;   // the ranking and AUC metrics read the transformed prediction
  if (rank || auc) {
    pred.ensure((size_t)std::max<int64_t>(m->n * K, 1));
    if (m->n > 0) CUDA_CHECK(cudaMemcpyAsync(pred.p, margin, (size_t)(m->n * K) * sizeof(float), cudaMemcpyDeviceToDevice, s));
    LAUNCH_CHECK(b2_launch_transform(p.objective, K, pred.p, m->n, sms, s));
  }
  switch (mt.family) {
    case kEvalRank: {
      // ndcg / map / pre: per query group on the prediction order (rank_kernel.cu), averaged over the groups of all workers
      DevBuf<double> vals; RankOrder po, lo;
      po.run(m, pred.p, sms, s);
      if (mt.id == kMetricNdcg) lo.run(m, m->label.p, sms, s);
      ensure_rank_disc(b, m->max_qgroup);
      vals.ensure((size_t)std::max<int64_t>(m->n_qgroups, 1));
      LAUNCH_CHECK(b2_launch_rank_metric(mt.id, (int)mparam, minus, p.ndcg_exp_gain ? 1 : 0, m->qgroup_ptr.p, m->n_qgroups,
                                         po.rows.p, m->label.p, mt.id == kMetricNdcg ? lo.keys_sorted.p : nullptr,
                                         b->rank_disc.p, vals.p, b->d_metric.p, sms, s));
      break;
    }
    case kEvalAuc: {
      // ROC / PR AUC (auc_kernel.cu; DESIGN.md §2 item 17): per class a worker's triple (ROC: area, fp*tp, tp; PR: aucpr,
      // 1, 1) plus the count of out-of-range labels, summed over the workers
      DevBuf<uint8_t> tmp;
      const size_t tb = b2_auc_temp_bytes(m->n);
      tmp.ensure(tb);
      LAUNCH_CHECK(b2_auc(mt.id == kMetricAucPr ? 1 : 0, K, pred.p, m->label.p, w, m->n, tmp.p, tb, b->d_metric.p, sms, s));
      const std::vector<double> h = metric_sums(b, 3 * (size_t)K + 1, s);
      if (h[3 * (size_t)K] > 0)
        fail("metric '%s': label must be in [0, num_class), num_class = %d (%.0f rows outside)", name, K, h[3 * (size_t)K]);
      // ROC with only one class present: xgboost reports 0.5
      if (K == 1) return mt.id == kMetricAuc ? (h[1] > 0 ? h[0] / h[1] : 0.5) : h[0] / h[1];
      // one-vs-rest: sum_c (A_c / L_c) T_c / sum_c T_c; NaN when some class has L_c = 0 or no class has T_c
      double num = 0.0, den = 0.0;
      for (int c = 0; c < K; ++c) {
        const double A = h[3 * c], L = h[3 * c + 1], T = h[3 * c + 2];
        if (!(L > 0)) return NAN;
        num += A / L * T; den += T;
      }
      return den > 0 ? num / den : NAN;
    }
    case kEvalAft:
      LAUNCH_CHECK(b2_launch_aft_metric(p.aft_dist, mt.id, (double)p.aft_sigma, margin, m->lower.p, m->upper.p, w, m->n,
                                        partial, b->d_metric.p, sms, s));
      break;
    case kEvalQuantile:
      // pinball loss averaged over the rows and the alphas, weighted (sum, K * sum w summed over the workers)
      if (!b->d_alpha.p || b->d_alpha.cap < p.quantile_alpha.size()) {
        upload(b->d_alpha, p.quantile_alpha, s);
        CUDA_CHECK(cudaStreamSynchronize(s));
      }
      LAUNCH_CHECK(b2_launch_quantile_metric(K, b->d_alpha.p, margin, m->label.p, w, m->n, partial, b->d_metric.p, sms, s));
      break;
    default: {
      // elementwise (over the n x T outputs of a multi-target model, each with its row's weight: xgboost's EvalEWiseBase)
      // and class metrics: (sum, wsum, rows with a label outside [0, num_class)), so every rank fails together
      if (p.num_target > 1)
        LAUNCH_CHECK(b2_launch_metric_multi_target(p.objective, mt.id, p.num_target, mparam, margin, m->label.p, w, m->n,
                                                   partial, b->d_metric.p, sms, s));
      else
        LAUNCH_CHECK(b2_launch_metric(p.objective, mt.id, K, mparam, margin, m->label.p, w, m->n, partial, b->d_metric.p,
                                      sms, s));
      const std::vector<double> h = metric_sums(b, 3, s);
      if (h[2] > 0) fail("metric '%s': label must be in [0, num_class), num_class = %d (%.0f rows outside)", name, K, h[2]);
      const double v = h[1] > 0 ? h[0] / h[1] : 0.0;
      return (mt.id == kMetricRmse || mt.id == kMetricRmsle) ? sqrt(v) : v;
    }
  }
  const std::vector<double> h = metric_sums(b, 2, s);   // ranking, aft and quantile: (sum, weight sum)
  return h[1] > 0 ? h[0] / h[1] : 0.0;
}

// the checks every prediction entry makes (each checks its output length where it can); resolves tree_end <= 0 to all trees
static void check_predict_args(Booster* b, Matrix* m, int tree_begin, int* tree_end) {
  if (!m->has_raw) fail("prediction matrix has no raw data on the device (B2_MatrixEnsureRaw)");
  if (m->F != b->n_features) fail("feature count mismatch: matrix has %d, model has %d", m->F, b->n_features);
  const int nt = (int)b->trees.size();
  if (*tree_end <= 0 || *tree_end > nt) *tree_end = nt;
  if (tree_begin < 0 || tree_begin > *tree_end) fail("invalid tree range [%d, %d)", tree_begin, *tree_end);
  if (m->n_base_margin > 0 && m->n_base_margin != m->n * b->p.num_class)
    fail("base_margin has %lld values, expected %lld", (long long)m->n_base_margin, (long long)(m->n * b->p.num_class));
}

// rows per output block, so that the device scratch of one block stays within 1 GiB whatever the row count, and within
// one raw tile
static int64_t rows_per_block(Matrix* m, size_t bytes_per_row) {
  const size_t budget = (size_t)1 << 30;
  int64_t r = (int64_t)std::max<size_t>(1, budget / std::max<size_t>(bytes_per_row, 1));
  return std::min(std::max<int64_t>(1, std::min<int64_t>(r, m->n)), raw_tile_rows(m));
}

void predict(Booster* b, Matrix* m, bool output_margin, int tree_begin, int tree_end, float* out, int64_t out_len) {
  cudaStream_t s = b->ctx->stream; const int K = b->p.num_class;
  if (out_len != m->n * K) fail("output buffer has %lld values, expected %lld", (long long)out_len, (long long)(m->n * K));
  check_predict_args(b, m, tree_begin, &tree_end);
  DevBuf<float> tmp; tmp.ensure((size_t)std::max<int64_t>(out_len, 1));
  init_margin(b, tmp.p, m);
  predict_trees(b, m, tree_begin, tree_end, tmp.p);
  if (!output_margin) LAUNCH_CHECK(b2_launch_transform(b->p.objective, K, tmp.p, m->n, b->ctx->num_sms, s));
  if (out_len > 0) CUDA_CHECK(cudaMemcpyAsync(out, tmp.p, out_len * sizeof(float), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
}

void predict_contribs(Booster* b, Matrix* m, int tree_begin, int tree_end, bool interactions, float* out, int64_t out_len) {
  cudaStream_t s = b->ctx->stream; const int K = b->p.num_class; const int F = m->F;
  const size_t per_row = (size_t)K * (F + 1) * (interactions ? (size_t)(F + 1) : 1);
  if (b->p.vector_leaf())
    fail("%s is not supported for vector-leaf trees (multi_strategy=multi_output_tree)",
         interactions ? "pred_interactions" : "pred_contribs");
  if (out_len != m->n * (int64_t)per_row) fail("output buffer has %lld values, expected %lld", (long long)out_len, (long long)(m->n * (int64_t)per_row));
  check_predict_args(b, m, tree_begin, &tree_end);
  build_paths(b);
  std::vector<double> bias(K, 0.0);   // sum of the expected values of the trees in range, in tree order
  for (int t = tree_begin; t < tree_end; ++t) bias[(t / std::max(1, b->p.num_parallel_tree)) % K] += b->tree_expected[t];
  DevBuf<double> d_bias; upload(d_bias, bias, s);
  const int p_begin = b->tree_path_offset[tree_begin], p_end = b->tree_path_offset[tree_end];
  const float* bm = m->n_base_margin > 0 ? m->base_margin.p : nullptr;
  const float base_value = base_margin_value(b->p);
  // contributions: the row accumulators live in shared memory (up to 8 warps of K (F+1) doubles in <= 200 KiB),
  // otherwise in global scratch; interactions always accumulate in global scratch
  int warps = 8; size_t smem = 0;
  if (!interactions) {
    while (warps > 1 && b2_shap_contribs_smem(K, F, warps) > (size_t)200 * 1024) warps /= 2;
    smem = b2_shap_contribs_smem(K, F, warps);
    if (smem > (size_t)200 * 1024) { smem = 0; warps = 8; }
  }
  const bool gscratch = interactions || smem == 0;
  if (m->n == 0) { CUDA_CHECK(cudaStreamSynchronize(s)); return; }   // for_raw_tiles calls once, with no rows
  const int64_t blk = rows_per_block(m, per_row * (sizeof(float) + (gscratch ? sizeof(double) : 0)));
  DevBuf<float> d_out; DevBuf<double> d_acc;
  d_out.ensure((size_t)blk * per_row);
  if (gscratch) d_acc.ensure((size_t)blk * per_row);
  std::vector<cudaEvent_t> ev;
  for_raw_tiles(m, [&](const float* X, int64_t r0, int64_t rows) {   // row 0 of X is row r0 of the matrix
    cudaEvent_t e0, e1; CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
    ev.push_back(e0); ev.push_back(e1);
    const float* bm_rows = bm ? bm + (size_t)r0 * K : nullptr;
    CUDA_CHECK(cudaEventRecord(e0, s));
    if (interactions)
      LAUNCH_CHECK(b2_launch_shap_interactions(X, 0, rows, F, m->missing, b->d_path_elems.p, b->d_paths.p, p_begin, p_end,
                                               b->d_path_cats.p, K, d_bias.p, bm_rows, base_value, d_acc.p, d_out.p, b->ctx->num_sms, s));
    else
      LAUNCH_CHECK(b2_launch_shap_contribs(X, 0, rows, F, m->missing, b->d_path_elems.p, b->d_paths.p, p_begin, p_end,
                                           b->d_path_cats.p, K, d_bias.p, bm_rows, base_value, gscratch ? d_acc.p : nullptr, warps,
                                           smem, d_out.p, b->ctx->num_sms, s));
    CUDA_CHECK(cudaEventRecord(e1, s));
    CUDA_CHECK(cudaMemcpyAsync(out + (size_t)r0 * per_row, d_out.p, (size_t)rows * per_row * sizeof(float), cudaMemcpyDeviceToHost, s));
  }, blk);
  CUDA_CHECK(cudaStreamSynchronize(s));
  for (size_t i = 0; i < ev.size(); i += 2) {
    float ms = 0; cudaEventElapsedTime(&ms, ev[i], ev[i + 1]);
    b->t.shap_ms += ms;
    cudaEventDestroy(ev[i]); cudaEventDestroy(ev[i + 1]);
  }
  b->t.shap_rows += m->n;
}

void predict_leaf(Booster* b, Matrix* m, int tree_begin, int tree_end, float* out, int64_t out_len) {
  cudaStream_t s = b->ctx->stream;
  check_predict_args(b, m, tree_begin, &tree_end);
  const int T = tree_end - tree_begin;
  if (out_len != m->n * T) fail("output buffer has %lld values, expected %lld", (long long)out_len, (long long)(m->n * T));
  if (T == 0 || m->n == 0) return;
  sync_device_trees(b);
  // row blocks stage the output; the rows are read in place
  const int64_t blk = rows_per_block(m, (size_t)T * sizeof(float));
  DevBuf<float> d_out; d_out.ensure((size_t)blk * T);
  const B2RawRows src = raw_source(m);
  for (int64_t r0 = 0; r0 < m->n; r0 += blk) {
    const int64_t rows = std::min(blk, m->n - r0);
    LAUNCH_CHECK(b2_launch_leaf_index(src, r0, rows, m->F, m->missing, b->d_nodes.p, b->d_tree_offset.p, b->d_cat_table.p,
                                      tree_begin, tree_end, d_out.p, b->ctx->num_sms, s));
    CUDA_CHECK(cudaMemcpyAsync(out + (size_t)r0 * T, d_out.p, (size_t)rows * T * sizeof(float), cudaMemcpyDeviceToHost, s));
  }
  CUDA_CHECK(cudaStreamSynchronize(s));
}

}  // namespace b2host
