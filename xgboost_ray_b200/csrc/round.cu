// round.cu -- one boosting round: label checks, the base_score estimate, gradients (objectives and learning to rank),
// the pipelined round (enqueue round r+1 before round r is drained), DART dropout and the refresh updater.
#include <math.h>

#include "host.h"
#include "launch.h"
#include "sampling.cuh"

namespace b2host __attribute__((visibility("hidden"))) {

// timing events of the round being enqueued
cudaEvent_t get_event(Booster* b) {
  Booster::RoundBuffers& R = b->rb[b->rb_cur];
  if (R.ev_used == R.ev_pool.size()) { cudaEvent_t e; CUDA_CHECK(cudaEventCreate(&e)); R.ev_pool.push_back(e); }
  return R.ev_pool[R.ev_used++];
}
void mark_phase(Booster* b, int phase) {
  if (b->p.profile < 2) return;
  cudaEvent_t e = get_event(b);
  CUDA_CHECK(cudaEventRecord(e, b->ctx->stream));
  b->rb[b->rb_cur].phase_marks.push_back({phase, e});
}
void resolve_events(Booster* b, Booster::RoundBuffers& R) {
  for (size_t i = 1; i < R.phase_marks.size(); ++i) {
    float ms = 0.f;
    if (R.phase_marks[i].first >= 0 && cudaEventElapsedTime(&ms, R.phase_marks[i - 1].second, R.phase_marks[i].second) == cudaSuccess)
      b->t.phase_ms[R.phase_marks[i].first] += ms;
  }
  R.phase_marks.clear();
  for (auto& pr : R.hist_events) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, pr.first, pr.second) == cudaSuccess) b->t.hist_ms += ms;
  }
  R.hist_events.clear();
  for (auto& pr : R.refresh_events) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, pr.first, pr.second) == cudaSuccess) b->t.refresh_ms += ms;
  }
  R.refresh_events.clear();
  R.ev_used = 0;
}

// the train matrix holds one label per row and target: a label whose width differs from the model's targets (set after
// the booster was created) names both
void check_train_labels(const Booster* b) {
  const Matrix* m = b->train; const int T = b->p.num_target;
  if (m->n_label > 0 && m->n_targets != T)
    fail("the train matrix's label has %d columns, the model has %d targets", m->n_targets, T);
  if (m->n_label != m->n * T) fail("train matrix has %lld labels for %lld rows", (long long)m->n_label, (long long)m->n);
}

void init_margin(Booster* b, float* margin, Matrix* m) {
  const int K = b->p.num_class; cudaStream_t s = b->ctx->stream;
  if (m->n_base_margin > 0) {
    if (m->n_base_margin != m->n * K) fail("base_margin has %lld values, expected %lld", (long long)m->n_base_margin, (long long)(m->n * K));
    CUDA_CHECK(cudaMemcpyAsync(margin, m->base_margin.p, (size_t)m->n * K * sizeof(float), cudaMemcpyDeviceToDevice, s));
  } else {
    LAUNCH_CHECK(b2_launch_fill(margin, m->n * K, base_margin_value(b->p), b->ctx->num_sms, s));
  }
}

// the n flags launch(bad) sets, maxed over the ranks so that every rank fails together (synchronises the stream)
template <typename Launch>
std::vector<uint32_t> check_flags(Booster* b, int n, Launch launch) {
  cudaStream_t s = b->ctx->stream;
  DevBuf<uint32_t> bad; bad.ensure(n);
  CUDA_CHECK(cudaMemsetAsync(bad.p, 0, n * sizeof(uint32_t), s));
  LAUNCH_CHECK(launch(bad.p));
  allreduce(b->comm, bad.p, n, kNcclUint32, kNcclMax, s);
  std::vector<uint32_t> h(n);
  CUDA_CHECK(cudaMemcpyAsync(h.data(), bad.p, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  return h;
}

// survival:aft reads the label bounds instead of the label: both present, no NaN, 0 <= lower (finite) <= upper, and an
// uncensored row (lower == upper) needs y > 0.  Once per train matrix, like check_labels.
void check_bounds(Booster* b) {
  Matrix* m = b->train;
  if (b->labels_checked) return;
  if (!m->has_bounds()) fail("survival:aft needs label_lower_bound and label_upper_bound");
  const std::vector<uint32_t> h = check_flags(b, 4, [&](uint32_t* bad) {
    return b2_launch_aft_bounds_check(m->lower.p, m->upper.p, m->n, bad, b->ctx->num_sms, b->ctx->stream);
  });
  if (h[0]) fail("survival:aft: label bounds must not be NaN");
  if (h[1]) fail("survival:aft: label_lower_bound must be finite and >= 0");
  if (h[2]) fail("survival:aft: label_upper_bound must be >= label_lower_bound");
  if (h[3]) fail("survival:aft: an uncensored row (lower == upper) needs a label > 0");
  b->labels_checked = true;
}

// the rank objectives need query groups and labels that are finite, >= 0 and, with the exponential gain, <= 31;
// rank:map needs binary relevance (0 or 1) and ignores ndcg_exp_gain
void check_rank_labels(Booster* b) {
  Matrix* m = b->train;
  if (!m->has_qgroups())
    fail("%s needs query groups on the train matrix: pass qid (or group) to the DMatrix", b->p.objective_name.c_str());
  if (b->labels_checked) return;
  check_train_labels(b);
  const bool map = b->p.objective == kObjRankMap;
  const std::vector<uint32_t> h = check_flags(b, 3, [&](uint32_t* bad) {
    return b2_launch_rank_label_check(m->label.p, m->n, !map && b->p.ndcg_exp_gain ? 1 : 0, map ? 1 : 0, bad,
                                      b->ctx->num_sms, b->ctx->stream);
  });
  if (h[2]) fail("rank:map: labels must be 0 or 1 (binary relevance); use rank:ndcg for graded relevance");
  if (h[0]) fail("%s: labels must be finite and >= 0", b->p.objective_name.c_str());
  if (h[1]) fail("%s: with ndcg_exp_gain the labels must be <= 31 (the gain is 2^label - 1); set ndcg_exp_gain=false "
                 "for larger relevance degrees", b->p.objective_name.c_str());
  b->labels_checked = true;
}

// discount table ln2 / log(r + 2) for model positions r < len
void ensure_rank_disc(Booster* b, int64_t len) {
  len = std::max<int64_t>(len, 1);
  if (b->rank_disc_len >= len) return;
  b->rank_disc.ensure((size_t)len);
  LAUNCH_CHECK(b2_launch_rank_disc(b->rank_disc.p, len, b->ctx->num_sms, b->ctx->stream));
  b->rank_disc_len = len;
}

// LambdaMART gradients of the train matrix (rank_kernel.cu): order the margins per group, then one pass over the groups
void rank_gradient(Booster* b, const float* margin, float2* gh, uint32_t* absmax, uint32_t* err) {
  Matrix* m = b->train; cudaStream_t s = b->ctx->stream; const Params& p = b->p; const int sms = b->ctx->num_sms;
  ensure_rank_disc(b, m->max_qgroup);
  const bool ndcg = p.objective == kObjRankNdcg;
  if (ndcg && (b->idcg_uid != m->uid || b->idcg_version != m->rank_version || b->idcg_k != p.rank_k ||
               b->idcg_gain != (int)p.ndcg_exp_gain)) {
    // 1/IDCG depends on the labels, k and the gain only: computed once per (matrix, k, gain)
    RankOrder lo;
    lo.run(m, m->label.p, sms, s);
    b->rank_inv_idcg.ensure((size_t)std::max<int64_t>(m->n_qgroups, 1));
    LAUNCH_CHECK(b2_launch_rank_inv_idcg(m->qgroup_ptr.p, m->n_qgroups, lo.keys_sorted.p, b->rank_disc.p, p.rank_k,
                                         p.ndcg_exp_gain ? 1 : 0, b->rank_inv_idcg.p, sms, s));
    CUDA_CHECK(cudaStreamSynchronize(s));   // lo's buffers go back to the pool
    b->idcg_uid = m->uid; b->idcg_version = m->rank_version; b->idcg_k = p.rank_k; b->idcg_gain = (int)p.ndcg_exp_gain;
  }
  b->rank_order.run(m, margin, sms, s);
  const bool map = p.objective == kObjRankMap;
  if (m->max_qgroup > b2_rank_stage_rows()) {
    const size_t rows = (size_t)std::max<int64_t>(m->n, 1);
    b->rank_scratch_m.ensure(rows); b->rank_scratch_y.ensure(rows); b->rank_scratch_p.ensure(rows);
    if (map) { b->rank_scratch_a.ensure(rows); b->rank_scratch_r.ensure(rows); }
  }
  const B2RankMode mode = map ? kRankMap : ndcg ? kRankNdcg : kRankPairwise;
  LAUNCH_CHECK(b2_launch_lambdarank_gradient(mode, m->qgroup_ptr.p, m->n_qgroups, m->max_qgroup,
                                             b->rank_order.keys_sorted.p, b->rank_order.rows.p, m->label.p,
                                             ndcg ? b->rank_inv_idcg.p : nullptr, b->rank_disc.p, p.rank_k,
                                             p.ndcg_exp_gain ? 1 : 0, b->rank_scratch_m.p, b->rank_scratch_y.p,
                                             b->rank_scratch_p.p, map ? b->rank_scratch_a.p : nullptr,
                                             map ? b->rank_scratch_r.p : nullptr, gh, absmax, err, sms, s));
}

// labels outside the objective's domain fail training (xgboost's CheckLabel); once per train matrix, before the first tree
void check_labels(Booster* b) {
  Matrix* m = b->train; const Params& p = b->p; const Objective& o = objective_row(p);
  if (o.labels == kLabelsBounds) { check_bounds(b); return; }
  if (o.labels == kLabelsRank) { check_rank_labels(b); return; }
  if (b->labels_checked) return;
  check_train_labels(b);
  const std::vector<uint32_t> h = check_flags(b, 1, [&](uint32_t* bad) {
    return b2_launch_label_check(p.objective, p.num_class, m->label.p, m->n * p.num_target, bad, b->ctx->num_sms,
                                 b->ctx->stream);
  });
  if (h[0]) fail(o.label_rule, p.objective_name.c_str(), p.num_class);
  b->labels_checked = true;
}

// the gradient pairs at margin [n][K] into gh [K][n]; nullable absmax (|g|, |h| maxima per class) and err (non-finite)
void objective_gradient(Booster* b, const float* margin, float2* gh, uint32_t* absmax, uint32_t* err) {
  Matrix* m = b->train; const Params& p = b->p; const Objective& o = objective_row(p);
  const float* w = m->n_weight ? m->weight.p : nullptr;
  const float param = o.param ? p.*o.param : 0.0f;
  const int K = p.num_class, sms = b->ctx->num_sms; cudaStream_t s = b->ctx->stream;
  if (o.grad == kGradRank)
    rank_gradient(b, margin, gh, absmax, err);
  else if (o.grad == kGradAft)
    LAUNCH_CHECK(b2_launch_gradient_aft(p.aft_dist, (double)p.aft_sigma, margin, m->lower.p, m->upper.p, w, m->n, gh,
                                        absmax, err, sms, s));
  else if (o.grad == kGradQuantile) {
    ensure_quantile_buffers(b, 1 << p.max_depth);
    LAUNCH_CHECK(b2_launch_gradient_quantile(K, b->d_alpha.p, margin, m->label.p, w, m->n, gh, absmax, sms, s));
  } else if (p.num_target > 1) {   // kGradScalar, one column per target
    LAUNCH_CHECK(b2_launch_gradient_multi_target(p.objective, K, margin, m->label.p, w, m->n, p.scale_pos_weight, param,
                                                 gh, absmax, err, sms, s));
  } else {   // kGradScalar and kGradSoftprob, one column per class
    LAUNCH_CHECK(b2_launch_gradient(p.objective, K, margin, m->label.p, w, m->n, p.scale_pos_weight, param, gh, absmax, err,
                                    sms, s));
  }
}

// base_score when the user gave none (xgboost >= 2.0: ObjFunction::InitEstimation -> FitIntercept, tree::FitStump;
// SURVEY.md A.3): one Newton step of a stump at margin 0, -sum(g)/sum(h) over ALL workers, then the inverse link.
// Sums are 40-bit fixed-point integers (exact below 2^31 rows), so every rank (and the oracle) computes the same value.
void estimate_base_score(Booster* b) {
  Matrix* m = b->train; cudaStream_t s = b->ctx->stream; Params& p = b->p; const Objective& o = objective_row(p);
  if (p.base_score_set || o.intercept == kInterceptNone) { p.base_score_set = true; return; }
  // existing trees were fitted around the intercept of the model they came from: never assume the default for them
  if (!b->trees.empty()) fail("continuing from existing trees needs an explicit base_score (the source model's intercept)");
  check_train_labels(b);
  const int64_t n = m->n;
  b->d_absmax.ensure(2); b->d_qexp.ensure(2);
  if (o.intercept == kInterceptQuantile) {
    // the fp32 mean over k of the weighted alpha_k-quantile of the labels (the leaf refresh's selection, one segment)
    const int K = p.num_class;
    ensure_quantile_buffers(b, 1);
    DevBuf<float2> gq; DevBuf<float> q;
    gq.ensure((size_t)std::max<int64_t>(n, 1)); q.ensure((size_t)K);
    CUDA_CHECK(cudaMemsetAsync(q.p, 0, (size_t)K * sizeof(float), s));
    for (int k = 0; k < K; ++k) {
      LAUNCH_CHECK(b2_launch_gradient_quantile(1, b->d_alpha.p + k, nullptr, m->label.p, m->n_weight ? m->weight.p : nullptr, n,
                                               gq.p, nullptr, b->ctx->num_sms, s));
      CUDA_CHECK(cudaMemsetAsync(b->d_absmax.p, 0, 2 * sizeof(uint32_t), s));
      LAUNCH_CHECK(b2_launch_absmax(gq.p, n, b->d_absmax.p, b->ctx->num_sms, s));
      allreduce(b->comm, b->d_absmax.p, 2, kNcclUint32, kNcclMax, s);
      LAUNCH_CHECK(b2_launch_quant_exponent(b->d_absmax.p, b->d_qexp.p, s));
      quantile_select(b, k, nullptr, nullptr, gq.p, b->d_qexp.p, b->d_one.p, 1, 1.0f, nullptr, q.p + k, nullptr);
    }
    std::vector<float> h((size_t)K);
    CUDA_CHECK(cudaMemcpyAsync(h.data(), q.p, (size_t)K * sizeof(float), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    float sum = 0.0f;
    for (float v : h) sum += v;
    p.base_score = sum / (float)K;
    p.base_score_set = true;
    return;
  }
  // T targets (DESIGN.md 2 item 18): one stump per target from its own slice of the class-major pairs, with its own
  // exponents; the intercept is the fp32 sum over k, in k order, of fp32(stump_k / T) (stump_0 itself for T = 1)
  const int T = p.num_target;
  const size_t nt = (size_t)std::max<int64_t>(n * T, 1);
  DevBuf<float> zeros; DevBuf<float2> gh; DevBuf<long long> sums;
  zeros.ensure(nt); gh.ensure(nt); sums.ensure(4);
  CUDA_CHECK(cudaMemsetAsync(zeros.p, 0, nt * sizeof(float), s));
  objective_gradient(b, zeros.p, gh.p, nullptr, nullptr);
  auto limbs_to_double = [](long long hi, long long lo) {   // b2_limbs_to_double on the host: one rounding
    hi += lo >> B2_LIMB_SHIFT; lo &= (1ll << B2_LIMB_SHIFT) - 1;
    return (double)hi * (double)(1ll << B2_LIMB_SHIFT) + (double)lo;
  };
  float stump = 0.0f;
  for (int k = 0; k < T; ++k) {
    const float2* ghk = gh.p + (size_t)k * n;
    CUDA_CHECK(cudaMemsetAsync(b->d_absmax.p, 0, 2 * sizeof(uint32_t), s));
    LAUNCH_CHECK(b2_launch_absmax(ghk, n, b->d_absmax.p, b->ctx->num_sms, s));
    allreduce(b->comm, b->d_absmax.p, 2, kNcclUint32, kNcclMax, s);
    LAUNCH_CHECK(b2_launch_quant_exponent(b->d_absmax.p, b->d_qexp.p, s));
    CUDA_CHECK(cudaMemsetAsync(sums.p, 0, 4 * sizeof(long long), s));
    LAUNCH_CHECK(b2_launch_sum_fixed(ghk, n, b->d_qexp.p, 40, sums.p, b->ctx->num_sms, s));
    allreduce(b->comm, sums.p, 4, kNcclInt64, kNcclSum, s);   // [g, h][hi, lo] limbs (common.cuh): exact over all ranks
    long long h_s[4]; int32_t h_e[2];
    CUDA_CHECK(cudaMemcpyAsync(h_s, sums.p, sizeof(h_s), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaMemcpyAsync(h_e, b->d_qexp.p, sizeof(h_e), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    const double G = limbs_to_double(h_s[0], h_s[1]) / ldexp(1.0, 40 - h_e[0]);
    const double H = limbs_to_double(h_s[2], h_s[3]) / ldexp(1.0, 40 - h_e[1]);
    const float stump_k = H <= 1e-6 ? 0.0f : (float)(-G / H);
    stump = k == 0 ? stump_k / (float)T : stump + stump_k / (float)T;
  }
  if (o.link == kLinkSigmoid || o.link == kLinkExp) {
    // margin -> output space with the engine's own sigmoid / exp (same IEEE sequence as the kernels): evaluated on the device
    DevBuf<float> one; one.ensure(1);
    CUDA_CHECK(cudaMemcpyAsync(one.p, &stump, sizeof(float), cudaMemcpyHostToDevice, s));
    LAUNCH_CHECK(b2_launch_transform(p.objective, 1, one.p, 1, b->ctx->num_sms, s));
    float prob = 0.5f;
    CUDA_CHECK(cudaMemcpyAsync(&prob, one.p, sizeof(float), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    p.base_score = prob;
  } else {
    p.base_score = stump;
  }
  p.base_score_set = true;
}

// update mode: tree to_update[src] with the statistics of its refresh_nodes_kernel block.  Structure, splits, default
// directions and categories are the old tree's; a leaf keeps its loss_chg (xgboost's refresher sets it on splits only).
void materialize_refreshed(Booster* b, const void* block, int src) {
  TreeHost t = b->to_update[src];
  const int nn = t.size();
  const double* sum_hess = (const double*)block;
  const float* base_weight = (const float*)((const char*)block + (size_t)nn * 8);
  const float* loss_chg = base_weight + nn;
  const float* value = loss_chg + nn;
  for (int i = 0; i < nn; ++i) {
    t.sum_hess[i] = sum_hess[i];
    t.base_weight[i] = base_weight[i];
    t.value[i] = value[i];
    if (t.feature[i] >= 0) t.loss_chg[i] = loss_chg[i];
  }
  b->trees.push_back(std::move(t));
}

// Finish an enqueued round: wait for its stop event, resolve its timers, raise a peer-memory or non-finite-gradient
// error, and turn its read-back blocks into host trees.
void finish_round(Booster* b, Booster::RoundBuffers& R, int n_trees, bool check_finite) {
  CUDA_CHECK(cudaEventSynchronize(R.stop));
  if (b->p.profile) {
    float ms = 0.f; CUDA_CHECK(cudaEventElapsedTime(&ms, R.start, R.stop));
    b->t.round_ms += ms;
    resolve_events(b, R);
  }
  if (b->p2p.enabled && *R.h_p2p_err) {
    const uint32_t perr = *R.h_p2p_err;
    fail("peer-memory exchange: %s while waiting for another rank (flag slot %u)",
         b->comm && b->comm->aborted.load() ? "communicator aborted" : "timed out", perr - 1);
  }
  if (check_finite && *b->h_grad_err) {
    // the trees of this round were grown with those rows zeroed and are dropped; the train margin already holds their
    // leaves, so it is rebuilt from the kept trees before the next round
    b->margin_ready = false;
    fail("%s: a gradient or hessian is not finite (the margin left the range where the objective's exp is finite)",
         b->p.objective_name.c_str());
  }
  for (int slot = 0; slot < n_trees; ++slot) {
    if (R.refresh) materialize_refreshed(b, R.rstaging[slot], R.rsrc[slot]);
    else if (b->p.vector_leaf()) materialize_vector_tree(b, R.staging[slot], R.vstaging);
    else materialize_tree(b, R.staging[slot]);
  }
  if (b->p.dart) {   // the weights are committed with the trees
    b->tree_w = R.dart_w;
    if (R.dart_dropped) b->weights_version++;
  }
  b->t.rounds++;
}
// Finish the round boost_round left pending.  Every entry point that reads the trees, the timers, the margin or the
// gradients calls this first.  The round stops being pending before anything can throw, so an error is raised once.
void drain_round(Booster* b) {
  const int n_trees = b->pending_trees;
  if (n_trees == 0) return;
  b->pending_trees = 0;
  finish_round(b, b->rb[b->rb_cur ^ 1], n_trees, b->pending_check_finite);
}

// B2_BoosterCreate: a booster that trains on m, or without m a prediction-only one (num_feature=<n> in params)
Booster* new_booster(const char* params, Matrix* m, Comm* comm) {
  std::unique_ptr<Booster> b(new Booster()); b->kind = kBooster; b->train = m; b->comm = comm;
  parse_params(params, &b->p, nullptr);
  if (m) {
    // the train matrix's label fixes the targets; a loaded model (num_target) must have as many
    if (b->p.num_target_set && b->p.num_target != m->n_targets)
      fail("the model has %d targets, the train matrix's label has %d columns", b->p.num_target, m->n_targets);
    set_targets(&b->p, m->n_targets);
    if (b->p.vector_leaf() && m->any_cat())
      fail("multi_strategy=multi_output_tree is not supported with categorical features (the train matrix has %zu)",
           m->cat_feats.size());
    b->ctx = m->ctx; b->n_features = m->F; CUDA_CHECK(cudaSetDevice(m->ctx->device));
    check_level_memory(b.get());
    if (!b->p.interaction_sets.empty()) {   // sets_of[f] bit k: feature f is in set k
      const int W = (int)((b->p.interaction_sets.size() + 63) / 64);
      std::vector<unsigned long long> sets_of((size_t)m->F * W, 0ull);
      for (size_t k = 0; k < b->p.interaction_sets.size(); ++k)
        for (int64_t f : b->p.interaction_sets[k]) {
          if (f >= m->F) fail("interaction_constraints: feature index %lld is out of range for %d features", (long long)f, m->F);
          sets_of[(size_t)f * W + k / 64] |= 1ull << (k % 64);
        }
      upload(b->d_ic_sets_of, sets_of, m->ctx->stream);   // pageable source: staged before return
      b->ic_words = W;
    }
  }
  else {  // prediction-only booster (model loaded with B2_BoosterAddTree)
    if (b->p.num_feature <= 0) fail("a booster without a train matrix needs num_feature=<n> in params");
    b->ctx = get_ctx(b->p.device); b->n_features = b->p.num_feature;
  }
  return b.release();
}

// B2_BoosterSetParam (DESIGN.md 2 item 22).  Every rule is checked before anything changes.  The pending round was
// enqueued with the old values and its host-side finish reads them (materialize_tree's base weights, the vector leaves'
// eta), so it is finished first; the next round is the first one to use the new values.
void set_booster_params(Booster* b, const char* params) {
  const Params q = changed_params(b->p, params);
  if (!b->train) { b->p = q; return; }   // prediction-only: nothing is pending or captured
  CUDA_CHECK(cudaSetDevice(b->ctx->device));
  drain_round(b);
  const Params old = b->p;
  b->p = q;
  if (q.eta != old.eta) b->dart_next.r = -1;   // DART's next-round weights normalise by eta
  tree_params_changed(b, old);
}

// Update mode, before anything reads the train margin: the trees added so far become the trees to update and the model
// starts empty (xgboost's gbtree moves them to trees_to_update).  Beyond check_tree, every node of a tree must be
// reached from node 0, each once, and a tree has at most 65,536 leaves (compact indices 0..65,535 fit pos).  The trees
// are copied to the device once: B2TreeNodeDev nodes whose pad holds the compact leaf index (leaves numbered in node
// order), the category sets, and the node ids grouped by depth.
void begin_update(Booster* b) {
  if (!b->p.update_mode || b->update_started) return;
  drain_round(b);
  b->update_started = true;
  b->to_update = std::move(b->trees);
  b->trees.clear();
  trees_edited(b);
  std::vector<B2TreeNodeDev> nodes; std::vector<uint32_t> cats; std::vector<int32_t> order, levels;
  size_t max_leaves = 1, max_nodes = 1, max_block = 8;
  b->rtrees.clear();
  for (size_t ti = 0; ti < b->to_update.size(); ++ti) {
    const TreeHost& t = b->to_update[ti];
    const int nn = t.size();
    Booster::RefreshTree rt;
    rt.node_off = (int32_t)nodes.size(); rt.n_nodes = nn; rt.level_off = (int32_t)levels.size();
    rt.order_off = (int32_t)order.size();
    std::vector<int32_t> leaf_of(nn, -1), depth(nn, -1);
    int n_leaves = 0;
    for (int i = 0; i < nn; ++i) if (t.feature[i] < 0) leaf_of[i] = n_leaves++;
    if (n_leaves > 65536) fail("tree %zu has %d leaves; the refresh updater supports at most 65536", ti, n_leaves);
    // breadth-first from the root (check_tree: the children are nodes, no split is reached twice): every node reached,
    // a leaf only once
    std::vector<int32_t> bfs{0}; depth[0] = 0;
    for (size_t q = 0; q < bfs.size(); ++q) {
      const int i = bfs[q];
      if (t.feature[i] < 0) continue;
      for (int c : {t.left[i], t.right[i]}) {
        if (depth[c] >= 0) fail("tree %zu is not a binary tree: node %d is reached twice from the root", ti, c);
        depth[c] = depth[i] + 1;
        bfs.push_back(c);
      }
    }
    if ((int)bfs.size() != nn) fail("tree %zu has %d nodes that the root does not reach", ti, nn - (int)bfs.size());
    const int n_levels = depth[bfs.back()] + 1;   // BFS order is by depth
    rt.n_leaves = n_leaves; rt.n_levels = n_levels;
    int d = -1;
    for (size_t q = 0; q < bfs.size(); ++q)
      while (d < depth[bfs[q]]) { levels.push_back((int32_t)(order.size() + q)); ++d; }
    levels.push_back((int32_t)(order.size() + bfs.size()));
    order.insert(order.end(), bfs.begin(), bfs.end());
    for (int i = 0; i < nn; ++i) {
      int32_t cat_slot = -1;
      if (t.feature[i] >= 0 && t.split_type[i]) {
        cat_slot = (int32_t)(cats.size() / 8);
        cats.insert(cats.end(), t.cat_bits.begin() + (size_t)i * 8, t.cat_bits.begin() + (size_t)i * 8 + 8);
      }
      nodes.push_back(B2TreeNodeDev{t.left[i], t.right[i], t.feature[i], t.cond[i], t.value[i], (int32_t)t.default_left[i],
                                    cat_slot, leaf_of[i]});
    }
    rt.block_bytes = (size_t)nn * (8 + 3 * 4);
    max_leaves = std::max(max_leaves, (size_t)n_leaves); max_nodes = std::max(max_nodes, (size_t)nn);
    max_block = std::max(max_block, rt.block_bytes);
    b->rtrees.push_back(rt);
  }
  // node ids are relative to the tree, level pointers relative to the tree's segment of the order table
  for (const Booster::RefreshTree& rt : b->rtrees)
    for (int l = 0; l <= rt.n_levels; ++l) levels[rt.level_off + l] -= rt.order_off;
  cudaStream_t s = b->ctx->stream;
  upload(b->d_rnodes, nodes, s); upload(b->d_rorder, order, s); upload(b->d_rlevels, levels, s);
  if (cats.empty()) cats.assign(8, 0u);
  upload(b->d_rcats, cats, s);
  b->d_rsums.ensure(4 * max_leaves); b->d_rlimbs.ensure(4 * max_nodes); b->d_rleaf.ensure(max_leaves);
  b->d_rblock.ensure(max_block);
  CUDA_CHECK(cudaStreamSynchronize(s));
  b->rstaging_bytes = max_block;
}

// DART walks the train matrix's bins: every numeric split of a tree must name the bin whose cut is its condition (trees
// grown by this engine on these cuts do; a model from elsewhere, or one continued on a matrix with other cuts, does not)
void check_dart_split_bins(Booster* b) {
  const Matrix* m = b->train;
  for (size_t ti = 0; ti < b->trees.size(); ++ti) {
    const TreeHost& t = b->trees[ti];
    for (int i = 0; i < t.size(); ++i) {
      const int f = t.feature[i];
      if (f < 0 || t.split_type[i]) continue;
      const int sb = t.split_bin[i];
      const bool ok = sb < 0 ? (sb == -1 && t.cond[i] == m->min_vals[f])
                             : (sb < m->nbins[f] && t.cond[i] == m->cut_vals[m->cut_ptrs[f] + sb]);
      if (!ok)
        fail("continuing a DART model needs the split bins of the train matrix's cuts: tree %zu node %d (feature %d, "
             "condition %g) has none; continue on the matrix the model was trained on, with the model this engine wrote",
             ti, i, f, (double)t.cond[i]);
    }
  }
}

// Rebuild margins of the train rows from the trees on the device (dart_kernel.cu): drop (nullable) without the trees
// flagged in dropped, with weights w_old; full with weights w_full.  Both hold the starting margin on entry.
void dart_margins(Booster* b, const std::vector<float>& w_old, const std::vector<uint8_t>& dropped,
                  const std::vector<float>& w_full, float* drop, float* full) {
  Matrix* m = b->train; cudaStream_t s = b->ctx->stream; const int T = (int)b->trees.size();
  sync_device_trees(b);
  upload(b->d_dart_w_full, w_full, s);
  if (drop) { upload(b->d_dart_w_old, w_old, s); upload(b->d_dart_dropped, dropped, s); }
  LAUNCH_CHECK(b2_launch_dart_margins(bin_source(m), m->n, m->d_has_missing.p, b->d_nodes.p, b->d_tree_offset.p,
                                      b->d_cat_table.p, T, b->p.num_class, b->p.num_parallel_tree,
                                      drop ? b->d_dart_w_old.p : nullptr, drop ? b->d_dart_dropped.p : nullptr,
                                      b->d_dart_w_full.p, drop, full, b->ctx->num_sms, s));
}

void ensure_train_margin(Booster* b) {
  begin_update(b);
  if (b->margin_ready) return;
  drain_round(b);   // the margin is rebuilt from every tree of the model
  Matrix* m = b->train;
  check_labels(b);
  estimate_base_score(b);
  b->margin.ensure((size_t)std::max<int64_t>(m->n * b->p.num_class, 1));
  init_margin(b, b->margin.p, m);
  b->dart_next.r = -1;
  if (!b->trees.empty() && b->p.dart) {
    check_dart_split_bins(b);
    dart_margins(b, {}, {}, b->tree_w, nullptr, b->margin.p);
  } else if (!b->trees.empty()) {
    if (!m->has_raw) fail("continuing training from existing trees needs the raw data of the train matrix (B2_MatrixEnsureRaw)");
    predict_trees(b, m, 0, (int)b->trees.size(), b->margin.p);
  }
  b->margin_ready = true;
}

// The DART drop set of round r over trees with weights w (DESIGN.md 2): u_j = hash(seed, r, j, B2_SCOPE_DART) / 2^32.
// Keyed by the round, never by the rank, so every worker drops the same trees and a restart replays the same drops.
std::vector<uint8_t> dart_drop_set(const Params& p, uint32_t r, const std::vector<float>& w) {
  const size_t T = w.size();
  std::vector<uint8_t> dropped(T, 0);
  if (T == 0) return dropped;
  auto u = [&](uint32_t j) { return (double)b2_hash4((uint32_t)p.seed, r, j, B2_SCOPE_DART) * 0x1p-32; };
  if (p.skip_drop > 0.0 && u(0xFFFFFFFFu) < p.skip_drop) return dropped;
  // S > 0: the newest trees of a trained model have positive weights, and B2_BoosterSetTreeWeights refuses a total
  // that is not finite and positive
  float S = 0.0f;
  for (float x : w) S += x;   // binary32, in tree order
  size_t k = 0;
  for (size_t t = 0; t < T; ++t) {
    const double thr = p.dart_weighted ? p.rate_drop * (double)T * (double)w[t] / (double)S : p.rate_drop;
    if (u((uint32_t)t) < thr) { dropped[t] = 1; ++k; }
  }
  if (p.one_drop && k == 0) {
    const double v = u(0xFFFFFFFEu);
    size_t pick = T - 1;
    if (!p.dart_weighted) {
      pick = std::min(T - 1, (size_t)floor(v * (double)T));
    } else {
      double cum = 0.0;
      for (size_t t = 0; t < T; ++t) { cum += (double)w[t]; if (cum > v * (double)S) { pick = t; break; } }
    }
    dropped[pick] = 1;
  }
  return dropped;
}

// Decide the next round's drops (once per round: B2_BoosterGetTrainMargin and the round itself share the decision) and,
// when it drops trees, rebuild its drop margin and full-margin prefix in one pass over the bin matrix.  The weights
// before the round include a pending round's; a dropping round needs that round's trees on the device, so it is drained.
void dart_prepare(Booster* b) {
  ensure_train_margin(b);
  const Params& p = b->p; const int K = p.num_class, npt = p.num_parallel_tree;
  const int64_t T = (int64_t)b->trees.size() + b->pending_trees;
  const int64_t r = T / (K * npt);
  Booster::DartNext& dn = b->dart_next;
  if (dn.r == r && (int64_t)dn.dropped.size() == T) return;
  const std::vector<float> w = b->pending_trees ? b->rb[b->rb_cur ^ 1].dart_w : b->tree_w;
  if ((int64_t)w.size() != T) fail("DART: %zu tree weights for %lld trees", w.size(), (long long)T);
  dn.dropped = dart_drop_set(p, (uint32_t)r, w);
  dn.n_dropped = 0;
  for (uint8_t d : dn.dropped) dn.n_dropped += d;
  // normalisation (Dart::NormalizeTrees) for the round's n_new trees
  const int n_new = K * npt;
  const float lr = (float)((double)p.eta / (double)n_new);
  const int k = dn.n_dropped;
  float w_new = 1.0f;
  dn.w_after = w;
  if (k > 0) {
    const float f = p.dart_forest ? (float)(1.0 / (1.0 + (double)lr)) : (float)((double)k / ((double)k + (double)lr));
    for (int64_t t = 0; t < T; ++t) if (dn.dropped[t]) dn.w_after[t] *= f;
    w_new = p.dart_forest ? f : (float)(1.0 / ((double)k + (double)lr));
  }
  dn.w_after.insert(dn.w_after.end(), n_new, w_new);
  if (k > 0) {
    drain_round(b);   // the weights of the drained round are w
    Matrix* m = b->train;
    const size_t nk = (size_t)std::max<int64_t>(m->n * K, 1);
    b->dart_drop.ensure(nk); b->dart_prefix.ensure(nk);
    init_margin(b, b->dart_drop.p, m);
    init_margin(b, b->dart_prefix.p, m);
    dart_margins(b, w, dn.dropped, std::vector<float>(dn.w_after.begin(), dn.w_after.begin() + T), b->dart_drop.p,
                 b->dart_prefix.p);
    b->t.kernel_launches++;
  }
  dn.r = r;
}

// Update mode: refresh tree to_update[src] (class k) from gh[k] on the raw train rows, update margin[:, k] with its
// leaf values and copy its statistics into pinned block `slot` (materialize_refreshed, when the round is drained).
// Every row counts (no row or column sampling); the leaf sums are the only exchange between the ranks.
void refresh_tree(Booster* b, int k, int slot, int src) {
  Matrix* m = b->train; Ctx* ctx = b->ctx; cudaStream_t s = ctx->stream; const Params& p = b->p;
  const int64_t n = m->n;
  const Booster::RefreshTree& rt = b->rtrees[src];
  const float2* gh = b->gh.p + (size_t)k * n;
  uint32_t* d_absmax = b->d_absmax.p + 2 * k;
  b->pos.ensure((size_t)std::max<int64_t>(n, 1));
  Booster::RoundBuffers& R = b->rb[b->rb_cur];
  while ((int)R.rstaging.size() <= slot) {
    void* h = nullptr; CUDA_CHECK(cudaMallocHost(&h, b->rstaging_bytes)); R.rstaging.push_back(h);
  }
  if (!b->absmax_fused) {
    CUDA_CHECK(cudaMemsetAsync(d_absmax, 0, 2 * sizeof(uint32_t), s));
    LAUNCH_CHECK(b2_launch_absmax(gh, n, d_absmax, ctx->num_sms, s));
    b->t.kernel_launches++;
  }
  allreduce(b->comm, d_absmax, 2, kNcclUint32, kNcclMax, s);
  LAUNCH_CHECK(b2_launch_quant_exponent(d_absmax, b->d_qexp.p, s));
  CUDA_CHECK(cudaMemsetAsync(b->d_rsums.p, 0, 4 * (size_t)rt.n_leaves * sizeof(long long), s));
  const B2TreeNodeDev* nodes = b->d_rnodes.p + rt.node_off;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (p.profile) { e0 = get_event(b); e1 = get_event(b); CUDA_CHECK(cudaEventRecord(e0, s)); }
  LAUNCH_CHECK(b2_launch_refresh(raw_source(m), n, m->F, m->missing, nodes, rt.n_nodes, b->d_rcats.p, rt.n_leaves, gh, b->d_qexp.p,
                                 40, b->pos.p, b->d_rsums.p, ctx->num_sms, s));
  if (p.profile) { CUDA_CHECK(cudaEventRecord(e1, s)); R.refresh_events.push_back({e0, e1}); }
  b->t.refresh_launches++;
  allreduce(b->comm, b->d_rsums.p, 4 * (size_t)rt.n_leaves, kNcclInt64, kNcclSum, s);   // limb by limb: exact
  if (b->comm && b->comm->world > 1) b->t.allreduce_bytes += 4.0 * rt.n_leaves * 8;
  const B2CtlParams cp = ctl_params(p);
  LAUNCH_CHECK(b2_launch_refresh_nodes(nodes, rt.n_nodes, b->d_rorder.p + rt.order_off, b->d_rlevels.p + rt.level_off, rt.n_levels,
                                       b->d_rsums.p, b->d_qexp.p, 40, cp, p.refresh_leaf ? 1 : 0, b->d_rlimbs.p, b->d_rblock.p,
                                       b->d_rleaf.p, s));
  LAUNCH_CHECK(b2_launch_margin_update(b->margin.p, p.num_class, k, b->pos.p, b->d_rleaf.p, nullptr, n, ctx->num_sms, s));
  CUDA_CHECK(cudaMemcpyAsync(R.rstaging[slot], b->d_rblock.p, rt.block_bytes, cudaMemcpyDeviceToHost, s));
  b->t.kernel_launches += 4;
}

// One boosting round, pipelined with the previous one: round r+1 (gradients, then its class trees) is enqueued first,
// round r is drained while the device works on r+1, and r+1 is left pending.  Nothing of r+1 needs the host: the margin
// it reads was updated on the device by r's margin_update_kernel, in stream order.  A round whose gradient kernel checks
// finiteness is drained before returning, so that its error is raised by its own call and its trees never exist.
void boost_round(Booster* b, const float* custom_g, const float* custom_h, int64_t len) {
  if (!b->train) fail("this booster has no train matrix (prediction-only)");
  Matrix* m = b->train; cudaStream_t s = b->ctx->stream; const int K = b->p.num_class; const int64_t n = m->n;
  CUDA_CHECK(cudaSetDevice(b->ctx->device));
  if (b->cancel.load()) { drain_round(b); fail("training cancelled"); }
  Booster::RoundBuffers& R = b->rb[b->rb_cur];   // not pending: the pending round (if any) is in the other set
  R.hist_events.clear(); R.refresh_events.clear(); R.phase_marks.clear(); R.ev_used = 0;   // left over from a round that failed while enqueuing
  if (!R.start) { CUDA_CHECK(cudaEventCreate(&R.start)); CUDA_CHECK(cudaEventCreate(&R.stop)); }
  if (b->p.profile) CUDA_CHECK(cudaEventRecord(R.start, s));
  ensure_train_margin(b);
  // update mode: round r refreshes the r-th round of the model's trees (refresh_tree) instead of growing new ones
  const bool refresh = b->p.update_mode;
  int refresh_round_index = 0;
  if (refresh) {
    const int per_round = K * b->p.num_parallel_tree;
    const int64_t have = (int64_t)b->to_update.size();
    if (have == 0) fail("process_type=update needs the trees of an existing model (xgb_model); this booster has none");
    if (have % per_round != 0)
      fail("the model to update has %lld trees, not a whole number of rounds of %d trees", (long long)have, per_round);
    if (!m->has_raw) fail("process_type=update needs the raw data of the train matrix (B2_MatrixEnsureRaw)");
    refresh_round_index = (int)(((int64_t)b->trees.size() + b->pending_trees) / per_round);
    if (refresh_round_index >= have / per_round)
      fail("the model to update has %lld rounds; process_type=update cannot refresh round %d (num_boost_round must be at "
           "most %lld)", (long long)(have / per_round), refresh_round_index + 1, (long long)(have / per_round));
  }
  R.refresh = refresh;
  // DART: the gradients are taken at the drop margin; the round's trees are added to the full-margin prefix
  const float* gm = b->margin.p;
  if (b->p.dart) {
    dart_prepare(b);
    const float w_new = b->dart_next.w_after.back();
    b->d_dart_w_new.ensure(1);
    CUDA_CHECK(cudaMemcpyAsync(b->d_dart_w_new.p, &w_new, sizeof(float), cudaMemcpyHostToDevice, s));   // staged before return
    if (b->dart_next.n_dropped > 0) {
      gm = b->dart_drop.p;
      CUDA_CHECK(cudaMemcpyAsync(b->margin.p, b->dart_prefix.p, (size_t)n * K * sizeof(float), cudaMemcpyDeviceToDevice, s));
    }
    R.dart_w = b->dart_next.w_after; R.dart_dropped = b->dart_next.n_dropped > 0;
    b->dart_next.r = -1;
  }
  b->gh.ensure((size_t)std::max<int64_t>(n * K, 1));
  b->d_absmax.ensure(2 * (size_t)K); b->d_qexp.ensure(2);
  b->absmax_fused = false;
  const Objective& o = objective_row(b->p);
  b->refresh_leaves = !custom_g && o.grad == kGradQuantile;
  bool check_finite = false;
  if (custom_g) {
    if (len != n * K) fail("custom gradient has %lld values, expected %lld", (long long)len, (long long)(n * K));
    b->d_custom_g.ensure((size_t)std::max<int64_t>(len, 1)); b->d_custom_h.ensure((size_t)std::max<int64_t>(len, 1));
    CUDA_CHECK(cudaMemcpyAsync(b->d_custom_g.p, custom_g, len * sizeof(float), cudaMemcpyHostToDevice, s));
    CUDA_CHECK(cudaMemcpyAsync(b->d_custom_h.p, custom_h, len * sizeof(float), cudaMemcpyHostToDevice, s));
    LAUNCH_CHECK(b2_launch_pack_custom(b->d_custom_g.p, b->d_custom_h.p, K, n, b->gh.p, b->ctx->num_sms, s));
  } else {
    if (o.labels != kLabelsBounds) check_train_labels(b);
    // the |g|,|h| maxima of every class tree come out of the same pass unless rows are dropped afterwards (subsample)
    b->absmax_fused = (b->p.subsample >= 1.0f || refresh) && K <= b2_gradient_fused_max_classes();
    if (b->absmax_fused) CUDA_CHECK(cudaMemsetAsync(b->d_absmax.p, 0, 2 * (size_t)K * sizeof(uint32_t), s));
    check_finite = o.checks_finite;
    if (check_finite) {
      if (!b->h_grad_err) { CUDA_CHECK(cudaMallocHost(&b->h_grad_err, sizeof(uint32_t))); b->d_grad_err.ensure(1); }
      CUDA_CHECK(cudaMemsetAsync(b->d_grad_err.p, 0, sizeof(uint32_t), s));
    }
    objective_gradient(b, gm, b->gh.p, b->absmax_fused ? b->d_absmax.p : nullptr, check_finite ? b->d_grad_err.p : nullptr);
  }
  b->gh_ready = true;
  b->t.kernel_launches++;
  const int npt = b->p.num_parallel_tree;
  // row sampling zeroes the dropped rows' gradient pairs in place: the parallel trees of a round each sample from the
  // round's ORIGINAL gradients, so those are kept aside and restored in front of every further tree
  const bool restore_gh = npt > 1 && b->p.subsample < 1.0f && !refresh;
  if (restore_gh) {
    b->gh_round.ensure((size_t)std::max<int64_t>(n * K, 1));
    CUDA_CHECK(cudaMemcpyAsync(b->gh_round.p, b->gh.p, (size_t)n * K * sizeof(float2), cudaMemcpyDeviceToDevice, s));
  }
  const int round_trees = b->p.vector_leaf() ? 1 : K * npt;   // a vector-leaf tree covers every target
  if (refresh) {
    R.rsrc.resize(round_trees);
    for (int slot = 0; slot < round_trees; ++slot) {
      R.rsrc[slot] = refresh_round_index * round_trees + slot;
      refresh_tree(b, slot / npt, slot, R.rsrc[slot]);
    }
  } else if (b->p.vector_leaf()) run_tree(b, 0, 0);
  else
  for (int k = 0; k < K; ++k)
    for (int j = 0; j < npt; ++j) {
      if (restore_gh && j > 0)
        CUDA_CHECK(cudaMemcpyAsync(b->gh.p + (size_t)k * n, b->gh_round.p + (size_t)k * n, (size_t)n * sizeof(float2), cudaMemcpyDeviceToDevice, s));
      run_tree(b, k, k * npt + j);
    }
  if (check_finite) {
    // every rank fails the round together; the flag is read back when the round is drained (pinned memory: the copy
    // is ordered on the stream)
    allreduce(b->comm, b->d_grad_err.p, 1, kNcclUint32, kNcclMax, s);
    CUDA_CHECK(cudaMemcpyAsync(b->h_grad_err, b->d_grad_err.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  }
  if (b->p2p.enabled) {
    if (!R.h_p2p_err) CUDA_CHECK(cudaMallocHost(&R.h_p2p_err, sizeof(uint32_t)));
    CUDA_CHECK(cudaMemcpyAsync(R.h_p2p_err, b->p2p.pp.err, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  }
  CUDA_CHECK(cudaEventRecord(R.stop, s));
  // this round is queued behind the previous one: make it the pending round, then finish the previous one while the
  // device works (its buffers are the set the next round enqueues into)
  const int prev_trees = b->pending_trees; const bool prev_check = b->pending_check_finite;
  b->pending_trees = round_trees; b->pending_check_finite = check_finite;
  b->rb_cur ^= 1;
  if (prev_trees) finish_round(b, b->rb[b->rb_cur], prev_trees, prev_check);
  if (check_finite) drain_round(b);
}

}  // namespace b2host
