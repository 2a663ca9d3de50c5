// params.cu -- the booster parameters: parsing the "key=value" text of B2_BoosterCreate and B2_CheckParams with every
// rule about which parameters go together, the objective table, the host replicas of the leaf-weight formula, and the
// eval_metric names.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <tuple>

#include "host.h"

namespace b2host __attribute__((visibility("hidden"))) {

// the label_rule messages; a class label is an index (non-integer labels truncate like xgboost's, NaN is rejected)
constexpr char kIn01[] = "label must be in [0, 1] for %s", kNonneg[] = "label must be nonnegative for %s",
               kAboveMinus1[] = "label must be greater than -1 for %s", kPositive[] = "label must be positive for %s",
               kFinite[] = "label must be finite for %s",
               kClassIndex[] = "label must be in [0, num_class) for %s, num_class = %d";

// Every accepted objective name.  Every objective has a label rule: the ones without a narrower domain need a finite
// label (kFinite), so that a NaN or infinite label fails training instead of reaching the gradient pairs, their
// quantisation scale or the intercept.  reg:quantileerror's gradient pairs are finite for finite labels and weights
// (both checked before the first round), so its rounds stay pipelined.
constexpr Objective kObjectives[] = {
  // name, id, link, grad, param, multi_target, checks_finite, labels, intercept[, label_rule]
  {"reg:squarederror", kObjSquaredError, kLinkIdentity, kGradScalar, nullptr, true, false, kLabelsDomain, kInterceptStump, kFinite},
  {"reg:linear", kObjSquaredError, kLinkIdentity, kGradScalar, nullptr, true, false, kLabelsDomain, kInterceptStump, kFinite},
  {"reg:logistic", kObjRegLogistic, kLinkSigmoid, kGradScalar, nullptr, true, false, kLabelsDomain, kInterceptStump, kIn01},
  {"binary:logistic", kObjLogistic, kLinkSigmoid, kGradScalar, nullptr, true, false, kLabelsDomain, kInterceptStump, kFinite},
  {"binary:logitraw", kObjLogitRaw, kLinkIdentity, kGradScalar, nullptr, true, false, kLabelsDomain, kInterceptStump, kIn01},
  {"reg:squaredlogerror", kObjSquaredLog, kLinkIdentity, kGradScalar, nullptr, true, true, kLabelsDomain, kInterceptStump, kAboveMinus1},
  {"reg:pseudohubererror", kObjPseudoHuber, kLinkIdentity, kGradScalar, &Params::huber_slope, true, true, kLabelsDomain, kInterceptStump, kFinite},
  {"count:poisson", kObjPoisson, kLinkExp, kGradScalar, &Params::max_delta_step, false, true, kLabelsDomain, kInterceptStump, kNonneg},
  {"reg:gamma", kObjGamma, kLinkExp, kGradScalar, nullptr, false, true, kLabelsDomain, kInterceptStump, kPositive},
  {"reg:tweedie", kObjTweedie, kLinkExp, kGradScalar, &Params::tweedie_variance_power, false, true, kLabelsDomain, kInterceptStump, kNonneg},
  {"survival:aft", kObjAft, kLinkExp, kGradAft, nullptr, false, true, kLabelsBounds, kInterceptFixed},
  {"rank:pairwise", kObjRankPairwise, kLinkIdentity, kGradRank, nullptr, false, true, kLabelsRank, kInterceptFixed},
  {"rank:ndcg", kObjRankNdcg, kLinkIdentity, kGradRank, nullptr, false, true, kLabelsRank, kInterceptFixed},
  {"rank:map", kObjRankMap, kLinkIdentity, kGradRank, nullptr, false, true, kLabelsRank, kInterceptFixed},
  {"reg:quantileerror", kObjQuantile, kLinkIdentity, kGradQuantile, nullptr, false, false, kLabelsDomain, kInterceptQuantile, kFinite},
  {"multi:softprob", kObjSoftprob, kLinkSoftmax, kGradSoftprob, nullptr, false, false, kLabelsDomain, kInterceptNone, kClassIndex},
  {"multi:softmax", kObjSoftprob, kLinkSoftmax, kGradSoftprob, nullptr, false, false, kLabelsDomain, kInterceptNone, kClassIndex},
};

const Objective& objective_row(const Params& p) { return kObjectives[p.objective_index]; }

constexpr int kMaxVectorTargets = 64;   // vector-leaf trees: the level histograms are T times a scalar tree's

// "0,1;2,3,4" -> {{0, 1}, {2, 3, 4}}; empty sets are dropped, the indices are checked against F in B2_BoosterCreate
std::vector<std::vector<int64_t>> parse_interaction_sets(const std::string& v) {
  std::vector<std::vector<int64_t>> sets;
  size_t pos = 0;
  while (pos <= v.size()) {
    size_t semi = v.find(';', pos);
    if (semi == std::string::npos) semi = v.size();
    std::vector<int64_t> set;
    size_t q = pos;
    while (q < semi) {
      size_t comma = v.find(',', q);
      if (comma == std::string::npos || comma > semi) comma = semi;
      const std::string tok = v.substr(q, comma - q);
      char* end = nullptr;
      const long long f = strtoll(tok.c_str(), &end, 10);
      if (tok.empty() || *end != '\0' || f < 0)
        fail("interaction_constraints: '%s' is not a feature index (expected sets like 0,1;2,3,4)", tok.c_str());
      set.push_back(f);
      q = comma + 1;
    }
    if (!set.empty()) sets.push_back(set);
    pos = semi + 1;
  }
  return sets;
}

// quantile_alpha as "a,b,c" (brackets allowed): every alpha finite with 0 < alpha < 1
std::vector<float> parse_quantile_alpha(std::string v) {
  for (char& c : v) if (c == '[' || c == ']' || c == '(' || c == ')') c = ' ';
  std::vector<float> out;
  size_t pos = 0;
  while (pos <= v.size()) {
    size_t comma = v.find(',', pos);
    if (comma == std::string::npos) comma = v.size();
    std::string tok = v.substr(pos, comma - pos);
    const size_t a = tok.find_first_not_of(" \t"), b = tok.find_last_not_of(" \t");
    tok = a == std::string::npos ? std::string() : tok.substr(a, b - a + 1);
    char* end = nullptr;
    const double x = strtod(tok.c_str(), &end);
    const float f = (float)x;
    if (tok.empty() || *end != '\0' || !(f > 0.0f && f < 1.0f))
      fail("quantile_alpha: '%s' is not a number in (0, 1)", tok.c_str());
    out.push_back(f);
    pos = comma + 1;
  }
  return out;
}

// T label columns: one output and one tree per round for each (xgboost's multi_strategy=one_output_per_tree)
void set_targets(Params* p, int T) {
  if (T < 1 || T > kMaxTargets) fail("num_target must be in [1, %d], got %d", kMaxTargets, T);
  if (T > 1) {
    if (!objective_row(*p).multi_target)
      fail("objective '%s' does not support a label with %d columns (multi-target objectives: reg:squarederror, "
           "reg:squaredlogerror, reg:pseudohubererror, reg:logistic, binary:logistic, binary:logitraw)",
           p->objective_name.c_str(), T);
    if (p->num_class_set)
      fail("num_class must not be set with a label of %d columns: a multi-target model has one output per column", T);
    p->num_class = T;
  }
  p->num_target = T;
  if (p->vector_leaf()) {   // DESIGN.md 2 item 19: the vector-leaf rules that need the label width
    if (T > kMaxVectorTargets)
      fail("multi_strategy='multi_output_tree' supports at most %d targets, the label has %d columns", kMaxVectorTargets, T);
    if (p->update_mode) fail("process_type='update' is not supported with multi_strategy='multi_output_tree'");
  }
}

// the "key=value" lines of a params text, in order; a line without '=' is skipped
std::vector<std::pair<std::string, std::string>> param_lines(const char* text) {
  std::vector<std::pair<std::string, std::string>> out;
  const std::string s(text ? text : "");
  size_t pos = 0;
  while (pos < s.size()) {
    size_t nl = s.find('\n', pos);
    if (nl == std::string::npos) nl = s.size();
    const std::string line = s.substr(pos, nl - pos);
    pos = nl + 1;
    const size_t eq = line.find('=');
    if (eq != std::string::npos) out.push_back({line.substr(0, eq), line.substr(eq + 1)});
  }
  return out;
}

// One key into p.  The DART keys go to dart_text (checked once booster=dart is known); max_bin to *max_bin_out.
// Returns false for a key the engine does not know.
bool apply_param(Params* p, const std::string& k, const std::string& v, std::map<std::string, std::string>* dart_text,
                 int* max_bin_out) {
  auto f = [&]() { return (float)atof(v.c_str()); };
  auto i = [&]() { return atoi(v.c_str()); };
  if (k == "objective") {
    p->objective_name = v;
    const Objective* row = std::find_if(std::begin(kObjectives), std::end(kObjectives),
                                        [&](const Objective& o) { return v == o.name; });
    if (row == std::end(kObjectives))
      fail("unsupported objective '%s' (supported: reg:squarederror, reg:logistic, binary:logistic, binary:logitraw, "
           "reg:squaredlogerror, reg:pseudohubererror, count:poisson, reg:gamma, reg:tweedie, survival:aft, "
           "rank:pairwise, rank:ndcg, rank:map, reg:quantileerror, multi:softprob, multi:softmax)", v.c_str());
    p->objective_index = (int)(row - kObjectives);
    p->objective = row->id;
  } else if (k == "num_class") { p->num_class = i(); p->num_class_set = true; }
  else if (k == "num_target") { p->num_target = i(); p->num_target_set = true; }
  else if (k == "quantile_alpha") p->quantile_alpha = parse_quantile_alpha(v);
  else if (k == "num_parallel_tree") p->num_parallel_tree = i();
  else if (k == "max_depth") p->max_depth = i();
  else if (k == "eta" || k == "learning_rate") p->eta = f();
  else if (k == "gamma" || k == "min_split_loss") p->gamma = f();
  else if (k == "min_child_weight") p->min_child_weight = f();
  else if (k == "lambda" || k == "reg_lambda") p->lambda = f();
  else if (k == "alpha" || k == "reg_alpha") p->alpha = f();
  else if (k == "base_score") { p->base_score = f(); p->base_score_set = true; }
  else if (k == "hist_qbits") p->qbits = i();
  else if (k == "hist_chunk_rows") p->hist_chunk_rows = i();
  else if (k == "profile") p->profile = i();
  else if (k == "num_feature") p->num_feature = i();
  else if (k == "device") p->device = i();
  else if (k == "subsample") p->subsample = f();
  else if (k == "colsample_bytree") p->colsample_bytree = f();
  else if (k == "colsample_bylevel") p->colsample_bylevel = f();
  else if (k == "colsample_bynode") p->colsample_bynode = f();
  else if (k == "seed" || k == "random_state") p->seed = i();
  else if (k == "scale_pos_weight") p->scale_pos_weight = f();
  else if (k == "max_delta_step") { p->max_delta_step = f(); p->max_delta_step_set = true; }
  else if (k == "huber_slope") p->huber_slope = f();
  else if (k == "tweedie_variance_power") p->tweedie_variance_power = f();
  else if (k == "aft_loss_distribution") {
    if (v == "normal") p->aft_dist = kAftNormal;
    else if (v == "logistic") p->aft_dist = kAftLogistic;
    else if (v == "extreme") p->aft_dist = kAftExtreme;
    else fail("aft_loss_distribution must be normal, logistic or extreme, got '%s'", v.c_str());
  }
  else if (k == "aft_loss_distribution_scale") p->aft_sigma = f();
  else if (k == "lambdarank_pair_method") {
    if (v != "topk") fail("lambdarank_pair_method='%s' is not supported (supported: topk; random pair sampling "
                          "(mean) is not implemented)", v.c_str());
  }
  else if (k == "lambdarank_num_pair_per_sample") {
    char* end = nullptr;
    const long long kv = strtoll(v.c_str(), &end, 10);
    if (v.empty() || *end != '\0' || kv < 1 || kv > INT32_MAX)
      fail("lambdarank_num_pair_per_sample must be an integer >= 1, got '%s'", v.c_str());
    p->rank_k = (int)kv;
  }
  else if (k == "lambdarank_unbiased" || k == "ndcg_exp_gain") {
    bool on;
    if (v == "1" || v == "true" || v == "True") on = true;
    else if (v == "0" || v == "false" || v == "False") on = false;
    else fail("%s must be a boolean, got '%s'", k.c_str(), v.c_str());
    if (k == "ndcg_exp_gain") p->ndcg_exp_gain = on;
    else if (on) fail("lambdarank_unbiased=true is not supported (position-bias estimation is not implemented)");
  }
  else if (k == "max_cat_to_onehot") p->max_cat_to_onehot = i();
  else if (k == "max_cat_threshold") p->max_cat_threshold = i();
  else if (k == "max_bin") { if (max_bin_out) *max_bin_out = i(); }
  else if (k == "interaction_constraints") p->interaction_sets = parse_interaction_sets(v);
  else if (k == "multi_strategy") {
    if (v == "one_output_per_tree") p->multi_strategy = 0;
    else if (v == "multi_output_tree") p->multi_strategy = 1;
    else fail("multi_strategy='%s' is not supported (supported: one_output_per_tree, multi_output_tree)", v.c_str());
  }
  else if (k == "booster") {
    if (v == "gbtree") p->dart = false;
    else if (v == "dart") p->dart = true;
    else fail("booster='%s' is not supported (supported: gbtree, dart)", v.c_str());
  }
  else if (k == "rate_drop" || k == "skip_drop" || k == "sample_type" || k == "normalize_type" || k == "one_drop")
    (*dart_text)[k] = v;   // checked by apply_dart_params, and only for booster=dart (gbtree ignores them, like xgboost)
  else if (k == "process_type") {
    if (v == "default") p->update_mode = false;
    else if (v == "update") p->update_mode = true;
    else fail("process_type='%s' is not supported (supported: 'default', 'update')", v.c_str());
  }
  else if (k == "updater") {
    if (v != "refresh" && v != "grow_quantile_histmaker" && v != "grow_gpu_hist")
      fail("updater='%s' is not supported (supported: grow_quantile_histmaker, grow_gpu_hist, and refresh with "
           "process_type='update')", v.c_str());
    p->updater = v;
  }
  else if (k == "refresh_leaf") {
    if (v == "1" || v == "true" || v == "True") p->refresh_leaf = true;
    else if (v == "0" || v == "false" || v == "False") p->refresh_leaf = false;
    else fail("refresh_leaf must be 0 or 1, got '%s'", v.c_str());
  }
  else return false;   // unknown keys (nthread, tree_method, verbosity, ...) are accepted and ignored, like xgboost
  return true;
}

void apply_dart_params(Params* p, const std::map<std::string, std::string>& dart_text) {
  if (p->dart) {
    for (const auto& kv : dart_text) {
      const std::string& k = kv.first; const std::string& v = kv.second;
      if (k == "sample_type") {
        if (v != "uniform" && v != "weighted") fail("sample_type must be uniform or weighted, got '%s'", v.c_str());
        p->dart_weighted = v == "weighted";
      } else if (k == "normalize_type") {
        if (v != "tree" && v != "forest") fail("normalize_type must be tree or forest, got '%s'", v.c_str());
        p->dart_forest = v == "forest";
      } else if (k == "one_drop") {
        if (v == "1" || v == "true" || v == "True") p->one_drop = true;
        else if (v == "0" || v == "false" || v == "False") p->one_drop = false;
        else fail("one_drop must be 0 or 1, got '%s'", v.c_str());
      } else {
        char* end = nullptr;
        const double x = strtod(v.c_str(), &end);
        if (v.empty() || *end != '\0' || !(x >= 0.0 && x <= 1.0)) fail("%s must be a number in [0, 1], got '%s'", k.c_str(), v.c_str());
        (k == "rate_drop" ? p->rate_drop : p->skip_drop) = x;
      }
    }
  }
}

// The range rules of the keys that may change between rounds (round_param_key): B2_BoosterCreate and
// B2_BoosterSetParam apply the same ones.  count:poisson's max_delta_step defaults to 0.7 until one is given.
void check_round_params(Params* p) {
  for (float v : {p->subsample, p->colsample_bytree, p->colsample_bylevel, p->colsample_bynode})
    if (!(v > 0.0f && v <= 1.0f)) fail("subsample / colsample_* must be in (0, 1], got %g", (double)v);
  if (p->max_cat_to_onehot < 1) fail("max_cat_to_onehot must be >= 1, got %d", p->max_cat_to_onehot);
  if (p->max_cat_threshold < 1) fail("max_cat_threshold must be >= 1, got %d", p->max_cat_threshold);
  if (p->objective == kObjPoisson) {
    if (!p->max_delta_step_set) p->max_delta_step = 0.7f;   // both the hessian's shift and the leaf-step clamp
    if (!(p->max_delta_step >= 0.0f)) fail("max_delta_step must be >= 0 for count:poisson, got %g", (double)p->max_delta_step);
  }
}

void parse_params(const char* text, Params* p, int* max_bin_out) {
  std::map<std::string, std::string> dart_text;
  for (const auto& kv : param_lines(text)) apply_param(p, kv.first, kv.second, &dart_text, max_bin_out);
  apply_dart_params(p, dart_text);
  const Objective& obj = objective_row(*p);
  if (obj.grad == kGradRank && p->num_class > 1)
    fail("%s has one output per row: num_class must be 1, got %d", p->objective_name.c_str(), p->num_class);
  if (obj.grad == kGradQuantile) {
    // rules of this engine (DESIGN.md 2): the outputs are the alphas, the leaf refresh needs the plain gbtree round
    if (p->num_class_set)
      fail("reg:quantileerror has one output per quantile_alpha: num_class must not be set (got %d)", p->num_class);
    if (p->dart) fail("reg:quantileerror is not supported with booster='dart'");
    if (p->num_parallel_tree > 1) fail("reg:quantileerror needs num_parallel_tree = 1 (got %d)", p->num_parallel_tree);
    p->num_class = (int)p->quantile_alpha.size();
  } else if (obj.grad != kGradSoftprob) p->num_class = 1;
  // vector-leaf trees (DESIGN.md 2 item 19): what they do not cover yet, refused for any number of targets
  if (p->multi_strategy == 1) {
    if (obj.grad == kGradSoftprob)
      fail("multi_strategy='multi_output_tree' is not supported with objective='%s': vector-leaf trees take the "
           "multi-target objectives (reg:squarederror, reg:squaredlogerror, reg:pseudohubererror, reg:logistic, "
           "binary:logistic, binary:logitraw)", p->objective_name.c_str());
    if (p->dart) fail("multi_strategy='multi_output_tree' is not supported with booster='dart'");
    if (p->num_parallel_tree > 1)
      fail("multi_strategy='multi_output_tree' needs num_parallel_tree = 1 (got %d)", p->num_parallel_tree);
  }
  if (obj.grad == kGradSoftprob && p->num_class < 2) fail("multi:softprob needs num_class >= 2");
  // update mode (DESIGN.md 2 item 20): only the refresh updater, and only where a refreshed leaf is a Newton step
  if (p->update_mode) {
    if (p->updater != "refresh")
      fail("process_type='update' needs updater='refresh', got updater='%s' (updater='prune' and 'refresh,prune' are "
           "not supported)", p->updater.c_str());
    if (p->dart) fail("process_type='update' is not supported with booster='dart'");
    if (obj.grad == kGradQuantile)
      fail("process_type='update' is not supported with objective='reg:quantileerror': its leaf values are residual "
           "quantiles, which the refresh updater does not recompute");
  } else if (p->updater == "refresh") {
    fail("updater='refresh' needs process_type='update': it refreshes the trees of an existing model (xgb_model)");
  }
  if (p->num_target_set) set_targets(p, p->num_target);
  // 16: a leaf index must fit the uint16_t row -> leaf map pos (2^16 leaves), DESIGN.md 9
  if (p->max_depth < 1 || p->max_depth > 16) fail("max_depth must be in [1, 16], got %d", p->max_depth);
  if (p->num_parallel_tree < 1 || p->num_parallel_tree > 4096) fail("num_parallel_tree must be in [1, 4096], got %d", p->num_parallel_tree);
  if (p->qbits < 8 || p->qbits > 24) fail("hist_qbits must be in [8, 24], got %d", p->qbits);
  check_round_params(p);
  if (p->objective == kObjPseudoHuber && !(p->huber_slope > 0.0f))
    fail("huber_slope must be > 0 for reg:pseudohubererror, got %g", (double)p->huber_slope);
  if (p->objective == kObjTweedie && !(p->tweedie_variance_power >= 1.0f && p->tweedie_variance_power < 2.0f))
    fail("tweedie_variance_power must be in [1, 2), got %g", (double)p->tweedie_variance_power);
  if (!(p->aft_sigma > 0.0f) || std::isinf(p->aft_sigma))
    fail("aft_loss_distribution_scale must be finite and > 0, got %g", (double)p->aft_sigma);
  // survival:aft fits no intercept (margin log 0.5), and the rank objectives' margin is the score itself (identity
  // transform): base_score defaults to 0.5 and is never estimated
  if (obj.intercept == kInterceptFixed && !p->base_score_set) { p->base_score = 0.5f; p->base_score_set = true; }
  if (p->base_score_set) {
    if (p->objective == kObjRegLogistic && !(p->base_score > 0.0f && p->base_score < 1.0f))
      fail("base_score must be in (0, 1) for reg:logistic, got %g", (double)p->base_score);
    if (obj.link == kLinkExp && !(p->base_score > 0.0f))
      fail("base_score must be > 0 for %s, got %g", p->objective_name.c_str(), (double)p->base_score);
  }
}

// The keys B2_BoosterSetParam applies between rounds (DESIGN.md 2 item 22): they enter a round's gradients, split scan,
// sampling and leaf values only, never the model's shape or the size of a device buffer
bool round_param_key(const std::string& k) {
  static const std::set<std::string> keys{
      "eta", "learning_rate", "gamma", "min_split_loss", "min_child_weight", "lambda", "reg_lambda", "alpha",
      "reg_alpha", "max_delta_step", "subsample", "colsample_bytree", "colsample_bylevel", "colsample_bynode",
      "max_cat_to_onehot", "max_cat_threshold"};
  return keys.count(k) != 0;
}

// every field a key outside round_param_key sets (not the *_set bookkeeping): equal when such a key kept its value
bool same_fixed_params(const Params& a, const Params& b) {
  return std::tie(a.objective_name, a.num_class, a.num_target, a.num_parallel_tree, a.max_depth, a.base_score, a.qbits,
                  a.hist_chunk_rows, a.profile, a.num_feature, a.device, a.scale_pos_weight, a.huber_slope,
                  a.tweedie_variance_power, a.aft_dist, a.aft_sigma, a.rank_k, a.ndcg_exp_gain, a.seed,
                  a.interaction_sets, a.dart, a.rate_drop, a.skip_drop, a.dart_weighted, a.dart_forest, a.one_drop,
                  a.quantile_alpha, a.multi_strategy, a.update_mode, a.refresh_leaf, a.updater) ==
         std::tie(b.objective_name, b.num_class, b.num_target, b.num_parallel_tree, b.max_depth, b.base_score, b.qbits,
                  b.hist_chunk_rows, b.profile, b.num_feature, b.device, b.scale_pos_weight, b.huber_slope,
                  b.tweedie_variance_power, b.aft_dist, b.aft_sigma, b.rank_k, b.ndcg_exp_gain, b.seed,
                  b.interaction_sets, b.dart, b.rate_drop, b.skip_drop, b.dart_weighted, b.dart_forest, b.one_drop,
                  b.quantile_alpha, b.multi_strategy, b.update_mode, b.refresh_leaf, b.updater);
}

// B2_BoosterSetParam's rules: `live` with the round keys of text applied, each checked by its B2_BoosterCreate rule.
// Any other key the engine knows must keep its value; unknown keys are ignored.  Fails before anything is applied.
Params changed_params(const Params& live, const char* text) {
  Params q = live;
  for (const auto& kv : param_lines(text)) {
    const std::string& k = kv.first;
    if (round_param_key(k)) { apply_param(&q, k, kv.second, nullptr, nullptr); continue; }
    Params r = live;
    std::map<std::string, std::string> dart_text;
    if (!apply_param(&r, k, kv.second, &dart_text, nullptr)) continue;
    apply_dart_params(&r, dart_text);
    if (!same_fixed_params(r, live))
      fail("parameter %s cannot change after training started: %s; pass it to train()", k.c_str(),
           k == "max_depth" ? "the level buffers and read-back blocks are sized by it"
           : k == "objective" || k == "num_class" || k == "num_target" || k == "quantile_alpha" ||
                   k == "multi_strategy" || k == "num_parallel_tree"
               ? "it sets the model's outputs and the trees of a round"
               : "it is fixed when the booster is created");
  }
  check_round_params(&q);
  return q;
}

// margin of base_score (the inverse of the prediction transform), evaluated on the host with libm's logf
float base_margin_value(const Params& p) {
  if (objective_row(p).link == kLinkSigmoid) return -logf(1.0f / p.base_score - 1.0f);
  if (objective_row(p).link == kLinkExp) return logf(p.base_score);
  return p.base_score;   // identity, and every class of a softmax
}

// -- host replicas of the gain / weight formulas (A.6, A.7); same IEEE sequence as the kernels
double h_thr_l1(double g, double a) { if (g > a) return g - a; if (g < -a) return g + a; return 0.0; }
float h_calc_weight(const Params& p, double G, double H) {
  if (H < (double)p.min_child_weight || H <= 0.0) return 0.0f;
  double t = p.alpha == 0.0f ? G : h_thr_l1(G, (double)p.alpha);
  double dw = -t / (H + (double)p.lambda);
  if (p.max_delta_step != 0.0f && fabs(dw) > (double)p.max_delta_step) dw = copysign((double)p.max_delta_step, dw);
  return (float)dw;
}

// Every eval_metric name.  A name is matched whole, except tweedie-nloglik[@rho] and the ranking metrics ndcg / map /
// pre[@k][-]; those come last, so that "mape" is not read as map@k.
constexpr Metric kMetrics[] = {
  {"rmse", kMetricRmse, kEvalElementwise, true},
  {"rmsle", kMetricRmsle, kEvalElementwise, true},
  {"mae", kMetricMae, kEvalElementwise, true},
  {"mape", kMetricMape, kEvalElementwise, true},
  {"mphe", kMetricMphe, kEvalElementwise, true},
  {"logloss", kMetricLogloss, kEvalElementwise, true},
  {"error", kMetricError, kEvalElementwise, true},
  {"poisson-nloglik", kMetricPoissonNloglik, kEvalElementwise, false},
  {"gamma-nloglik", kMetricGammaNloglik, kEvalElementwise, false},
  {"gamma-deviance", kMetricGammaDeviance, kEvalElementwise, false},
  {"mlogloss", kMetricMlogloss, kEvalClass, false},
  {"merror", kMetricMerror, kEvalClass, false},
  {"auc", kMetricAuc, kEvalAuc, false},
  {"aucpr", kMetricAucPr, kEvalAuc, false},
  {"aft-nloglik", kMetricAftNloglik, kEvalAft, false},
  {"interval-regression-accuracy", kMetricIntervalAccuracy, kEvalAft, false},
  {"quantile", kMetricQuantile, kEvalQuantile, false},
  {"tweedie-nloglik", kMetricTweedieNloglik, kEvalElementwise, false},
  {"ndcg", kMetricNdcg, kEvalRank, false},
  {"map", kMetricMap, kEvalRank, false},
  {"pre", kMetricPre, kEvalRank, false},
};

// the row of an eval_metric name; *param receives its parameter (tweedie-nloglik@rho, mphe's huber_slope, k of a ranking
// metric's @k, 0: the whole group), *minus a ranking metric's trailing '-' (groups without relevant rows score 0, not 1)
const Metric& metric_id(const char* name, const Params& p, float* param, int* minus) {
  const std::string s(name ? name : "");
  *param = 0.0f; *minus = 0;
  for (const Metric& r : kMetrics) {
    if (s.compare(0, strlen(r.name), r.name) != 0) continue;
    std::string rest = s.substr(strlen(r.name));
    if (r.id == kMetricTweedieNloglik) {
      *param = 1.5f;   // xgboost's default when the name carries no @rho
      if (rest.empty()) return r;
      char* end = nullptr;
      const double v = rest[0] == '@' ? strtod(rest.c_str() + 1, &end) : NAN;
      if (rest[0] != '@' || rest.size() < 2 || *end != '\0' || !(v >= 1.0 && v < 2.0))
        fail("eval metric '%s': the Tweedie power must be given as tweedie-nloglik@rho with rho in [1, 2)", s.c_str());
      *param = (float)v;
    } else if (r.family == kEvalRank) {
      if (!rest.empty() && rest.back() == '-') { *minus = 1; rest.pop_back(); }
      if (rest.empty()) return r;
      char* end = nullptr;
      const long long k = rest[0] == '@' && rest.size() > 1 ? strtoll(rest.c_str() + 1, &end, 10) : -1;
      if (rest[0] != '@' || rest.size() < 2 || *end != '\0' || k < 1 || k > (1 << 24))
        fail("eval metric '%s': the cut-off must be given as %s@k with an integer k >= 1", s.c_str(), r.name);
      *param = (float)k;
    } else if (!rest.empty()) {
      continue;
    } else if (r.id == kMetricMphe) {
      *param = p.huber_slope;
    }
    return r;
  }
  fail("unsupported eval metric '%s' (supported: rmse, mae, logloss, error, auc, aucpr, mlogloss, merror, rmsle, mape, mphe, "
       "poisson-nloglik, gamma-nloglik, gamma-deviance, tweedie-nloglik@rho, aft-nloglik, interval-regression-accuracy, "
       "quantile, ndcg[@k][-], map[@k][-], pre[@k][-])", s.c_str());
}

}  // namespace b2host
