/*
 * hist_oracle.c -- CPU ORACLE for the histogram-tree training path.
 *
 * THIS FILE IS TEST INFRASTRUCTURE.  It is the checker the CUDA path is compared
 * against (tests/, __graft_entry__.smoke(), bench.py's cpu_baseline / --impl
 * reference legs).  Nothing under xgboost_ray_b200/ may import, link or call it.
 *
 * PARITY UNPINNED: the arithmetic of this path lives in the third-party `xgboost`
 * wheel (dmlc/xgboost, unpinned: reference setup.py:18 "xgboost>=0.90"), which is
 * not vendored under /root/reference and not installable here.  The reference holds
 * no golden vectors for it (SURVEY.md 8c), only relational known-answer tests, which
 * tests/test_oracle_*.py port.  This file restates the PUBLISHED algorithm of
 * XGBoost 2.x CPU `tree_method="hist"` (SURVEY.md Appendix A), anchored on the
 * reference call sites:
 *   xgb.DMatrix / QuantileDMatrix construction ... xgboost_ray/main.py:386,418,437
 *   xgb.train(...)                              ... xgboost_ray/main.py:745-752
 *   model.predict(...)                          ... xgboost_ray/main.py:804
 *
 * Sections (upstream file the restatement follows, from Appendix A):
 *   A.2  cuts & bins      (src/common/quantile.{h,cc}: WQSummary::SetPrune, AddCutPoint)
 *   A.4  gradients        (src/objective/regression_loss.h, multiclass_obj.cu)
 *   A.5  histogram        (src/tree/hist/histogram.h) -- exact-integer (fixed point)
 *                          or float64 accumulation
 *   A.6  split enumeration(src/tree/hist/evaluate_splits.h, src/tree/param.h)
 *   A.7  tree bookkeeping (src/tree/updater_quantile_hist.cc, driver.h)
 *   A.8  row partition    (src/tree/common_row_partitioner.h)
 *   A.9  prediction       (src/predictor/cpu_predictor.cc)
 *   A.10 metrics          (src/metric/elementwise_metric.cu, multiclass_metric.cu)
 *   A.2/A.6/A.8 categorical features (src/common/categorical.h, evaluate_splits.h
 *                          EnumerateOneHot / EnumeratePart): bin = category code, one-hot
 *                          splits below max_cat_to_onehot categories, otherwise categories
 *                          sorted by leaf weight and scanned from both ends; the split stores
 *                          the set of categories that go RIGHT
 *
 * Deliberate, documented deviations (DESIGN.md "Oracle decisions"):
 *   - sketch ranks are exact (int64) instead of fp32 GK summaries: the exact summary
 *     is what XGBoost's sketch approximates and equals it for small inputs;
 *   - a feature that has missing values is capped at 255 real bins (bin 255 is the
 *     missing sentinel of the uint8 matrix);
 *   - exp() in the objectives is a fixed IEEE-only sequence (or_expf) so that the
 *     CUDA path can reproduce gradients bit-for-bit;
 *   - histogram sums are exact integers of gradients quantised to `qbits` bits
 *     (qbits==0 selects float64 accumulation, XGBoost's CPU behaviour).
 *
 * Build: see oracle/Makefile (gcc -O2 -ffp-contract=off -fopenmp).
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define OR_MISSING_BIN 255
#define OR_RT_EPS 1e-6f
#define OR_LEAF_BITS 40

/* A row's 40-bit fixed-point value q has |q| <= 2^40, so one int64 sum wraps past 2^23 rows.  Leaf and intercept
 * sums are kept as two int64 limbs instead, value = hi * 2^24 + lo with hi += q >> 24, lo += q & (2^24 - 1): for
 * fewer than 2^31 rows |hi| < 2^48 and 0 <= lo < 2^55, so neither wraps. */
#define OR_LIMB_SHIFT 24
#define OR_LIMB_MASK ((INT64_C(1) << OR_LIMB_SHIFT) - 1)
/* the correctly rounded value of hi * 2^24 + lo: after the carry both terms are exact doubles, one rounding in the
 * add -- the same double as (double)sum whenever the sum fits in an int64 */
static double or_limbs_to_double(int64_t hi, int64_t lo) {
  hi += lo >> OR_LIMB_SHIFT;
  lo &= OR_LIMB_MASK;
  return (double)hi * (double)(INT64_C(1) << OR_LIMB_SHIFT) + (double)lo;
}

/* 2^s as two binary32 factors of at most 2^127 each (b = 1 for s <= 127): a quantisation scale 2^(bits - e) passes
 * 2^127 when the maximum is tiny, and v * a * b is then still exactly v * 2^s with no infinite intermediate */
static void or_pow2_split(int s, float *a, float *b) {
  const int sa = s < 127 ? s : 127;
  *a = ldexpf(1.0f, sa);
  *b = ldexpf(1.0f, s - sa);
}

enum { OR_OBJ_SQUAREDERROR = 0, OR_OBJ_LOGISTIC = 1, OR_OBJ_SOFTPROB = 2 };

typedef struct {
  int32_t objective;
  int32_t num_class;     /* 1 unless softprob */
  int32_t max_depth;
  int32_t max_bin;
  float eta;
  float gamma;
  float min_child_weight;
  float lambda;
  float alpha;
  float base_score;      /* probability space for logistic */
  int32_t qbits;         /* 0 => float64 histogram */
  int32_t nthread;       /* 0 => omp default */
  int32_t max_cat_to_onehot;  /* categorical: one-hot splits when n_categories < this (xgboost default 4) */
  int32_t max_cat_threshold;  /* categorical: at most this many categories scanned per direction (default 64) */
  float scale_pos_weight;     /* binary:logistic: weight multiplier of the positive rows (A.4), default 1 */
  float max_delta_step;       /* 0 = off; otherwise |leaf weight| is clipped and the gain uses the clipped weight (A.7) */
  float subsample;            /* row sampling per tree (1 = off) */
  float colsample_bytree, colsample_bylevel, colsample_bynode;   /* nested column sampling (1 = off) */
  int32_t seed;
  int32_t rank;               /* worker rank: part of the row-sampling hash (each worker samples its own rows) */
} OrParams;

typedef struct {
  int32_t n_features;
  int32_t max_bin;
  int32_t *cut_ptrs;    /* [F+1] */
  float *cut_vals;      /* [cut_ptrs[F]] */
  float *min_vals;      /* [F] */
  uint8_t *has_missing; /* [F] */
  uint8_t *is_cat;      /* [F] 1 = categorical feature: cuts are the codes 0..max, bin = code */
} OrCuts;

typedef struct {
  int32_t n_nodes, cap;
  int32_t *left, *right, *parent;
  int32_t *split_feature; /* -1 for leaf */
  int32_t *split_bin;
  float *split_cond;
  uint8_t *default_left;
  float *value;           /* leaf value (eta applied) for leaves, base_weight for internal */
  float *base_weight;
  float *loss_chg;
  double *sum_hess;
  double *sum_grad;
  uint8_t *is_cat_split;  /* 1 = categorical split: categories (= bins) whose bit is set go right */
  uint32_t *cat_bits;     /* [cap][8] bit b of word b>>5 (LSB first) = category b */
} OrTree;

typedef struct {
  OrParams p;
  int32_t n_features;
  int32_t n_trees, cap_trees;
  OrTree **trees;
  uint32_t *fwq;          /* feature_weights in Q16 (NULL = all 1.0) */
} OrModel;

/* ------------------------------------------------------------------ util */
static int is_missing(float x, float missing) {
  return isnan(x) || (!isnan(missing) && x == missing);
}

/* Deterministic expf: only IEEE-754 binary32 add/mul (no fma contraction; the file is
 * compiled with -ffp-contract=off) so CUDA can replay it bit-for-bit with __fmul_rn /
 * __fadd_rn.  |rel err| <~ 2 ulp on [-88, 88]. */
float or_expf(float x) {
  if (x > 88.7f) x = 88.7f;
  if (x < -103.0f) return 0.0f;
  const float log2e = 1.44269504088896341f;
  const float ln2_hi = 0.693359375f;          /* 0x3f318000 */
  const float ln2_lo = -2.12194440e-4f;
  float t = x * log2e;
  float n = rintf(t);
  float r = x - n * ln2_hi;
  r = r - n * ln2_lo;
  /* minimax-ish polynomial for exp(r), r in [-ln2/2, ln2/2] */
  float p = 1.9875691500e-4f;
  p = p * r + 1.3981999507e-3f;
  p = p * r + 8.3334519073e-3f;
  p = p * r + 4.1665795894e-2f;
  p = p * r + 1.6666665459e-1f;
  p = p * r + 5.0000001201e-1f;
  float r2 = r * r;
  float e = p * r2 + r;
  e = e + 1.0f;
  /* scale by 2^n in two steps to stay in range */
  int ni = (int)n;
  int n1 = ni / 2, n2 = ni - n1;
  union { uint32_t u; float f; } s1, s2;
  s1.u = (uint32_t)(n1 + 127) << 23;
  s2.u = (uint32_t)(n2 + 127) << 23;
  e = e * s1.f;
  e = e * s2.f;
  return e;
}

static float or_sigmoid(float x) {
  /* regression_loss.h Sigmoid: 1/(1+exp(min(-x,88.7))+1e-16) */
  float nx = -x;
  if (nx > 88.7f) nx = 88.7f;
  float denom = or_expf(nx) + 1.0f;
  denom = denom + 1e-16f;
  return 1.0f / denom;
}

/* ------------------------------------------------------------------ A.2 cuts */
/* LSD radix sort of floats via order-preserving keys */
static uint32_t f2key(float f) {
  union { float f; uint32_t u; } v; v.f = f;
  return (v.u & 0x80000000u) ? ~v.u : (v.u | 0x80000000u);
}
static float key2f(uint32_t k) {
  union { float f; uint32_t u; } v;
  v.u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return v.f;
}
static void radix_sort_keys(uint32_t *a, uint32_t *tmp, int64_t n) {
  const int shifts[3] = {0, 11, 22};
  const int bits[3] = {11, 11, 10};
  for (int pass = 0; pass < 3; ++pass) {
    int nb = 1 << bits[pass];
    int64_t *cnt = (int64_t *)calloc((size_t)nb + 1, sizeof(int64_t));
    uint32_t mask = (uint32_t)nb - 1;
    for (int64_t i = 0; i < n; ++i) cnt[((a[i] >> shifts[pass]) & mask) + 1]++;
    for (int b = 0; b < nb; ++b) cnt[b + 1] += cnt[b];
    for (int64_t i = 0; i < n; ++i) tmp[cnt[(a[i] >> shifts[pass]) & mask]++] = a[i];
    memcpy(a, tmp, (size_t)n * sizeof(uint32_t));
    free(cnt);
  }
}

/* (key, integer weight) pairs sorted by key: LSD radix over the key half of key<<32 | weight */
static void radix_sort_pairs(uint64_t *a, uint64_t *tmp, int64_t n) {
  for (int pass = 0; pass < 4; ++pass) {
    const int sh = 32 + 8 * pass;
    int64_t cnt[257]; memset(cnt, 0, sizeof(cnt));
    for (int64_t i = 0; i < n; ++i) cnt[((a[i] >> sh) & 255u) + 1]++;
    for (int b = 0; b < 256; ++b) cnt[b + 1] += cnt[b];
    for (int64_t i = 0; i < n; ++i) tmp[cnt[(a[i] >> sh) & 255u]++] = a[i];
    memcpy(a, tmp, (size_t)n * sizeof(uint64_t));
  }
}

/* One feature: exact summary (distinct values, int64 rmin/rmax) -> SetPrune -> cuts.
 * sorted_wq (NULL = every row counts 1): integer sample weights aligned with sorted_keys; ranks are then sums
 * of weights (weighted quantile sketch).  Returns number of cuts written to out_cuts (<= 256). */
static int make_cuts_feature(const uint32_t *sorted_keys, const int32_t *sorted_wq, int64_t cnt, int max_num_bins_cap,
                             float *out_cuts, float *out_min) {
  /* distinct summary */
  int64_t m = 0;
  for (int64_t i = 0; i < cnt; ++i)
    if (i == 0 || sorted_keys[i] != sorted_keys[i - 1]) ++m;
  if (m == 0) {
    float mval = 0.0f;
    *out_min = mval - fabsf(mval) - 1e-5f;
    float cpt = *out_min;
    out_cuts[0] = cpt + (fabsf(cpt) + 1e-5f);
    return 1;
  }
  float *val = (float *)malloc((size_t)m * sizeof(float));
  int64_t *rmin = (int64_t *)malloc((size_t)m * sizeof(int64_t));
  int64_t *rmax = (int64_t *)malloc((size_t)m * sizeof(int64_t));
  int64_t u = -1, pre = 0;
  for (int64_t i = 0; i < cnt; ++i) {
    const int64_t wi = sorted_wq ? (int64_t)sorted_wq[i] : 1;
    if (i == 0 || sorted_keys[i] != sorted_keys[i - 1]) {
      ++u; val[u] = key2f(sorted_keys[i]); rmin[u] = pre; rmax[u] = pre + wi;
    } else rmax[u] = pre + wi;
    pre += wi;
  }
  int64_t max_num_bins = m < max_num_bins_cap ? m : max_num_bins_cap;
  int64_t maxsize = max_num_bins + 1;
  /* WQSummary::SetPrune(src, maxsize) on the exact summary; wmin = rmax-rmin */
  float *sel = (float *)malloc((size_t)(maxsize + 1) * sizeof(float));
  int64_t size = 0;
  if (m <= maxsize) {
    for (int64_t i = 0; i < m; ++i) sel[size++] = val[i];
  } else {
    const double begin = (double)rmax[0];
    const double range = (double)rmin[m - 1] - (double)rmax[0];
    const int64_t n = maxsize - 1;
    sel[size++] = val[0];
    int64_t i = 1, lastidx = 0;
    for (int64_t k = 1; k < n; ++k) {
      double dx2 = 2.0 * (((double)k * range) / (double)n + begin);
      while (i < m - 1 && dx2 >= (double)(rmax[i + 1] + rmin[i + 1])) ++i;
      if (i == m - 1) break;
      /* RMinNext(i) = rmin+wmin = rmax[i]; RMaxPrev(i+1) = rmax-wmin = rmin[i+1] */
      if (dx2 < (double)(rmax[i] + rmin[i + 1])) {
        if (i != lastidx) { sel[size++] = val[i]; lastidx = i; }
      } else {
        if (i + 1 != lastidx) { sel[size++] = val[i + 1]; lastidx = i + 1; }
      }
    }
    if (lastidx != m - 1) sel[size++] = val[m - 1];
  }
  /* HistogramCuts: min_val, AddCutPoint(a, max_num_bins), last */
  float mval = sel[0];
  *out_min = mval - fabsf(mval) - 1e-5f;
  int64_t required = size < max_num_bins ? size : max_num_bins;
  int nc = 0;
  for (int64_t i = 1; i < required; ++i) {
    float cpt = sel[i];
    if (i == 1 || cpt > out_cuts[nc - 1]) out_cuts[nc++] = cpt;
  }
  float cpt = sel[size - 1];
  out_cuts[nc++] = cpt + (fabsf(cpt) + 1e-5f);
  free(sel); free(val); free(rmin); free(rmax);
  return nc;
}

void or_cuts_free(OrCuts *c);

/* is_cat (may be NULL): categorical features get the cuts [0, 1, ..., max code] (HistogramCuts::AddCategories,
 * src/common/quantile.cc); a code must be an integer in [0, 255] ([0, 254] if the feature has missing values,
 * bin 255 being the sentinel).  Returns NULL on an invalid category value. */
OrCuts *or_cuts_create_w(const float *X, int64_t n, int32_t F, float missing, int32_t max_bin, const uint8_t *is_cat,
                         const float *weight);
OrCuts *or_cuts_create_cat(const float *X, int64_t n, int32_t F, float missing, int32_t max_bin, const uint8_t *is_cat) {
  return or_cuts_create_w(X, n, F, missing, max_bin, is_cat, NULL);
}
/* weight (may be NULL): sample weights -> weighted quantile sketch (SketchContainer pushes info.weights_,
 * src/common/quantile.cc).  Weights are quantised to integers wq = rint(w * 2^(30-e)), 2^e > max w, so that the
 * weighted ranks are exact (order independent); negative / non-finite weights are rejected (NULL). */
OrCuts *or_cuts_create_w(const float *X, int64_t n, int32_t F, float missing, int32_t max_bin, const uint8_t *is_cat,
                         const float *weight) {
  if (max_bin < 2 || max_bin > 256) return NULL;
  int32_t *wq = NULL;
  if (weight) {
    float vmax = 0.0f;
    for (int64_t i = 0; i < n; ++i) {
      if (!(weight[i] >= 0.0f) || isinf(weight[i])) return NULL;
      if (weight[i] > vmax) vmax = weight[i];
    }
    int e = 0;
    if (vmax > 0.0f) frexpf(vmax, &e);
    float sa, sb;
    or_pow2_split(30 - e, &sa, &sb);
    wq = (int32_t *)malloc((size_t)(n > 0 ? n : 1) * sizeof(int32_t));
    for (int64_t i = 0; i < n; ++i) wq[i] = (int32_t)lrintf(weight[i] * sa * sb);
  }
  OrCuts *c = (OrCuts *)calloc(1, sizeof(OrCuts));
  c->n_features = F; c->max_bin = max_bin;
  c->cut_ptrs = (int32_t *)calloc((size_t)F + 1, sizeof(int32_t));
  c->min_vals = (float *)calloc((size_t)F, sizeof(float));
  c->has_missing = (uint8_t *)calloc((size_t)F, 1);
  c->is_cat = (uint8_t *)calloc((size_t)F, 1);
  if (is_cat) memcpy(c->is_cat, is_cat, (size_t)F);
  float *tmpc = (float *)malloc((size_t)F * 256 * sizeof(float));
  int32_t *ncut = (int32_t *)calloc((size_t)F, sizeof(int32_t));
  int invalid = 0;
#pragma omp parallel for schedule(dynamic, 1)
  for (int32_t f = 0; f < F; ++f) {
    if (c->is_cat[f]) {
      int miss = 0; int32_t mx = -1; int bad = 0;
      for (int64_t i = 0; i < n; ++i) {
        float x = X[i * F + f];
        if (is_missing(x, missing)) { miss = 1; continue; }
        if (!(x >= 0.0f) || x > 255.0f || x != (float)(int32_t)x) { bad = 1; continue; }
        if ((int32_t)x > mx) mx = (int32_t)x;
      }
      if (miss && mx > 254) bad = 1;
      if (bad) {
#pragma omp atomic write
        invalid = 1;
      }
      c->has_missing[f] = (uint8_t)miss;
      c->min_vals[f] = -1e-5f;
      ncut[f] = mx < 0 ? 1 : mx + 1;
      for (int32_t k = 0; k < ncut[f]; ++k) tmpc[(size_t)f * 256 + k] = (float)k;
      continue;
    }
    uint32_t *keys = (uint32_t *)malloc((size_t)(n > 0 ? n : 1) * sizeof(uint32_t));
    uint32_t *tmp = (uint32_t *)malloc((size_t)(n > 0 ? n : 1) * sizeof(uint32_t));
    int32_t *swq = NULL;
    int64_t cnt = 0; int miss = 0;
    if (wq) {
      uint64_t *pairs = (uint64_t *)malloc((size_t)(n > 0 ? n : 1) * sizeof(uint64_t));
      uint64_t *ptmp = (uint64_t *)malloc((size_t)(n > 0 ? n : 1) * sizeof(uint64_t));
      for (int64_t i = 0; i < n; ++i) {
        float x = X[i * F + f];
        if (is_missing(x, missing)) { miss = 1; continue; }
        if (x == 0.0f) x = 0.0f;
        pairs[cnt++] = ((uint64_t)f2key(x) << 32) | (uint32_t)wq[i];
      }
      radix_sort_pairs(pairs, ptmp, cnt);
      swq = (int32_t *)malloc((size_t)(cnt > 0 ? cnt : 1) * sizeof(int32_t));
      for (int64_t i = 0; i < cnt; ++i) { keys[i] = (uint32_t)(pairs[i] >> 32); swq[i] = (int32_t)(uint32_t)pairs[i]; }
      free(pairs); free(ptmp);
    } else {
      for (int64_t i = 0; i < n; ++i) {
        float x = X[i * F + f];
        if (is_missing(x, missing)) { miss = 1; continue; }
        if (x == 0.0f) x = 0.0f; /* -0 -> +0 */
        keys[cnt++] = f2key(x);
      }
      radix_sort_keys(keys, tmp, cnt);
    }
    c->has_missing[f] = (uint8_t)miss;
    int cap = max_bin;
    if (miss && cap > 255) cap = 255;
    ncut[f] = make_cuts_feature(keys, swq, cnt, cap, tmpc + (size_t)f * 256, &c->min_vals[f]);
    free(keys); free(tmp); free(swq);
  }
  for (int32_t f = 0; f < F; ++f) c->cut_ptrs[f + 1] = c->cut_ptrs[f] + ncut[f];
  c->cut_vals = (float *)malloc((size_t)(c->cut_ptrs[F] > 0 ? c->cut_ptrs[F] : 1) * sizeof(float));
  for (int32_t f = 0; f < F; ++f)
    memcpy(c->cut_vals + c->cut_ptrs[f], tmpc + (size_t)f * 256, (size_t)ncut[f] * sizeof(float));
  free(tmpc); free(ncut); free(wq);
  if (invalid) { or_cuts_free(c); return NULL; }
  return c;
}
OrCuts *or_cuts_create(const float *X, int64_t n, int32_t F, float missing, int32_t max_bin) {
  return or_cuts_create_cat(X, n, F, missing, max_bin, NULL);
}
void or_cuts_set_cat(OrCuts *c, const uint8_t *is_cat) { memcpy(c->is_cat, is_cat, (size_t)c->n_features); }
void or_cuts_get_cat(const OrCuts *c, uint8_t *is_cat) { memcpy(is_cat, c->is_cat, (size_t)c->n_features); }

/* build cuts from caller-supplied arrays (e.g. downloaded from the device path) */
OrCuts *or_cuts_from_arrays(int32_t F, int32_t max_bin, const int32_t *ptrs, const float *vals,
                            const float *mins, const uint8_t *has_missing) {
  OrCuts *c = (OrCuts *)calloc(1, sizeof(OrCuts));
  c->n_features = F; c->max_bin = max_bin;
  c->cut_ptrs = (int32_t *)malloc(((size_t)F + 1) * sizeof(int32_t));
  memcpy(c->cut_ptrs, ptrs, ((size_t)F + 1) * sizeof(int32_t));
  c->cut_vals = (float *)malloc((size_t)ptrs[F] * sizeof(float));
  memcpy(c->cut_vals, vals, (size_t)ptrs[F] * sizeof(float));
  c->min_vals = (float *)malloc((size_t)F * sizeof(float));
  memcpy(c->min_vals, mins, (size_t)F * sizeof(float));
  c->has_missing = (uint8_t *)calloc((size_t)F, 1);
  if (has_missing) memcpy(c->has_missing, has_missing, (size_t)F);
  c->is_cat = (uint8_t *)calloc((size_t)F, 1);
  return c;
}

void or_cuts_free(OrCuts *c) {
  if (!c) return;
  free(c->cut_ptrs); free(c->cut_vals); free(c->min_vals); free(c->has_missing); free(c->is_cat); free(c);
}
int32_t or_cuts_total(const OrCuts *c) { return c->cut_ptrs[c->n_features]; }
void or_cuts_get(const OrCuts *c, int32_t *ptrs, float *vals, float *mins, uint8_t *has_missing) {
  memcpy(ptrs, c->cut_ptrs, ((size_t)c->n_features + 1) * sizeof(int32_t));
  memcpy(vals, c->cut_vals, (size_t)c->cut_ptrs[c->n_features] * sizeof(float));
  memcpy(mins, c->min_vals, (size_t)c->n_features * sizeof(float));
  memcpy(has_missing, c->has_missing, (size_t)c->n_features);
}

/* bin = upper_bound(cuts_f, x) clamped to the last bin; missing -> 255 (A.2) */
void or_bin_matrix(const OrCuts *c, const float *X, int64_t n, float missing, uint8_t *bins) {
  int32_t F = c->n_features;
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < n; ++i) {
    for (int32_t f = 0; f < F; ++f) {
      float x = X[i * F + f];
      if (is_missing(x, missing)) { bins[i * F + f] = OR_MISSING_BIN; continue; }
      const float *cv = c->cut_vals + c->cut_ptrs[f];
      int32_t nf = c->cut_ptrs[f + 1] - c->cut_ptrs[f];
      if (c->is_cat[f]) {  /* bin = category code; codes the cuts have not seen clamp like numeric values */
        int32_t b = x >= 0.0f ? (x > 255.0f ? 255 : (int32_t)x) : 0;
        bins[i * F + f] = (uint8_t)(b >= nf ? nf - 1 : b);
        continue;
      }
      int32_t lo = 0, hi = nf;
      while (lo < hi) { int32_t mid = (lo + hi) >> 1; if (cv[mid] > x) hi = mid; else lo = mid + 1; }
      if (lo >= nf) lo = nf - 1;
      bins[i * F + f] = (uint8_t)lo;
    }
  }
}

/* ------------------------------------------------------------------ A.4 gradients */
/* margin [n*K] row-major, out g,h [n*K] */
void or_gradients_spw(int32_t objective, int32_t K, const float *margin, const float *label,
                      const float *weight, int64_t n, float scale_pos_weight, float *g, float *h);
void or_gradients(int32_t objective, int32_t K, const float *margin, const float *label,
                  const float *weight, int64_t n, float *g, float *h) {
  or_gradients_spw(objective, K, margin, label, weight, n, 1.0f, g, h);
}
/* scale_pos_weight (regression_obj.cu, RegLossObj::GetGradient): w *= scale_pos_weight for rows with label 1 */
void or_gradients_spw(int32_t objective, int32_t K, const float *margin, const float *label,
                      const float *weight, int64_t n, float scale_pos_weight, float *g, float *h) {
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < n; ++i) {
    float w = weight ? weight[i] : 1.0f;
    if (objective == OR_OBJ_LOGISTIC && label[i] == 1.0f) w = w * scale_pos_weight;
    if (objective == OR_OBJ_SQUAREDERROR) {
      g[i] = (margin[i] - label[i]) * w;
      h[i] = 1.0f * w;
    } else if (objective == OR_OBJ_LOGISTIC) {
      float p = or_sigmoid(margin[i]);
      float hh = p * (1.0f - p);
      if (hh < 1e-16f) hh = 1e-16f;
      g[i] = (p - label[i]) * w;
      h[i] = hh * w;
    } else {
      const float *m = margin + i * K;
      float mx = m[0];
      for (int k = 1; k < K; ++k) if (m[k] > mx) mx = m[k];
      float s = 0.0f;
      for (int k = 0; k < K; ++k) { float e = or_expf(m[k] - mx); s = s + e; }
      int y = (int)label[i];
      for (int k = 0; k < K; ++k) {
        float p = or_expf(m[k] - mx) / s;
        float hh = 2.0f * p * (1.0f - p);
        if (hh < 1e-16f) hh = 1e-16f;
        g[i * K + k] = (k == y ? p - 1.0f : p) * w;
        h[i * K + k] = hh * w;
      }
    }
  }
}

/* fixed-point quantisation: scale = 2^(qbits - e) with max|v| < 2^e  (exact products) */
int32_t or_quant_exponent(float vmax) {
  if (!(vmax > 0.0f)) return 0;
  int e; frexpf(vmax, &e); /* vmax = m*2^e, m in [0.5,1), subnormals included */
  return e;
}
void or_quantize(const float *v, int64_t n, int64_t stride, int32_t qbits, int32_t *q, int32_t *out_exp) {
  float vmax = 0.0f;
  for (int64_t i = 0; i < n; ++i) { float a = fabsf(v[i * stride]); if (a > vmax) vmax = a; }
  int32_t e = or_quant_exponent(vmax);
  float sa, sb;
  or_pow2_split(qbits - e, &sa, &sb);
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < n; ++i) q[i] = (int32_t)rintf(v[i * stride] * sa * sb);
  *out_exp = e;
}

/* persistent per-thread scratch for row-parallel histograms (a fresh calloc per node is a page-fault
 * storm with many threads) */
static void *g_pool = NULL;
static size_t g_pool_bytes = 0;
static void *pool_get(size_t bytes) {
  if (bytes > g_pool_bytes) { free(g_pool); g_pool = malloc(bytes); g_pool_bytes = g_pool ? bytes : 0; }
  return g_pool;
}
/* persistent scratch slots (per-tree / per-level buffers): large malloc/free pairs are mmap/munmap calls and
 * fresh pages fault on first touch -- with 100+ threads that serialises on the kernel's mmap lock */
#define OR_N_SLOTS 16
static void *g_slot[OR_N_SLOTS];
static size_t g_slot_bytes[OR_N_SLOTS];
static void *slot_get(int slot, size_t bytes) {
  if (bytes > g_slot_bytes[slot]) {
    free(g_slot[slot]);
    g_slot[slot] = malloc(bytes + (bytes >> 2));
    g_slot_bytes[slot] = g_slot[slot] ? bytes + (bytes >> 2) : 0;
  }
  return g_slot[slot];
}
enum { SLOT_RIDX = 0, SLOT_RTMP, SLOT_QG, SLOT_QH, SLOT_G, SLOT_H, SLOT_HIST0, SLOT_HIST1, SLOT_IHIST0, SLOT_IHIST1 };
#define OR_ROWS_PER_THREAD 8192
static int hist_threads(int64_t nrows) {
#ifdef _OPENMP
  if (omp_in_parallel()) return 1;
  int64_t nt = nrows / OR_ROWS_PER_THREAD;
  int mx = omp_get_max_threads();
  if (nt > mx) nt = mx;
  return nt < 1 ? 1 : (int)nt;
#else
  (void)nrows; return 1;
#endif
}

/* ------------------------------------------------------------------ A.5 histogram */
/* hist layout [F][256][2] int64 (g,h); rows given by ridx (or NULL = 0..n-1) */
static void hist_int_serial(const uint8_t *bins, int32_t F, const int32_t *qg, const int32_t *qh, const int32_t *ridx,
                            int64_t k0, int64_t k1, int64_t *hist) {
  for (int64_t k = k0; k < k1; ++k) {
    int64_t r = ridx ? ridx[k] : k;
    const uint8_t *b = bins + r * F;
    int64_t g = qg[r], h = qh[r];
    for (int32_t f = 0; f < F; ++f) {
      int64_t *e = hist + ((size_t)f * 256 + b[f]) * 2;
      e[0] += g; e[1] += h;
    }
  }
}
void or_hist_int(const uint8_t *bins, int32_t F, const int32_t *qg, const int32_t *qh,
                 const int32_t *ridx, int64_t nrows, int64_t *hist) {
  size_t hsz = (size_t)F * 256 * 2;
  memset(hist, 0, hsz * sizeof(int64_t));
  int nt = hist_threads(nrows);
  if (nt == 1) { hist_int_serial(bins, F, qg, qh, ridx, 0, nrows, hist); return; }
  int64_t *priv = (int64_t *)pool_get(hsz * (size_t)nt * sizeof(int64_t));
#pragma omp parallel num_threads(nt)
  {
#ifdef _OPENMP
    int t = omp_get_thread_num();
#else
    int t = 0;
#endif
    int64_t *ph = priv + hsz * (size_t)t;
    memset(ph, 0, hsz * sizeof(int64_t));
    hist_int_serial(bins, F, qg, qh, ridx, nrows * t / nt, nrows * (t + 1) / nt, ph);
#pragma omp barrier
#pragma omp for schedule(static)
    for (int64_t jj = 0; jj < (int64_t)hsz; ++jj) {
      int64_t sacc = 0;
      for (int t2 = 0; t2 < nt; ++t2) sacc += priv[hsz * (size_t)t2 + (size_t)jj];
      hist[jj] = sacc;
    }
  }
}

/* Cache blocking: a node's histogram is F x 256 x 16 bytes (410 KB for 100 features), far beyond L1.  Rows are taken
 * in blocks of OR_ROW_BLOCK (their bin bytes stay in L2) and, inside a block, features in blocks of OR_FEAT_BLOCK whose
 * 32 KB of cells stay in L1 while the row block streams over them.  Every cell still receives its rows in row order, so
 * the float64 sums are bit-identical to the unblocked loop. */
#define OR_ROW_BLOCK 2048
#define OR_FEAT_BLOCK 8
static void hist_f64_serial(const uint8_t *bins, int32_t F, const float *g, const float *h, int64_t gstride,
                            const int32_t *ridx, int64_t k0, int64_t k1, double *hist) {
  for (int64_t kb = k0; kb < k1; kb += OR_ROW_BLOCK) {
    const int64_t ke = kb + OR_ROW_BLOCK < k1 ? kb + OR_ROW_BLOCK : k1;
    for (int32_t f0 = 0; f0 < F; f0 += OR_FEAT_BLOCK) {
      const int32_t f1 = f0 + OR_FEAT_BLOCK < F ? f0 + OR_FEAT_BLOCK : F;
      for (int64_t k = kb; k < ke; ++k) {
        int64_t r = ridx ? ridx[k] : k;
        const uint8_t *b = bins + r * F;
        double gg = g[r * gstride], hh = h[r * gstride];
        for (int32_t f = f0; f < f1; ++f) {
          double *e = hist + ((size_t)f * 256 + b[f]) * 2;
          e[0] += gg; e[1] += hh;
        }
      }
    }
  }
}
/* float64 accumulation (XGBoost CPU hist arithmetic).  Row-parallel with per-thread private
 * histograms when called outside a parallel region on a large node, serial otherwise. */
static void hist_f64(const uint8_t *bins, int32_t F, const float *g, const float *h, int64_t gstride,
                     const int32_t *ridx, int64_t nrows, double *hist) {
  size_t hsz = (size_t)F * 512;
  memset(hist, 0, hsz * sizeof(double));
  int nt = hist_threads(nrows);
  if (nt == 1) { hist_f64_serial(bins, F, g, h, gstride, ridx, 0, nrows, hist); return; }
  double *priv = (double *)pool_get(hsz * (size_t)nt * sizeof(double));
#pragma omp parallel num_threads(nt)
  {
#ifdef _OPENMP
    int t = omp_get_thread_num();
#else
    int t = 0;
#endif
    memset(priv + hsz * (size_t)t, 0, hsz * sizeof(double));
    hist_f64_serial(bins, F, g, h, gstride, ridx, nrows * t / nt, nrows * (t + 1) / nt, priv + hsz * (size_t)t);
#pragma omp barrier
#pragma omp for schedule(static)
    for (int64_t j2 = 0; j2 < (int64_t)hsz; ++j2) {
      double sacc = 0;
      for (int t2 = 0; t2 < nt; ++t2) sacc += priv[hsz * (size_t)t2 + (size_t)j2];
      hist[j2] = sacc;
    }
  }
}

/* ------------------------------------------------------------------ sampling (subsample / colsample_* / feature_weights)
 * XGBoost draws row and column samples from per-worker Mersenne twisters (src/common/random.h ColumnSampler,
 * src/tree/hist/sampler.h); that stream cannot be reproduced by another implementation, so the contract is the
 * PUBLISHED behaviour with a counter-based integer hash instead of the twister:
 *   - a row is kept for tree t iff hash(seed, t, rank, row) < subsample * 2^32 (Bernoulli per row and tree;
 *     dropped rows get a zero gradient pair but are still partitioned and receive the leaf value);
 *   - bytree / bylevel / bynode are nested: each scope keeps n = max(1, int(frac * |parent set|)) features of
 *     its parent scope's set; with feature_weights the choice is weighted sampling without replacement
 *     (exponential race: smallest -log2(u)/w), weight 0 sorts last (test_end_to_end.py:429-467). */
static uint64_t mix64(uint64_t x) {
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27; x *= 0x94d049bb133111ebull;
  x ^= x >> 31;
  return x;
}
static uint32_t hash4(uint32_t seed, uint32_t a, uint32_t b, uint32_t c) {
  uint64_t h = mix64((uint64_t)seed * 0x9e3779b97f4a7c15ull + a);
  h = mix64(h + b);
  h = mix64(h + c);
  return (uint32_t)(h >> 32);
}
/* -log2((u | 1) / 2^32) in Q16, integer shift-and-square */
static uint32_t neg_log2_q16(uint32_t u) {
  u |= 1u;
  int e = 0;
  while (!(u & 0x80000000u)) { u <<= 1; ++e; }
  uint64_t x = u;
  uint32_t frac = 0;
  for (int k = 0; k < 16; ++k) {
    x = (x * x) >> 31;
    frac <<= 1;
    if (x >= (1ull << 32)) { frac |= 1u; x >>= 1; }
  }
  return ((uint32_t)(e + 1) << 16) - frac;
}
#define OR_SCOPE_TREE 1u
#define OR_SCOPE_LEVEL(d) (16u + (uint32_t)(d))
#define OR_SCOPE_NODE(nid) (4096u + (uint32_t)(nid))
static uint64_t col_key(uint32_t seed, uint32_t tree, uint32_t scope, uint32_t f, uint32_t wq) {
  if (wq == 0) return 0xffffffffffffffffull;
  return ((uint64_t)neg_log2_q16(hash4(seed, tree, scope, f)) << 24) / wq;
}
/* out[f] = 1 for the n smallest keys among parent (NULL = all features); returns the number selected */
static int select_features(uint32_t seed, uint32_t tree, uint32_t scope, const uint8_t *parent, const uint32_t *fwq,
                           int32_t F, double frac, uint8_t *out) {
  int n_parent = 0;
  for (int32_t f = 0; f < F; ++f) n_parent += (!parent || parent[f]) ? 1 : 0;
  int n_sel = (int)(frac * (double)n_parent);
  if (n_sel < 1) n_sel = 1;
  uint64_t *key = (uint64_t *)malloc((size_t)F * sizeof(uint64_t));
  for (int32_t f = 0; f < F; ++f) key[f] = col_key(seed, tree, scope, (uint32_t)f, fwq ? fwq[f] : 65536u);
  int cnt = 0;
  for (int32_t f = 0; f < F; ++f) {
    out[f] = 0;
    if (parent && !parent[f]) continue;
    int rank = 0;
    for (int32_t g = 0; g < F; ++g) {
      if (g == f || (parent && !parent[g])) continue;
      rank += (key[g] < key[f] || (key[g] == key[f] && g < f)) ? 1 : 0;
    }
    if (rank < n_sel) { out[f] = 1; ++cnt; }
  }
  free(key);
  return cnt;
}
/* select_features as the tree loop calls it, for the column-sampling tests */
int or_select_features(uint32_t seed, uint32_t tree, uint32_t scope, const uint8_t *parent, const uint32_t *fwq, int32_t F,
                       double frac, uint8_t *out) {
  return select_features(seed, tree, scope, parent, fwq, F, frac, out);
}

/* ------------------------------------------------------------------ A.6 split */
static double thr_l1(double g, double a) {
  if (g > a) return g - a;
  if (g < -a) return g + a;
  return 0.0;
}
/* CalcWeight / CalcGain / CalcGainGivenWeight (src/tree/param.h) */
static double calc_weight_d(const OrParams *p, double G, double H) {
  if (H < (double)p->min_child_weight || H <= 0.0) return 0.0;
  double t = p->alpha == 0.0f ? G : thr_l1(G, (double)p->alpha);
  double dw = -t / (H + (double)p->lambda);
  if (p->max_delta_step != 0.0f && fabs(dw) > (double)p->max_delta_step) dw = copysign((double)p->max_delta_step, dw);
  return dw;
}
static double calc_gain(const OrParams *p, double G, double H) {
  if (H < (double)p->min_child_weight || H <= 0.0) return 0.0;
  if (p->max_delta_step == 0.0f) {
    double t = p->alpha == 0.0f ? G : thr_l1(G, (double)p->alpha);
    return (t * t) / (H + (double)p->lambda);
  }
  const double w = calc_weight_d(p, G, H);
  const double ret = -((2.0 * G) * w + (H + (double)p->lambda) * (w * w));
  return p->alpha == 0.0f ? ret : ret + (double)p->alpha * fabs(w);
}
static float calc_weight(const OrParams *p, double G, double H) { return (float)calc_weight_d(p, G, H); }

typedef struct {
  float loss_chg; int32_t feature; int32_t bin; float cond; int default_left;
  double GL, HL, GR, HR; int valid;
  int is_cat; uint32_t cat_bits[8];   /* categorical split: categories (bins) that go right */
} SplitCand;

static void bits_set(uint32_t *b, int i) { b[i >> 5] |= 1u << (i & 31); }
static int bits_test(const uint32_t *b, int i) { return (int)((b[i >> 5] >> (i & 31)) & 1u); }

/* SplitEntry::Update / NeedReplace (src/tree/param.h) */
static int need_replace(const SplitCand *best, float new_chg, int32_t feat) {
  if (isinf(new_chg)) return 0;
  if (!best->valid) return new_chg > best->loss_chg; /* best->loss_chg initialised 0 */
  if (best->feature <= feat) return new_chg > best->loss_chg;
  return !(best->loss_chg > new_chg);
}

#define OR_TRY_CAT(chg_, lg_, lh_, rg_, rh_, bin_, cond_, dl_)                                    \
  if (need_replace(best, (chg_), f)) {                                                           \
    best->loss_chg = (chg_); best->feature = f; best->bin = (bin_); best->cond = (cond_);        \
    best->default_left = (dl_); best->GL = (lg_); best->HL = (lh_); best->GR = (rg_); best->HR = (rh_); \
    best->valid = 1; best->is_cat = 1; memset(best->cat_bits, 0, sizeof(best->cat_bits));       \
    updated = 1;                                                                                 \
  }

/* EnumerateOneHot (evaluate_splits.h): one category against the rest; the chosen category goes right.
 * Per category: first with the missing rows on the left (default_left), then with them on the right. */
static void eval_cat_onehot(const OrParams *p, const float *cv, const double *hf, int32_t nf, int32_t f, double G,
                            double H, float root_gain, SplitCand *best) {
  const double mcw = (double)p->min_child_weight;
  double fg = 0.0, fh = 0.0;
  for (int32_t i = 0; i < nf; ++i) { fg += hf[i * 2]; fh += hf[i * 2 + 1]; }
  const double mg = G - fg, mh = H - fh;   /* missing rows of this node */
  for (int32_t i = 0; i < nf; ++i) {
    for (int pass = 0; pass < 2; ++pass) {
      const double rg = pass ? hf[i * 2] + mg : hf[i * 2], rh = pass ? hf[i * 2 + 1] + mh : hf[i * 2 + 1];
      const double lg = G - rg, lh = H - rh;
      if (lh >= mcw && rh >= mcw) {
        float chg = (float)(calc_gain(p, lg, lh) + calc_gain(p, rg, rh) - (double)root_gain);
        int updated = 0;
        OR_TRY_CAT(chg, lg, lh, rg, rh, i, cv[i], pass ? 0 : 1)
        if (updated) bits_set(best->cat_bits, i);
      }
    }
  }
}

/* EnumeratePart<+1>, <-1> (evaluate_splits.h): categories stable-sorted by leaf weight; forward the
 * lightest k categories go right (missing left), backward the heaviest k go left (missing right); at most
 * min(max_cat_threshold, n) - 1 steps per direction, so neither side is ever empty of categories. */
static void eval_cat_partition(const OrParams *p, const double *hf, int32_t nf, int32_t f, double G, double H,
                               float root_gain, SplitCand *best) {
  const double mcw = (double)p->min_child_weight;
  float w[256]; int32_t idx[256];
  for (int32_t i = 0; i < nf; ++i) { w[i] = calc_weight(p, hf[i * 2], hf[i * 2 + 1]); idx[i] = i; }
  for (int32_t i = 1; i < nf; ++i) {   /* stable insertion sort, ascending weight */
    int32_t v = idx[i], j = i - 1;
    while (j >= 0 && w[idx[j]] > w[v]) { idx[j + 1] = idx[j]; --j; }
    idx[j + 1] = v;
  }
  const int32_t n_bins = p->max_cat_threshold < nf ? p->max_cat_threshold : nf;
  const float nanv = (float)NAN;
  double rg = 0.0, rh = 0.0;
  for (int32_t it = 0; it < n_bins - 1; ++it) {
    rg += hf[idx[it] * 2]; rh += hf[idx[it] * 2 + 1];
    const double lg = G - rg, lh = H - rh;
    if (lh >= mcw && rh >= mcw) {
      float chg = (float)(calc_gain(p, lg, lh) + calc_gain(p, rg, rh) - (double)root_gain);
      int updated = 0;
      OR_TRY_CAT(chg, lg, lh, rg, rh, -1, nanv, 1)
      if (updated) for (int32_t k = 0; k <= it; ++k) bits_set(best->cat_bits, idx[k]);
    }
  }
  double lg = 0.0, lh = 0.0;
  for (int32_t t = 0; t < n_bins - 1; ++t) {
    const int32_t i = nf - 1 - t;
    lg += hf[idx[i] * 2]; lh += hf[idx[i] * 2 + 1];
    const double rg2 = G - lg, rh2 = H - lh;
    if (lh >= mcw && rh2 >= mcw) {
      float chg = (float)(calc_gain(p, lg, lh) + calc_gain(p, rg2, rh2) - (double)root_gain);
      int updated = 0;
      OR_TRY_CAT(chg, lg, lh, rg2, rh2, -1, nanv, 0)
      if (updated) for (int32_t k = 0; k < i; ++k) bits_set(best->cat_bits, idx[k]);
    }
  }
}

/* hist for this node as doubles [F][256][2]; total (G,H) */
static void evaluate_node(const OrParams *p, const OrCuts *c, const double *hist, double G, double H,
                          float root_gain, const uint8_t *feat_mask /* NULL = all features */, SplitCand *best) {
  memset(best, 0, sizeof(*best));
  best->loss_chg = 0.0f; best->feature = 0; best->valid = 0;
  int32_t F = c->n_features;
  for (int32_t f = 0; f < F; ++f) {
    if (feat_mask && !feat_mask[f]) continue;
    const double *hf = hist + (size_t)f * 512;
    int32_t nf = c->cut_ptrs[f + 1] - c->cut_ptrs[f];
    const float *cv = c->cut_vals + c->cut_ptrs[f];
    if (c->is_cat[f]) {
      if (nf < p->max_cat_to_onehot) eval_cat_onehot(p, cv, hf, nf, f, G, H, root_gain, best);
      else eval_cat_partition(p, hf, nf, f, G, H, root_gain, best);
      continue;
    }
    /* forward: missing -> right */
    double eg = 0.0, eh = 0.0;
    for (int32_t i = 0; i < nf; ++i) {
      eg += hf[i * 2]; eh += hf[i * 2 + 1];
      if (eh >= (double)p->min_child_weight) {
        double rg = G - eg, rh = H - eh;
        if (rh >= (double)p->min_child_weight) {
          float chg = (float)(calc_gain(p, eg, eh) + calc_gain(p, rg, rh) - (double)root_gain);
          if (need_replace(best, chg, f)) {
            best->loss_chg = chg; best->feature = f; best->bin = i; best->cond = cv[i];
            best->default_left = 0; best->GL = eg; best->HL = eh; best->GR = rg; best->HR = rh;
            best->valid = 1; best->is_cat = 0;
          }
        }
      }
    }
    /* SplitContainsMissingValues: forward total != node total */
    if (eg != G || eh != H) {
      double bg = 0.0, bh = 0.0;
      for (int32_t i = nf - 1; i >= 0; --i) {
        bg += hf[i * 2]; bh += hf[i * 2 + 1];
        if (bh >= (double)p->min_child_weight) {
          double lg = G - bg, lh = H - bh;
          if (lh >= (double)p->min_child_weight) {
            float chg = (float)(calc_gain(p, lg, lh) + calc_gain(p, bg, bh) - (double)root_gain);
            if (need_replace(best, chg, f)) {
              best->loss_chg = chg; best->feature = f; best->bin = i - 1; /* rows with bin<=i-1 go left */
              best->cond = (i == 0) ? c->min_vals[f] : cv[i - 1];
              best->default_left = 1; best->GL = lg; best->HL = lh; best->GR = bg; best->HR = bh;
              best->valid = 1; best->is_cat = 0;
            }
          }
        }
      }
    }
  }
}

/* ------------------------------------------------------------------ A.7 tree */
static OrTree *tree_new(void) {
  OrTree *t = (OrTree *)calloc(1, sizeof(OrTree));
  t->cap = 64;
#define ALLOC(field, type) t->field = (type *)calloc((size_t)t->cap, sizeof(type))
  ALLOC(left, int32_t); ALLOC(right, int32_t); ALLOC(parent, int32_t); ALLOC(split_feature, int32_t);
  ALLOC(split_bin, int32_t); ALLOC(split_cond, float); ALLOC(default_left, uint8_t); ALLOC(value, float);
  ALLOC(base_weight, float); ALLOC(loss_chg, float); ALLOC(sum_hess, double); ALLOC(sum_grad, double);
  ALLOC(is_cat_split, uint8_t);
  t->cat_bits = (uint32_t *)calloc((size_t)t->cap * 8, sizeof(uint32_t));
#undef ALLOC
  return t;
}
static void tree_free(OrTree *t) {
  free(t->left); free(t->right); free(t->parent); free(t->split_feature); free(t->split_bin);
  free(t->split_cond); free(t->default_left); free(t->value); free(t->base_weight); free(t->loss_chg);
  free(t->sum_hess); free(t->sum_grad); free(t->is_cat_split); free(t->cat_bits); free(t);
}
static int32_t tree_add_node(OrTree *t, int32_t parent) {
  if (t->n_nodes == t->cap) {
    int32_t nc = t->cap * 2;
#define GROW(field, type) t->field = (type *)realloc(t->field, (size_t)nc * sizeof(type))
    GROW(left, int32_t); GROW(right, int32_t); GROW(parent, int32_t); GROW(split_feature, int32_t);
    GROW(split_bin, int32_t); GROW(split_cond, float); GROW(default_left, uint8_t); GROW(value, float);
    GROW(base_weight, float); GROW(loss_chg, float); GROW(sum_hess, double); GROW(sum_grad, double);
    GROW(is_cat_split, uint8_t);
    t->cat_bits = (uint32_t *)realloc(t->cat_bits, (size_t)nc * 8 * sizeof(uint32_t));
#undef GROW
    t->cap = nc;
  }
  int32_t id = t->n_nodes++;
  t->left[id] = t->right[id] = -1; t->parent[id] = parent; t->split_feature[id] = -1; t->split_bin[id] = -1;
  t->split_cond[id] = 0; t->default_left[id] = 0; t->value[id] = 0; t->base_weight[id] = 0;
  t->loss_chg[id] = 0; t->sum_hess[id] = 0; t->sum_grad[id] = 0;
  t->is_cat_split[id] = 0; memset(t->cat_bits + (size_t)id * 8, 0, 32);
  return id;
}

typedef struct {
  int32_t nid, depth;
  int64_t begin, count;   /* segment in ridx */
  double G, H;
  double *hist;           /* [F][256][2] doubles (decoded) */
  int64_t *ihist;         /* exact integer hist when qbits>0 */
  SplitCand split;
} NodeWork;

/* A.8 stable partition of ridx[begin, begin+count) into [left | right]; returns #left.
 * Block-parallel (count, prefix, scatter) for large segments. */
static int64_t partition_segment(int32_t *ridx, int32_t *rtmp, int64_t begin, int64_t count, const uint8_t *bins,
                                 int32_t F, int32_t feature, int32_t split_bin, int has_missing, int default_left,
                                 const uint32_t *cat_bits /* NULL = numeric split */) {
#define GO_LEFT(row) ((bins[(int64_t)(row) * F + feature] == OR_MISSING_BIN && has_missing) \
                          ? default_left                                                      \
                          : (cat_bits ? !bits_test(cat_bits, bins[(int64_t)(row) * F + feature]) \
                                      : ((int32_t)bins[(int64_t)(row) * F + feature] <= split_bin)))
#ifdef _OPENMP
  int nt = omp_in_parallel() ? 1 : omp_get_max_threads();
#else
  int nt = 1;
#endif
  if (count < 65536) nt = 1;
  if (nt == 1) {
    int64_t nl = 0, nr = 0;
    for (int64_t i = begin; i < begin + count; ++i) {
      int32_t row = ridx[i];
      if (GO_LEFT(row)) ridx[begin + nl++] = row; else rtmp[begin + nr++] = row;
    }
    memcpy(ridx + begin + nl, rtmp + begin, (size_t)nr * sizeof(int32_t));
    return nl;
  }
  int64_t *cl = (int64_t *)calloc((size_t)nt + 1, sizeof(int64_t));
  int64_t nl_total = 0;
#pragma omp parallel num_threads(nt)
  {
#ifdef _OPENMP
    int t = omp_get_thread_num();
#else
    int t = 0;
#endif
    int64_t k0 = begin + count * t / nt, k1 = begin + count * (t + 1) / nt, c0 = 0;
    for (int64_t i = k0; i < k1; ++i) c0 += GO_LEFT(ridx[i]) ? 1 : 0;
    cl[t + 1] = c0;
#pragma omp barrier
#pragma omp single
    {
      for (int i = 0; i < nt; ++i) cl[i + 1] += cl[i];
      nl_total = cl[nt];
    }
    int64_t lpos = begin + cl[t], rpos = begin + nl_total + ((k0 - begin) - cl[t]);
    for (int64_t i = k0; i < k1; ++i) {
      int32_t row = ridx[i];
      if (GO_LEFT(row)) rtmp[lpos++] = row; else rtmp[rpos++] = row;
    }
#pragma omp barrier
    memcpy(ridx + k0, rtmp + k0, (size_t)(k1 - k0) * sizeof(int32_t));
  }
  free(cl);
  return nl_total;
#undef GO_LEFT
}

/* grow one tree on (bins, g, h); g/h may be strided (multi-class). Appends leaf values to margin
 * cache: margin[r*mstride] += leaf. */
static OrTree *grow_tree(const OrParams *p, const OrCuts *c, const uint8_t *bins, int64_t n,
                         const float *g, const float *h, int64_t gstride, float *margin, int64_t mstride,
                         int32_t tree_index, const uint32_t *fwq) {
  int32_t F = c->n_features;
  size_t hsz = (size_t)F * 512;
  OrTree *t = tree_new();
  /* row sampling: dropped rows keep their place in the partition but carry a zero gradient pair */
  float *gs = NULL, *hs = NULL;
  if (p->subsample < 1.0f) {
    const double thr_d = (double)p->subsample * 4294967296.0;
    const uint32_t thr = thr_d >= 4294967295.0 ? 0xffffffffu : (uint32_t)thr_d;
    gs = (float *)malloc((size_t)(n > 0 ? n : 1) * sizeof(float)); hs = (float *)malloc((size_t)(n > 0 ? n : 1) * sizeof(float));
    for (int64_t i = 0; i < n; ++i) {
      const int keep = hash4((uint32_t)p->seed, (uint32_t)tree_index, (uint32_t)p->rank, (uint32_t)i) < thr;
      gs[i] = keep ? g[i * gstride] : 0.0f; hs[i] = keep ? h[i * gstride] : 0.0f;
    }
    g = gs; h = hs; gstride = 1;
  }
  /* column sampling: tree set, then one set per level (sampled when the level is first evaluated) */
  const int use_cols = p->colsample_bytree < 1.0f || p->colsample_bylevel < 1.0f || p->colsample_bynode < 1.0f;
  uint8_t *mask_tree = NULL, *mask_level = NULL, *mask_node = NULL; int level_of_mask = -1;
  if (use_cols) {
    mask_tree = (uint8_t *)malloc((size_t)F); mask_level = (uint8_t *)malloc((size_t)F);
    select_features((uint32_t)p->seed, (uint32_t)tree_index, OR_SCOPE_TREE, NULL, fwq, F, (double)p->colsample_bytree, mask_tree);
  }
  int32_t *ridx = (int32_t *)slot_get(SLOT_RIDX, (size_t)(n > 0 ? n : 1) * sizeof(int32_t));
  int32_t *rtmp = (int32_t *)slot_get(SLOT_RTMP, (size_t)(n > 0 ? n : 1) * sizeof(int32_t));
  for (int64_t i = 0; i < n; ++i) ridx[i] = (int32_t)i;
  int32_t *qg = NULL, *qh = NULL; int32_t eg = 0, eh = 0; double inv_sg = 1.0, inv_sh = 1.0;
  if (p->qbits > 0) {
    qg = (int32_t *)slot_get(SLOT_QG, (size_t)(n > 0 ? n : 1) * sizeof(int32_t));
    qh = (int32_t *)slot_get(SLOT_QH, (size_t)(n > 0 ? n : 1) * sizeof(int32_t));
    or_quantize(g, n, gstride, p->qbits, qg, &eg);
    or_quantize(h, n, gstride, p->qbits, qh, &eh);
    inv_sg = ldexp(1.0, eg - p->qbits); inv_sh = ldexp(1.0, eh - p->qbits);
  }
  int32_t cap_level = 1; NodeWork *level = (NodeWork *)calloc(1, sizeof(NodeWork)); int32_t n_level = 1;
  level[0].nid = tree_add_node(t, -1); level[0].depth = 0; level[0].begin = 0; level[0].count = n;
  /* root histogram */
  /* node histograms of a level live in one of two persistent arenas (ping-pong by level parity) */
  int arena = 0;
  level[0].hist = (double *)slot_get(SLOT_HIST0, hsz * sizeof(double));
  if (p->qbits > 0) {
    level[0].ihist = (int64_t *)slot_get(SLOT_IHIST0, hsz * sizeof(int64_t));
    or_hist_int(bins, F, qg, qh, NULL, n, level[0].ihist);
    for (size_t j = 0; j < hsz; j += 2) {
      level[0].hist[j] = (double)level[0].ihist[j] * inv_sg;
      level[0].hist[j + 1] = (double)level[0].ihist[j + 1] * inv_sh;
    }
  } else {
    hist_f64(bins, F, g, h, gstride, NULL, n, level[0].hist);
  }
  { /* root sums = sum of feature-0 bins incl. the missing bin (every row lands in exactly one) */
    double G = 0, H = 0;
    if (p->qbits > 0) {
      int64_t sg = 0, sh = 0;
      for (int b = 0; b < 256; ++b) { sg += level[0].ihist[b * 2]; sh += level[0].ihist[b * 2 + 1]; }
      G = (double)sg * inv_sg; H = (double)sh * inv_sh;
    } else {
      for (int64_t i = 0; i < n; ++i) { G += g[i * gstride]; H += h[i * gstride]; }
    }
    level[0].G = G; level[0].H = H;
  }
  t->sum_grad[0] = level[0].G; t->sum_hess[0] = level[0].H;
  t->base_weight[0] = calc_weight(p, level[0].G, level[0].H);
  (void)cap_level;
  while (n_level > 0) {
    NodeWork *next = (NodeWork *)calloc((size_t)n_level * 2, sizeof(NodeWork)); int32_t n_next = 0;
    /* phase A: evaluate all nodes of the level (node-parallel) */
    int8_t *expand_flag = (int8_t *)calloc((size_t)n_level, 1);
    if (use_cols && n_level > 0 && level[0].depth != level_of_mask) {
      level_of_mask = level[0].depth;
      select_features((uint32_t)p->seed, (uint32_t)tree_index, OR_SCOPE_LEVEL(level_of_mask), mask_tree, fwq, F,
                      (double)p->colsample_bylevel, mask_level);
    }
    if (use_cols && p->colsample_bynode < 1.0f) mask_node = (uint8_t *)malloc((size_t)n_level * F);
#pragma omp parallel for schedule(dynamic, 1)
    for (int32_t k = 0; k < n_level; ++k) {
      NodeWork *w = &level[k];
      if (w->depth < p->max_depth || p->max_depth == 0) {
        float root_gain = (float)calc_gain(p, w->G, w->H);
        const uint8_t *fm = mask_level;
        if (mask_node) {
          select_features((uint32_t)p->seed, (uint32_t)tree_index, OR_SCOPE_NODE(w->nid), mask_level, fwq, F,
                          (double)p->colsample_bynode, mask_node + (size_t)k * F);
          fm = mask_node + (size_t)k * F;
        }
        evaluate_node(p, c, w->hist, w->G, w->H, root_gain, fm, &w->split);
        SplitCand *sc = &w->split;
        expand_flag[k] = sc->valid && sc->loss_chg > OR_RT_EPS && sc->HL != 0.0 && sc->HR != 0.0 &&
                         !(sc->loss_chg < p->gamma);
      }
    }
    /* phase B: apply in node order (ids are allocated consecutively, A.7) */
    int32_t n_pairs = 0;
    int32_t *pair_parent = (int32_t *)malloc((size_t)n_level * sizeof(int32_t));
    for (int32_t k = 0; k < n_level; ++k) {
      NodeWork *w = &level[k];
      int32_t nid = w->nid;
      if (!expand_flag[k]) {
        if (p->qbits > 0) {
          /* leaf refinement: leaf weight from 40-bit fixed-point sums of the fp32 gradients of the
           * leaf's rows (exact int64 limbs, order independent), so leaf values do not depend on qbits */
          int64_t ghi = 0, glo = 0, hhi = 0, hlo = 0;
          double kg = ldexp(1.0, OR_LEAF_BITS - eg), kh = ldexp(1.0, OR_LEAF_BITS - eh);
#pragma omp parallel for reduction(+ : ghi, glo, hhi, hlo) schedule(static) if (w->count > 65536)
          for (int64_t i = w->begin; i < w->begin + w->count; ++i) {
            int64_t r = ridx[i];
            const int64_t qg = llrint((double)g[r * gstride] * kg), qh = llrint((double)h[r * gstride] * kh);
            ghi += qg >> OR_LIMB_SHIFT; glo += qg & OR_LIMB_MASK; hhi += qh >> OR_LIMB_SHIFT; hlo += qh & OR_LIMB_MASK;
          }
          t->base_weight[nid] = calc_weight(p, or_limbs_to_double(ghi, glo) / kg, or_limbs_to_double(hhi, hlo) / kh);
        }
        t->value[nid] = t->base_weight[nid] * p->eta;
        const float lv = t->value[nid];
#pragma omp parallel for schedule(static) if (w->count > 65536)
        for (int64_t i = w->begin; i < w->begin + w->count; ++i)
          margin[(int64_t)ridx[i] * mstride] += lv;
        continue;
      }
      SplitCand *s = &w->split;
      int32_t l = tree_add_node(t, nid), r = tree_add_node(t, nid);
      t->left[nid] = l; t->right[nid] = r; t->split_feature[nid] = s->feature; t->split_bin[nid] = s->bin;
      t->split_cond[nid] = s->cond; t->default_left[nid] = (uint8_t)s->default_left;
      t->loss_chg[nid] = s->loss_chg; t->value[nid] = t->base_weight[nid];
      t->is_cat_split[nid] = (uint8_t)s->is_cat;
      if (s->is_cat) memcpy(t->cat_bits + (size_t)nid * 8, s->cat_bits, 32);
      t->sum_grad[l] = s->GL; t->sum_hess[l] = s->HL; t->sum_grad[r] = s->GR; t->sum_hess[r] = s->HR;
      t->base_weight[l] = calc_weight(p, s->GL, s->HL); t->base_weight[r] = calc_weight(p, s->GR, s->HR);
      /* A.8 partition (stable): left iff non-missing && bin <= split_bin, missing -> default */
      /* categorical: rows whose category is in the set go right (A.8) */
      int64_t nl = partition_segment(ridx, rtmp, w->begin, w->count, bins, F, s->feature, s->bin,
                                     c->has_missing[s->feature], s->default_left, s->is_cat ? s->cat_bits : NULL);
      int64_t nr = w->count - nl;
      NodeWork *wl = &next[n_next++], *wr = &next[n_next++];
      wl->nid = l; wl->depth = w->depth + 1; wl->begin = w->begin; wl->count = nl; wl->G = s->GL; wl->H = s->HL;
      wr->nid = r; wr->depth = w->depth + 1; wr->begin = w->begin + nl; wr->count = nr; wr->G = s->GR; wr->H = s->HR;
      pair_parent[n_pairs++] = k;
    }
    /* phase C: histograms of the children (A.5): build the smaller-hessian child from rows,
     * sibling = parent - built.  Node-parallel when there are many nodes, row-parallel otherwise. */
    if (n_pairs > 0 && ((level[pair_parent[0]].depth + 1 < p->max_depth) || p->max_depth == 0)) {
      const int na = arena ^ 1;
      double *hblock = (double *)slot_get(na ? SLOT_HIST1 : SLOT_HIST0, (size_t)n_next * hsz * sizeof(double));
      int64_t *iblock = p->qbits > 0 ? (int64_t *)slot_get(na ? SLOT_IHIST1 : SLOT_IHIST0, (size_t)n_next * hsz * sizeof(int64_t)) : NULL;
      for (int32_t q = 0; q < n_next; ++q) { next[q].hist = hblock + (size_t)q * hsz; next[q].ihist = iblock ? iblock + (size_t)q * hsz : NULL; }
      arena = na;
      /* pass 0: nodes big enough for a row-parallel build, one after the other;
       * pass 1: the remaining (small) nodes in parallel, each built serially into its own buffer */
      for (int pass = 0; pass < 2; ++pass) {
#pragma omp parallel for schedule(dynamic, 1) if (pass == 1)
        for (int32_t j = 0; j < n_pairs; ++j) {
          NodeWork *w = &level[pair_parent[j]];
          NodeWork *wl = &next[2 * j], *wr = &next[2 * j + 1];
          NodeWork *bw = (wl->H < wr->H) ? wl : wr, *sw = (bw == wl) ? wr : wl;
          int big = bw->count >= 2 * (int64_t)OR_ROWS_PER_THREAD;
          if (big != (pass == 0)) continue;
          if (p->qbits > 0) {
            or_hist_int(bins, F, qg, qh, ridx + bw->begin, bw->count, bw->ihist);
            for (size_t jj = 0; jj < hsz; ++jj) sw->ihist[jj] = w->ihist[jj] - bw->ihist[jj];
            for (size_t jj = 0; jj < hsz; jj += 2) {
              bw->hist[jj] = (double)bw->ihist[jj] * inv_sg; bw->hist[jj + 1] = (double)bw->ihist[jj + 1] * inv_sh;
              sw->hist[jj] = (double)sw->ihist[jj] * inv_sg; sw->hist[jj + 1] = (double)sw->ihist[jj + 1] * inv_sh;
            }
          } else {
            hist_f64(bins, F, g, h, gstride, ridx + bw->begin, bw->count, bw->hist);
            for (size_t jj = 0; jj < hsz; ++jj) sw->hist[jj] = w->hist[jj] - bw->hist[jj];
          }
        }
      }
    }
    free(expand_flag); free(pair_parent); free(mask_node); mask_node = NULL;
    free(level); level = next; n_level = n_next;
  }
  free(level); free(gs); free(hs); free(mask_tree); free(mask_level);
  return t;
}

/* ------------------------------------------------------------------ model */
OrModel *or_model_new(const OrParams *p, int32_t n_features) {
  OrModel *m = (OrModel *)calloc(1, sizeof(OrModel));
  m->p = *p; m->n_features = n_features; m->cap_trees = 16;
  m->trees = (OrTree **)calloc((size_t)m->cap_trees, sizeof(OrTree *));
  if (m->p.num_class < 1) m->p.num_class = 1;
  return m;
}
void or_model_free(OrModel *m) {
  if (!m) return;
  for (int i = 0; i < m->n_trees; ++i) tree_free(m->trees[i]);
  free(m->trees); free(m->fwq); free(m);
}
/* feature_weights (DMatrix.set_info(feature_weights=...), main.py:439-442): Q16, negative -> invalid (returns -1) */
int or_model_set_feature_weights(OrModel *m, const float *fw, int32_t len) {
  if (len != m->n_features) return -1;
  for (int32_t f = 0; f < len; ++f) if (!(fw[f] >= 0.0f) || isinf(fw[f])) return -1;
  free(m->fwq);
  m->fwq = (uint32_t *)malloc((size_t)len * sizeof(uint32_t));
  for (int32_t f = 0; f < len; ++f) {
    double q = (double)fw[f] * 65536.0;
    m->fwq[f] = q >= 4294967295.0 ? 0xffffffffu : (uint32_t)llrint(q);
  }
  return 0;
}
static void model_push(OrModel *m, OrTree *t) {
  if (m->n_trees == m->cap_trees) {
    m->cap_trees *= 2; m->trees = (OrTree **)realloc(m->trees, (size_t)m->cap_trees * sizeof(OrTree *));
  }
  m->trees[m->n_trees++] = t;
}
float or_base_margin(const OrParams *p) {
  if (p->objective == OR_OBJ_LOGISTIC) return -logf(1.0f / p->base_score - 1.0f);
  return p->base_score;
}

/* A.3 base_score when the user gave none (xgboost >= 2.0: ObjFunction::InitEstimation -> FitIntercept::InitEstimation,
 * tree::FitStump): one Newton step of a stump at margin 0, -sum(g)/sum(h) (no regularisation; 0 when sum(h) <= 1e-6),
 * then the inverse link (identity / sigmoid).  Multi-class keeps 0.5.  Sums are 40-bit fixed point (exact). */
float or_estimate_base_score(OrModel *m, const float *label, const float *weight, int64_t n) {
  if (m->p.objective == OR_OBJ_SOFTPROB) return m->p.base_score;
  float *zeros = (float *)calloc((size_t)(n > 0 ? n : 1), sizeof(float));
  float *g = (float *)malloc((size_t)(n > 0 ? n : 1) * sizeof(float)), *h = (float *)malloc((size_t)(n > 0 ? n : 1) * sizeof(float));
  or_gradients_spw(m->p.objective, 1, zeros, label, weight, n, m->p.scale_pos_weight, g, h);
  float mg = 0.0f, mh = 0.0f;
  for (int64_t i = 0; i < n; ++i) { if (fabsf(g[i]) > mg) mg = fabsf(g[i]); if (fabsf(h[i]) > mh) mh = fabsf(h[i]); }
  const int32_t eg = or_quant_exponent(mg), eh = or_quant_exponent(mh);
  const double kg = ldexp(1.0, OR_LEAF_BITS - eg), kh = ldexp(1.0, OR_LEAF_BITS - eh);
  int64_t ghi = 0, glo = 0, hhi = 0, hlo = 0;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t qg = llrint((double)g[i] * kg), qh = llrint((double)h[i] * kh);
    ghi += qg >> OR_LIMB_SHIFT; glo += qg & OR_LIMB_MASK; hhi += qh >> OR_LIMB_SHIFT; hlo += qh & OR_LIMB_MASK;
  }
  const double G = or_limbs_to_double(ghi, glo) / kg, H = or_limbs_to_double(hhi, hlo) / kh;
  const float stump = H <= 1e-6 ? 0.0f : (float)(-G / H);
  free(zeros); free(g); free(h);
  m->p.base_score = m->p.objective == OR_OBJ_LOGISTIC ? or_sigmoid(stump) : stump;
  return m->p.base_score;
}

/* One boosting round.  margin [n*K] is the prediction cache (in/out).  custom_g/custom_h
 * (may be NULL) replace the objective gradient (xgb.train(obj=...), test_xgboost_api.py:77-102). */
int or_boost_one_round(OrModel *m, const OrCuts *c, const uint8_t *bins, int64_t n, const float *label,
                       const float *weight, float *margin, const float *custom_g, const float *custom_h) {
#ifdef _OPENMP
  if (m->p.nthread > 0) omp_set_num_threads(m->p.nthread);
#endif
  int K = m->p.num_class;
  float *g = NULL, *h = NULL;
  const float *gg = custom_g, *hh = custom_h;
  if (!custom_g) {
    g = (float *)slot_get(SLOT_G, (size_t)(n * K > 0 ? n * K : 1) * sizeof(float));
    h = (float *)slot_get(SLOT_H, (size_t)(n * K > 0 ? n * K : 1) * sizeof(float));
    or_gradients_spw(m->p.objective, K, margin, label, weight, n, m->p.scale_pos_weight, g, h);
    gg = g; hh = h;
  }
  for (int k = 0; k < K; ++k) {
    OrTree *t = grow_tree(&m->p, c, bins, n, gg + k, hh + k, K, margin + k, K, m->n_trees, m->fwq);
    model_push(m, t);
  }
  return 0;
}

int32_t or_num_trees(const OrModel *m) { return m->n_trees; }
int32_t or_tree_num_nodes(const OrModel *m, int32_t t) { return m->trees[t]->n_nodes; }
void or_tree_get(const OrModel *m, int32_t ti, int32_t *left, int32_t *right, int32_t *parent,
                 int32_t *split_feature, int32_t *split_bin, float *split_cond, uint8_t *default_left,
                 float *value, float *base_weight, float *loss_chg, double *sum_hess) {
  const OrTree *t = m->trees[ti]; size_t n = (size_t)t->n_nodes;
  memcpy(left, t->left, n * 4); memcpy(right, t->right, n * 4); memcpy(parent, t->parent, n * 4);
  memcpy(split_feature, t->split_feature, n * 4); memcpy(split_bin, t->split_bin, n * 4);
  memcpy(split_cond, t->split_cond, n * 4); memcpy(default_left, t->default_left, n);
  memcpy(value, t->value, n * 4); memcpy(base_weight, t->base_weight, n * 4);
  memcpy(loss_chg, t->loss_chg, n * 4); memcpy(sum_hess, t->sum_hess, n * 8);
}

/* categorical part of a tree: split_type [n] (1 = categorical), cat_bits [n][8] */
void or_tree_get_cat(const OrModel *m, int32_t ti, uint8_t *split_type, uint32_t *cat_bits) {
  const OrTree *t = m->trees[ti]; size_t n = (size_t)t->n_nodes;
  memcpy(split_type, t->is_cat_split, n); memcpy(cat_bits, t->cat_bits, n * 32);
}

/* A.9 prediction on raw floats: x < split_cond -> left; missing -> default.  Categorical node
 * (common/categorical.h Decision): category in the set -> right; not in the set, negative or beyond the set -> left */
void or_predict_margin(const OrModel *m, const float *X, int64_t n, float missing, int32_t tree_begin,
                       int32_t tree_end, const float *base_margin, float *out) {
  int K = m->p.num_class; int32_t F = m->n_features;
  float bm = or_base_margin(&m->p);
  if (tree_end <= 0 || tree_end > m->n_trees) tree_end = m->n_trees;
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < n; ++i) {
    for (int k = 0; k < K; ++k) out[i * K + k] = base_margin ? base_margin[i * K + k] : bm;
    for (int32_t ti = tree_begin; ti < tree_end; ++ti) {
      const OrTree *t = m->trees[ti]; int32_t nid = 0;
      while (t->split_feature[nid] >= 0) {
        float x = X[i * F + t->split_feature[nid]];
        if (is_missing(x, missing)) nid = t->default_left[nid] ? t->left[nid] : t->right[nid];
        else if (t->is_cat_split[nid]) {
          const int in_set = x >= 0.0f && x < 256.0f && bits_test(t->cat_bits + (size_t)nid * 8, (int)x);
          nid = in_set ? t->right[nid] : t->left[nid];
        }
        else nid = (x < t->split_cond[nid]) ? t->left[nid] : t->right[nid];
      }
      out[i * K + (ti % K)] += t->value[nid];
    }
  }
}

/* margin -> output transform (identity / sigmoid / softmax) in place */
void or_transform(int32_t objective, int32_t K, float *m, int64_t n) {
  if (objective == OR_OBJ_LOGISTIC) {
    for (int64_t i = 0; i < n; ++i) m[i] = or_sigmoid(m[i]);
  } else if (objective == OR_OBJ_SOFTPROB) {
    for (int64_t i = 0; i < n; ++i) {
      float *r = m + i * K; float mx = r[0];
      for (int k = 1; k < K; ++k) if (r[k] > mx) mx = r[k];
      float s = 0.0f;
      for (int k = 0; k < K; ++k) { r[k] = or_expf(r[k] - mx); s = s + r[k]; }
      for (int k = 0; k < K; ++k) r[k] = r[k] / s;
    }
  }
}

/* A.10 metrics on margins: returns (sum, wsum) so callers can combine shards.  Metrics see the transformed
 * prediction (ObjFunction::EvalTransform): probability for binary:logistic, raw value for reg:squarederror.
 * metric: 0 rmse, 1 logloss, 2 error, 3 mlogloss, 4 merror, 5 mae */
void or_metric_sums_obj(int32_t objective, int32_t metric, int32_t K, const float *margin, const float *label,
                        const float *weight, int64_t n, double *out_sum, double *out_wsum);
void or_metric_sums(int32_t metric, int32_t K, const float *margin, const float *label, const float *weight,
                    int64_t n, double *out_sum, double *out_wsum) {
  /* historical entry point: logloss / error on margins of a logistic model, rmse on raw values */
  or_metric_sums_obj((metric == 1 || metric == 2) ? OR_OBJ_LOGISTIC : OR_OBJ_SQUAREDERROR, metric, K, margin, label, weight, n,
                     out_sum, out_wsum);
}
void or_metric_sums_obj(int32_t objective, int32_t metric, int32_t K, const float *margin, const float *label,
                        const float *weight, int64_t n, double *out_sum, double *out_wsum) {
  double s = 0.0, ws = 0.0;
  for (int64_t i = 0; i < n; ++i) {
    double w = weight ? weight[i] : 1.0; double v = 0.0;
    if (metric <= 2 || metric == 5) {
      float p = objective == OR_OBJ_LOGISTIC ? or_sigmoid(margin[i]) : margin[i];
      if (metric == 0) { double d = (double)p - (double)label[i]; v = d * d; }
      else if (metric == 5) v = fabs((double)p - (double)label[i]);
      else if (metric == 1) {
        const float eps = 1e-16f; float y = label[i];
        float pn = 1.0f - p;
        float a = p < eps ? eps : p, b = pn < eps ? eps : pn;
        v = -((double)y * log((double)a) + (1.0 - (double)y) * log((double)b));
      } else v = (p > 0.5f) != (label[i] > 0.5f) ? 1.0 : 0.0;
    }
    else {
      const float *r = margin + i * K; int y = (int)label[i]; float mx = r[0]; int am = 0;
      for (int k = 1; k < K; ++k) if (r[k] > mx) { mx = r[k]; am = k; }
      if (metric == 4) v = (am != y) ? 1.0 : 0.0;
      else {
        float ssum = 0.0f; for (int k = 0; k < K; ++k) ssum = ssum + or_expf(r[k] - mx);
        float p = or_expf(r[y] - mx) / ssum; if (p < 1e-16f) p = 1e-16f;
        v = -log((double)p);
      }
    }
    s += v * w; ws += w;
  }
  *out_sum = s; *out_wsum = ws;
}

void or_set_num_threads(int32_t n) {
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
#else
  (void)n;
#endif
}

int32_t or_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
