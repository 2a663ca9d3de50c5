// sampling.cuh -- row / column sampling decisions (subsample, colsample_by{tree,level,node}, feature_weights).
//
// XGBoost draws these from a Mersenne twister per worker (src/common/random.h ColumnSampler,
// src/tree/hist/sampler.h), which no other implementation can reproduce bit for bit; the parity contract here is
// with the oracle (oracle/hist_oracle.c restates the same functions).  Everything is integer arithmetic on a
// counter-based hash, so the host, the kernels and the oracle take identical decisions and the column choices do
// not depend on the number of GPUs:
//   row i of tree t on rank r is kept      iff  hash(seed, t, r, i) < subsample * 2^32
//   a scope (tree / level d / node nid) keeps the n = max(1, int(frac * |parent set|)) features of its parent set
//   with the smallest keys  key(f) = -log2(u_f) / w_f,  u_f = hash(seed, t, scope, f)  (exponential race =
//   weighted sampling without replacement, ColumnSampler's WeightedSamplingWithoutReplacement); ties -> lower f;
//   w_f = feature_weights[f] (1 when absent), features of weight 0 come last.
#pragma once
#include <stdint.h>
#include <stdlib.h>
#ifndef __cplusplus
#include <stdbool.h>
#endif

#ifdef __CUDACC__
#define B2_HD __host__ __device__ __forceinline__
#else
#define B2_HD static inline
#endif

B2_HD uint64_t b2_mix64(uint64_t x) {   // splitmix64 finaliser
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27; x *= 0x94d049bb133111ebull;
  x ^= x >> 31;
  return x;
}
B2_HD uint32_t b2_hash4(uint32_t seed, uint32_t a, uint32_t b, uint32_t c) {
  uint64_t h = b2_mix64((uint64_t)seed * 0x9e3779b97f4a7c15ull + a);
  h = b2_mix64(h + b);
  h = b2_mix64(h + c);
  return (uint32_t)(h >> 32);
}
// -log2((u | 1) / 2^32) in Q16 fixed point, integer only (shift-and-square)
B2_HD uint32_t b2_neg_log2_q16(uint32_t u) {
  u |= 1u;
  int e = 0;
  while (!(u & 0x80000000u)) { u <<= 1; ++e; }        // u = 1.xxx * 2^31, value = u / 2^(32+e) ... in [0.5,1) * 2^-e
  // log2(value) = -(e + 1) + log2(m), m = u / 2^31 in [1, 2)
  uint64_t x = u;                                       // Q31
  uint32_t frac = 0;
  for (int k = 0; k < 16; ++k) {
    x = (x * x) >> 31;                                  // Q31, in [1, 4)
    frac <<= 1;
    if (x >= (1ull << 32)) { frac |= 1u; x >>= 1; }
  }
  return ((uint32_t)(e + 1) << 16) - frac;              // (e + 1) - log2(m) >= 0
}
// scope ids of the column sampler
#define B2_SCOPE_TREE 1u
#define B2_SCOPE_LEVEL(d) (16u + (uint32_t)(d))
#define B2_SCOPE_NODE(nid) (4096u + (uint32_t)(nid))
// wq: feature weight in Q16 (65536 = 1.0); 0 sorts last
B2_HD uint64_t b2_col_key(uint32_t seed, uint32_t tree, uint32_t scope, uint32_t f, uint32_t wq) {
  if (wq == 0) return 0xffffffffffffffffull;
  return ((uint64_t)b2_neg_log2_q16(b2_hash4(seed, tree, scope, f)) << 24) / wq;
}
B2_HD int b2_sample_count(double frac, int n_parent) {
  int n = (int)(frac * (double)n_parent);
  return n < 1 ? 1 : n;
}
// is feature f among the n_sel smallest keys of the features with parent[f'] != 0 ?  One answer costs F key
// evaluations: the per-node path of the split scan asks it for the few slots of one CTA.
B2_HD bool b2_col_selected(uint32_t seed, uint32_t tree, uint32_t scope, int f, const uint8_t* parent, const uint32_t* wq, int F,
                           int n_sel) {
  if (parent && !parent[f]) return false;
  const uint64_t kf = b2_col_key(seed, tree, scope, (uint32_t)f, wq ? wq[f] : 65536u);
  int rank = 0;
  for (int g = 0; g < F; ++g) {
    if (g == f || (parent && !parent[g])) continue;
    const uint64_t kg = b2_col_key(seed, tree, scope, (uint32_t)g, wq ? wq[g] : 65536u);
    rank += (kg < kf || (kg == kf && g < f)) ? 1 : 0;
  }
  return rank < n_sel;
}
// Host-only whole-mask form of b2_col_selected: out[f] = 1 for the n_sel features of the parent set with the smallest
// (key, f), 0 elsewhere.  Each key is computed once and the parent set sorted, O(F log F) instead of F^2 key
// evaluations; (key, f) is a total order, so the set is exactly the one b2_col_selected picks.  scratch holds F
// entries.  Returns the number of features selected.
typedef struct { uint64_t key; int32_t f; } B2ColRank;
static inline int b2_col_rank_cmp(const void* a, const void* b) {
  const B2ColRank* x = (const B2ColRank*)a;
  const B2ColRank* y = (const B2ColRank*)b;
  if (x->key != y->key) return x->key < y->key ? -1 : 1;
  return (x->f > y->f) - (x->f < y->f);
}
static inline int b2_col_select(uint32_t seed, uint32_t tree, uint32_t scope, const uint8_t* parent, const uint32_t* wq, int F,
                                int n_sel, B2ColRank* scratch, uint8_t* out) {
  int m = 0;
  for (int f = 0; f < F; ++f) m += (!parent || parent[f]) ? 1 : 0;
  if (n_sel >= m) {                      // the whole parent set (a fraction of 1.0): no key is needed
    for (int f = 0; f < F; ++f) out[f] = (!parent || parent[f]) ? 1 : 0;
    return m;
  }
  m = 0;
  for (int f = 0; f < F; ++f) {
    out[f] = 0;
    if (parent && !parent[f]) continue;
    scratch[m].key = b2_col_key(seed, tree, scope, (uint32_t)f, wq ? wq[f] : 65536u);
    scratch[m].f = f;
    ++m;
  }
  qsort(scratch, (size_t)m, sizeof(B2ColRank), b2_col_rank_cmp);
  for (int i = 0; i < n_sel; ++i) out[scratch[i].f] = 1;
  return n_sel;
}
B2_HD uint32_t b2_subsample_threshold(double subsample) {
  const double t = subsample * 4294967296.0;
  return t >= 4294967295.0 ? 0xffffffffu : (uint32_t)t;
}
