// rank_kernel.cu -- learning to rank: the per-group model order, LambdaMART gradients of rank:pairwise / rank:ndcg
// (xgboost 2.x, lambdarank_pair_method=topk) and the per-group ndcg / map / pre metrics.
//
// A query group is a run of rows [gptr[g], gptr[g+1]) of one worker's matrix; the host keeps every group whole on one
// worker, so nothing here crosses a worker.  The rules (DESIGN.md 2, item 13) are restated operation for operation by
// tests/ranking_reference.py: binary32 where marked, binary64 otherwise, compiled with --fmad=false, so the gradient
// pairs are bit-equal.
//
// Order: one CUB segmented STABLE sort per round of 32-bit keys that sort descending by the canonicalised margin
// (m + 0.0f: -0.0 == +0.0), with the row index as value -- ties keep their row order.  Labels are ordered the same way
// once per matrix for IDCG.
#include <cub/device/device_segmented_sort.cuh>

#include <cfloat>
#include "common.cuh"
#include "objective_common.cuh"

namespace b2 {

constexpr double kRankLn2 = 0.69314718055994530942;   // the binary64 nearest ln 2 (numpy's log(2))
constexpr int kRankThreads = 128;
constexpr int kRankStageRows = 2048;                   // groups up to this size are staged in shared memory (32 KB)

// ascending sort key of a float that orders it DESCENDING; -0.0 is canonicalised to +0.0 first
__device__ __forceinline__ uint32_t rank_desc_key(float v) {
  uint32_t u = __float_as_uint(__fadd_rn(v, 0.0f));
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ~u;
}
__device__ __forceinline__ float rank_key_value(uint32_t key) {
  const uint32_t a = ~key;
  return __uint_as_float((a & 0x80000000u) ? (a & 0x7fffffffu) : ~a);
}

// gain of a label: 2^y - 1 (exact for an integer y, b2_exp(y ln2) - 1 otherwise) or y itself
__device__ __forceinline__ double rank_gain(float y, bool exp_gain) {
  const double yd = (double)y;
  if (!exp_gain) return yd;
  if (yd == floor(yd)) return B2_DS(ldexp(1.0, (int)yd), 1.0);
  return B2_DS(b2_exp(B2_DM(yd, kRankLn2)), 1.0);
}

__global__ void rank_keys_kernel(const float* __restrict__ v, int64_t n, uint32_t* __restrict__ keys) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    keys[i] = rank_desc_key(v[i]);
}
__global__ void rank_iota_kernel(int32_t* __restrict__ idx, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    idx[i] = (int32_t)i;
}

// discount of model position r: ln2 / log(r + 2), with the fdlibm log (b2_log)
__global__ void rank_disc_kernel(double* __restrict__ disc, int64_t len) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < len; r += (int64_t)gridDim.x * blockDim.x)
    disc[r] = B2_DD(kRankLn2, b2_log((double)(r + 2)));
}

// 1 / IDCG@k of every group from its labels sorted descending (0 when IDCG is 0); one thread per group, t ascending
__global__ void rank_inv_idcg_kernel(const int64_t* __restrict__ gptr, int64_t n_groups, const uint32_t* __restrict__ lkeys,
                                     const double* __restrict__ disc, int k, int exp_gain, double* __restrict__ inv_idcg) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = gptr[g], n = gptr[g + 1] - b, t_end = n < k ? n : k;
    double s = 0.0;
    for (int64_t t = 0; t < t_end; ++t) s = B2_DA(s, B2_DM(rank_gain(rank_key_value(lkeys[b + t]), exp_gain), disc[t]));
    inv_idcg[g] = s == 0.0 ? 0.0 : B2_DD(1.0, s);
  }
}

// labels of a rank objective (once per train matrix): bad[0] a label that is NaN, infinite or negative,
// bad[1] a label above 31 with ndcg_exp_gain (2^y - 1 would not be exact)
__global__ void rank_label_check_kernel(const float* __restrict__ label, int64_t n, int exp_gain, uint32_t* __restrict__ bad) {
  bool b0 = false, b1 = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float y = label[i];
    b0 |= !(y >= 0.0f) || isinf(y);
    b1 |= exp_gain && y > 31.0f;
  }
  if (__any_sync(0xffffffffu, b0) && (threadIdx.x & 31) == 0) atomicOr(&bad[0], 1u);
  if (__any_sync(0xffffffffu, b1) && (threadIdx.x & 31) == 0) atomicOr(&bad[1], 1u);
}

// the pair (a, b) of model positions ra < rb with different labels: returns (float lambda, float H); *a_high says
// whether a has the larger label
template <bool kNdcg>
__device__ __forceinline__ float2 lambda_pair(float sa, float ya, int ra, float sb, float yb, int rb, bool exp_gain,
                                              const double* __restrict__ disc, double inv_idcg, bool scale_by_diff,
                                              bool* a_high) {
  const bool ah = ya > yb;
  *a_high = ah;
  const float d = ah ? __fadd_rn(sa, -sb) : __fadd_rn(sb, -sa);
  const double sig = (double)b2_sigmoid(d);
  double delta = 1.0;
  if (kNdcg) {
    const double gh = rank_gain(ah ? ya : yb, exp_gain), gl = rank_gain(ah ? yb : ya, exp_gain);
    const double dh = disc[ah ? ra : rb], dl = disc[ah ? rb : ra];
    const double t = B2_DS(B2_DA(B2_DM(gh, dh), B2_DM(gl, dl)), B2_DA(B2_DM(gl, dh), B2_DM(gh, dl)));
    delta = fabs(B2_DM(t, inv_idcg));
  }
  if (scale_by_diff) delta = B2_DD(delta, B2_DA((double)fabsf(d), 0.01));
  const double lam = B2_DM(B2_DS(sig, 1.0), delta);
  const double hh = fmax(B2_DM(sig, B2_DS(1.0, sig)), 1e-16);
  const double H = B2_DM(B2_DM(hh, delta), 2.0);
  return make_float2(__double2float_rn(lam), __double2float_rn(H));
}

// One CTA per group at a time (grid-stride over groups).  The group's sorted margins and labels (and the per-position
// pair sums P) live in shared memory when the group has at most `stage` rows (the largest group, capped at
// kRankStageRows), in the global scratch otherwise -- the same code through a pointer switch.  The thread that owns
// model position r replays r's pairs in the order of the sequential `for i < min(k, n): for j > i` loop restricted to r:
// first (i, r) for i < min(r, k), then (r, j) for j > r when r < k, accumulating in binary32.  P_r = sum_j
// -2 lambda(r, j) in binary64, S = sum_r P_r by one thread in r order, then every row is scaled by log2(1 + S) / S when
// S > 0.  Writes gh[row], the block's |g|, |h| maxima and *err when a
// pair is not finite (written as (0, 0), like the other gradient kernels).
template <bool kNdcg>
__global__ void __launch_bounds__(kRankThreads)
lambdarank_gradient_kernel(const int64_t* __restrict__ gptr, int64_t n_groups, const uint32_t* __restrict__ skeys,
                           const int32_t* __restrict__ srow, const float* __restrict__ label,
                           const double* __restrict__ inv_idcg, const double* __restrict__ disc, int k, int exp_gain,
                           int stage, float* __restrict__ scratch_m, float* __restrict__ scratch_y, double* __restrict__ scratch_p,
                           float2* __restrict__ gh, uint32_t* __restrict__ absmax, uint32_t* __restrict__ err) {
  extern __shared__ __align__(16) unsigned char rank_smem[];
  __shared__ double s_norm;
  float mg = 0.0f, mh = 0.0f;
  bool bad = false;
  for (int64_t g = blockIdx.x; g < n_groups; g += gridDim.x) {
    const int64_t beg = gptr[g];
    const int n = (int)(gptr[g + 1] - beg);
    const bool staged = n <= stage;
    double* P = staged ? (double*)rank_smem : scratch_p + beg;
    float* M = staged ? (float*)(rank_smem + (size_t)stage * 8) : scratch_m + beg;
    float* Y = staged ? M + stage : scratch_y + beg;
    __syncthreads();                                   // the previous group's readers are done with the stage
    for (int p = threadIdx.x; p < n; p += blockDim.x) { M[p] = rank_key_value(skeys[beg + p]); Y[p] = label[srow[beg + p]]; }
    __syncthreads();
    const int kk = n < k ? n : k;
    const bool scale = n > 0 && M[0] != M[n - 1];
    const double inv = kNdcg ? inv_idcg[g] : 0.0;
    for (int r = threadIdx.x; r < n; r += blockDim.x) {
      const float sr = M[r], yr = Y[r];
      float gr = 0.0f, hr = 0.0f;
      bool hi;
      const int lim = r < k ? r : k;
      for (int i = 0; i < lim; ++i) {
        const float yi = Y[i];
        if (yi == yr) continue;
        const float2 pg = lambda_pair<kNdcg>(M[i], yi, i, sr, yr, r, exp_gain, disc, inv, scale, &hi);
        gr = __fadd_rn(gr, hi ? -pg.x : pg.x);         // hi: position i is the high member, r the low one
        hr = __fadd_rn(hr, pg.y);
      }
      if (r < k) {
        double pr = 0.0;
        for (int j = r + 1; j < n; ++j) {
          const float yj = Y[j];
          if (yj == yr) continue;
          const float2 pg = lambda_pair<kNdcg>(sr, yr, r, M[j], yj, j, exp_gain, disc, inv, scale, &hi);
          gr = __fadd_rn(gr, hi ? pg.x : -pg.x);
          hr = __fadd_rn(hr, pg.y);
          pr = B2_DA(pr, B2_DM(-2.0, (double)pg.x));
        }
        P[r] = pr;
      }
      gh[srow[beg + r]] = make_float2(gr, hr);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double S = 0.0;
      for (int i = 0; i < kk; ++i) S = B2_DA(S, P[i]);
      // S <= 0: no normalisation; x * 1.0 rounds back to x exactly
      s_norm = S > 0.0 ? B2_DD(B2_DD(b2_log(B2_DA(1.0, S)), kRankLn2), S) : 1.0;
    }
    __syncthreads();
    const double norm = s_norm;
    for (int r = threadIdx.x; r < n; r += blockDim.x) {
      const int32_t row = srow[beg + r];
      float2 v = gh[row];                              // written by this thread above
      v = make_float2(__double2float_rn(B2_DM((double)v.x, norm)), __double2float_rn(B2_DM((double)v.y, norm)));
      if (!(fabsf(v.x) <= FLT_MAX && fabsf(v.y) <= FLT_MAX)) { bad = true; v = make_float2(0.0f, 0.0f); }
      gh[row] = v;
      mg = fmaxf(mg, fabsf(v.x)); mh = fmaxf(mh, fabsf(v.y));
    }
  }
  if (bad && err) atomicOr(err, 1u);
  if (absmax) absmax_publish(mg, mh, absmax);
}

// metric ids (engine.cu): 16 ndcg, 17 map, 18 pre; k = 0 means the whole group; minus: the score of a group without a
// relevant row (IDCG = 0 / no label != 0) is 0 instead of 1.  One thread per group, positions ascending, binary64.
__global__ void rank_metric_kernel(int metric, int k, int minus, int exp_gain, const int64_t* __restrict__ gptr,
                                   int64_t n_groups, const int32_t* __restrict__ prow, const float* __restrict__ label,
                                   const uint32_t* __restrict__ lkeys, const double* __restrict__ disc,
                                   double* __restrict__ vals) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = gptr[g], n = gptr[g + 1] - b, kk = k > 0 ? k : n, t_end = n < kk ? n : kk;
    double v;
    if (metric == 16) {
      double dcg = 0.0, idcg = 0.0;
      for (int64_t t = 0; t < t_end; ++t) {
        dcg = B2_DA(dcg, B2_DM(rank_gain(label[prow[b + t]], exp_gain), disc[t]));
        idcg = B2_DA(idcg, B2_DM(rank_gain(rank_key_value(lkeys[b + t]), exp_gain), disc[t]));
      }
      v = idcg == 0.0 ? (minus ? 0.0 : 1.0) : B2_DD(dcg, idcg);
    } else if (metric == 17) {
      int64_t rel = 0;
      for (int64_t t = 0; t < n; ++t) rel += label[b + t] != 0.0f;
      if (rel == 0) {
        v = minus ? 0.0 : 1.0;
      } else {
        double ap = 0.0;
        int64_t hits = 0;
        for (int64_t t = 0; t < t_end; ++t)
          if (label[prow[b + t]] != 0.0f) { ++hits; ap = B2_DA(ap, B2_DD((double)hits, (double)(t + 1))); }
        v = B2_DD(ap, (double)rel);
      }
    } else {
      int64_t hits = 0;
      for (int64_t t = 0; t < t_end; ++t) hits += label[prow[b + t]] != 0.0f;
      v = B2_DD((double)hits, (double)kk);
    }
    vals[g] = v;
  }
}

// out[0] = sum of vals in a fixed order (strided per-thread sums, then a fixed tree), out[1] = n: the same bits on
// every call (no atomics on the value)
__global__ void __launch_bounds__(256) rank_sum_kernel(const double* __restrict__ vals, int64_t n, double* __restrict__ out) {
  __shared__ double s[256];
  double a = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += 256) a += vals[i];
  s[threadIdx.x] = a;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) { out[0] = s[0]; out[1] = (double)n; }
}

}  // namespace b2

static inline int rank_grid(int64_t n, int threads, int num_sms) {
  int64_t g = (n + threads - 1) / threads;
  const int64_t cap = (int64_t)num_sms * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

extern "C" {
int b2_rank_stage_rows() { return b2::kRankStageRows; }

// scratch bytes of b2_rank_order for n rows in n_groups groups
size_t b2_rank_order_temp_bytes(int64_t n, int64_t n_groups) {
  size_t bytes = 0;
  cub::DeviceSegmentedSort::StableSortPairs(nullptr, bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                            (const int32_t*)nullptr, (int32_t*)nullptr, (int)(n < 1 ? 1 : n),
                                            (int)(n_groups < 1 ? 1 : n_groups), (const int64_t*)nullptr,
                                            (const int64_t*)nullptr);
  return bytes;
}
int b2_launch_rank_iota(int32_t* idx, int64_t n, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::rank_iota_kernel<<<rank_grid(n, 256, num_sms), 256, 0, s>>>(idx, n);
  return (int)cudaGetLastError();
}
// per group, the rows in descending order of v (stable): keys_out[p] = key of the p-th row, rows_out[p] = its row index.
// iota = 0..n-1 (b2_launch_rank_iota), keys = scratch [n]
int b2_rank_order(const float* v, int64_t n, const int64_t* gptr, int64_t n_groups, const int32_t* iota, uint32_t* keys,
                  uint32_t* keys_out, int32_t* rows_out, void* temp, size_t temp_bytes, int num_sms, cudaStream_t s) {
  if (n <= 0 || n_groups <= 0) return 0;
  b2::rank_keys_kernel<<<rank_grid(n, 256, num_sms), 256, 0, s>>>(v, n, keys);
  size_t tb = temp_bytes;
  cudaError_t e = cub::DeviceSegmentedSort::StableSortPairs(temp, tb, keys, keys_out, iota, rows_out, (int)n, (int)n_groups,
                                                            gptr, gptr + 1, s);
  if (e != cudaSuccess) return (int)e;
  return (int)cudaGetLastError();
}
int b2_launch_rank_disc(double* disc, int64_t len, int num_sms, cudaStream_t s) {
  if (len <= 0) return 0;
  b2::rank_disc_kernel<<<rank_grid(len, 256, num_sms), 256, 0, s>>>(disc, len);
  return (int)cudaGetLastError();
}
int b2_launch_rank_inv_idcg(const int64_t* gptr, int64_t n_groups, const uint32_t* lkeys, const double* disc, int k,
                            int exp_gain, double* inv_idcg, int num_sms, cudaStream_t s) {
  if (n_groups <= 0) return 0;
  b2::rank_inv_idcg_kernel<<<rank_grid(n_groups, 128, num_sms), 128, 0, s>>>(gptr, n_groups, lkeys, disc, k, exp_gain, inv_idcg);
  return (int)cudaGetLastError();
}
int b2_launch_rank_label_check(const float* label, int64_t n, int exp_gain, uint32_t* bad, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::rank_label_check_kernel<<<rank_grid(n, 256, num_sms), 256, 0, s>>>(label, n, exp_gain, bad);
  return (int)cudaGetLastError();
}
// max_group: the largest group (sizes the shared-memory stage); scratch_*: [n] when max_group > b2_rank_stage_rows()
int b2_launch_lambdarank_gradient(int ndcg, const int64_t* gptr, int64_t n_groups, int64_t max_group, const uint32_t* skeys,
                                  const int32_t* srow, const float* label, const double* inv_idcg, const double* disc, int k,
                                  int exp_gain, float* scratch_m, float* scratch_y, double* scratch_p, float2* gh,
                                  uint32_t* absmax, uint32_t* err, int num_sms, cudaStream_t s) {
  if (n_groups <= 0) return 0;
  const int grid = (int)(n_groups < (int64_t)num_sms * 16 ? n_groups : (int64_t)num_sms * 16);
  // the stage holds the largest group (up to kRankStageRows rows: at most 32 KB, no opt-in to large shared memory)
  const int stage = (int)(max_group < b2::kRankStageRows ? (max_group < 1 ? 1 : max_group) : b2::kRankStageRows);
  const size_t smem = (size_t)stage * (8 + 4 + 4);
  if (ndcg)
    b2::lambdarank_gradient_kernel<true><<<grid, b2::kRankThreads, smem, s>>>(gptr, n_groups, skeys, srow, label, inv_idcg, disc, k,
                                                                            exp_gain, stage, scratch_m, scratch_y, scratch_p, gh,
                                                                            absmax, err);
  else
    b2::lambdarank_gradient_kernel<false><<<grid, b2::kRankThreads, smem, s>>>(gptr, n_groups, skeys, srow, label, inv_idcg, disc, k,
                                                                             exp_gain, stage, scratch_m, scratch_y, scratch_p, gh,
                                                                             absmax, err);
  return (int)cudaGetLastError();
}
// per-group metric values into vals [n_groups], then out[0] = their sum, out[1] = n_groups
int b2_launch_rank_metric(int metric, int k, int minus, int exp_gain, const int64_t* gptr, int64_t n_groups, const int32_t* prow,
                          const float* label, const uint32_t* lkeys, const double* disc, double* vals, double* out, int num_sms,
                          cudaStream_t s) {
  if (n_groups <= 0) return (int)cudaMemsetAsync(out, 0, 2 * sizeof(double), s);
  b2::rank_metric_kernel<<<rank_grid(n_groups, 128, num_sms), 128, 0, s>>>(metric, k, minus, exp_gain, gptr, n_groups, prow, label,
                                                                          lkeys, disc, vals);
  b2::rank_sum_kernel<<<1, 256, 0, s>>>(vals, n_groups, out);
  return (int)cudaGetLastError();
}
}
