// quantile_kernel.cu -- reg:quantileerror: pinball gradients, the quantile metric, and the leaf refresh that replaces
// every leaf value with a quantile of its rows' residuals (DESIGN.md 2, "Quantile regression").
//
// The refresh is an exact selection.  A residual r = fp32(y - m) becomes an order-preserving 32-bit key; four passes
// narrow the key of each leaf's target order statistics by 8 bits each.  A pass streams (pos, label, margin, hessian) in
// row order and counts the rows of every leaf whose key matches the leaf's prefix so far, per 256-way digit; a
// one-CTA-per-leaf scan then picks the digit where the running count (or fixed-point weight) reaches the target.  Two
// targets per leaf (order statistics j and j+1 of the interpolating rule) share the histogram while their prefixes agree.
// Histograms are int64 sums, so the result depends neither on the row order nor on how rows are split over GPUs: the
// caller sums them over the ranks between the count and the scan.  Every pass reads its sizes (the leaf count) on the
// device, so the sequence is capturable in the per-tree CUDA graph.
#include <cub/block/block_scan.cuh>
#include "common.cuh"
#include "objective_common.cuh"
#include "launch.h"

namespace b2 {

constexpr int kQDigits = 256;
constexpr int kQPasses = 4;
constexpr int kQScanThreads = kQDigits;
constexpr int kQCountThreads = 1024;
constexpr size_t kQSmemMax = 200 * 1024;

// per-leaf selection state, written by the scan of every pass
struct QSel {
  uint32_t prefix[2];      // resolved high bits of the keys of the two targets
  long long rank[2];       // remaining target inside the prefix: a 1-based row count, or fixed-point weight
  long long n;             // rows of the leaf with a nonzero hessian (all ranks); 0 = empty leaf, keeps its Newton value
  double frac;             // interpolation weight between the two order statistics (unweighted rule)
  int by_mass;             // the targets are fixed-point weights (weighted rule)
  int pad;
};

__device__ __forceinline__ uint32_t q_key(float r) {
  const uint32_t u = __float_as_uint(r);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float q_unkey(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
// the residual of a row; -0 becomes +0 so that equal residuals have one key
__device__ __forceinline__ float q_residual(float y, float m) {
  float r = __fadd_rn(y, -m);
  if (r == 0.0f) r = 0.0f;
  return r;
}
// fixed-point weight of a hessian: rint(h * 2^(32 - e)) with max h < 2^e over the tree's rows, so that a leaf's sum
// stays below 2^63 for fewer than 2^31 rows
__device__ __forceinline__ unsigned long long q_mass(float h, double scale) {
  return (unsigned long long)__double2ll_rn(__dmul_rn((double)h, scale));
}

// ---- gradients: d = p_k - y, g = (d >= 0 ? 1 - alpha_k : -alpha_k) * w, h = w.  gh is class-major [K][n].  Finite for
// finite labels and weights (checked before the first round), whatever the margin.
__global__ void __launch_bounds__(256)
gradient_quantile_kernel(int K, const float* __restrict__ alpha, const float* __restrict__ margin,
                         const float* __restrict__ label, const float* __restrict__ weight, int64_t n,
                         float2* __restrict__ gh, uint32_t* __restrict__ absmax) {
  for (int k = 0; k < K; ++k) {
    const float a = alpha[k], up = __fadd_rn(1.0f, -a);
    float mg = 0.0f, mh = 0.0f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
      const float w = weight ? weight[i] : 1.0f;
      const float d = margin ? __fadd_rn(margin[i * K + k], -label[i]) : -label[i];
      const float2 v = make_float2(__fmul_rn(d >= 0.0f ? up : -a, w), w);
      gh[(int64_t)k * n + i] = v;
      mg = fmaxf(mg, fabsf(v.x)); mh = fmaxf(mh, fabsf(v.y));
    }
    if (absmax) absmax_publish(mg, mh, absmax + 2 * k);
  }
}

// ---- the quantile metric: (sum_i w_i sum_k rho_{alpha_k}(y_i - p_ik), K sum_i w_i), rho_a(u) = u (a - [u < 0]), one
// pair per CTA in partial (b2_metric_partial)
__global__ void quantile_metric_kernel(int K, const float* __restrict__ alpha, const float* __restrict__ margin,
                                       const float* __restrict__ label, const float* __restrict__ weight, int64_t n,
                                       double* __restrict__ partial) {
  double s = 0.0, ws = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double w = weight ? (double)weight[i] : 1.0, y = (double)label[i];
    double v = 0.0;
    for (int k = 0; k < K; ++k) {
      const double u = y - (double)margin[i * K + k], a = (double)alpha[k];
      v += u >= 0.0 ? a * u : (a - 1.0) * u;
    }
    s += v * w; ws += w * (double)K;
  }
  b2_metric_partial(s, ws, partial);
}

// ---- count pass.  hist: count[L][2][256] then (weighted) mass[L][2][256], uint64.  Slot 1 holds the second target's
// digits only once its prefix differs from the first's.  With smem, slot 0 of every leaf is accumulated per CTA in
// shared memory (uint32 counts, uint64 masses) and added to the global histogram once; slot 1 matches few rows and
// goes to global memory directly.
__global__ void __launch_bounds__(kQCountThreads)
quantile_count_kernel(int pass, const uint16_t* __restrict__ pos, const float* __restrict__ label,
                      const float* __restrict__ margin, int K, int k, const float2* __restrict__ gh, int64_t n,
                      const int32_t* __restrict__ qexp, int weighted, const QSel* __restrict__ sel, int max_leaves,
                      int use_smem, unsigned long long* __restrict__ hist) {
  extern __shared__ __align__(16) unsigned char q_smem[];
  const int shift = 24 - 8 * pass;
  const size_t L2 = (size_t)max_leaves * 2 * kQDigits;
  unsigned long long* gcount = hist;
  unsigned long long* gmass = hist + L2;
  const double scale = weighted ? ldexp(1.0, 32 - qexp[1]) : 0.0;
  const int slot0_entries = max_leaves * kQDigits;
  uint32_t* scount = reinterpret_cast<uint32_t*>(q_smem);
  unsigned long long* smass = reinterpret_cast<unsigned long long*>(q_smem + (size_t)slot0_entries * 4);
  if (use_smem) {
    for (int i = threadIdx.x; i < slot0_entries; i += blockDim.x) {
      scount[i] = 0u;
      if (weighted) smass[i] = 0ull;
    }
    __syncthreads();
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float h = gh[i].y;
    if (h == 0.0f) continue;
    const int leaf = pos ? (int)pos[i] : 0;
    const uint32_t key = q_key(q_residual(label[i], margin ? margin[i * K + k] : 0.0f));
    const int digit = (int)((key >> shift) & 0xffu);
    bool in0 = true, in1 = false;
    if (pass > 0) {
      const QSel st = sel[leaf];
      if (st.n == 0) continue;
      const uint32_t hi = key >> (shift + 8);
      in0 = hi == (st.prefix[0] >> (shift + 8));
      in1 = st.prefix[0] != st.prefix[1] && hi == (st.prefix[1] >> (shift + 8));
    }
    const unsigned long long ms = weighted ? q_mass(h, scale) : 0ull;
    if (in0) {
      const size_t e = (size_t)leaf * kQDigits + digit;
      if (use_smem) {
        atomicAdd(&scount[e], 1u);
        if (weighted) atomicAdd(&smass[e], ms);
      } else {
        const size_t g = (size_t)leaf * 2 * kQDigits + digit;
        atomicAdd(&gcount[g], 1ull);
        if (weighted) atomicAdd(&gmass[g], ms);
      }
    }
    if (in1) {
      const size_t g = ((size_t)leaf * 2 + 1) * kQDigits + digit;
      atomicAdd(&gcount[g], 1ull);
      if (weighted) atomicAdd(&gmass[g], ms);
    }
  }
  if (use_smem) {
    __syncthreads();
    for (int i = threadIdx.x; i < slot0_entries; i += blockDim.x) {
      const uint32_t c = scount[i];
      if (c == 0u) continue;
      const size_t g = (size_t)(i / kQDigits) * 2 * kQDigits + (i % kQDigits);
      atomicAdd(&gcount[g], (unsigned long long)c);
      if (weighted) atomicAdd(&gmass[g], smass[i]);
    }
  }
}

// ---- scan pass: one CTA per leaf.  Reads (and zeroes, for the next pass) the leaf's digit histograms, picks each
// target's digit, and after the last pass writes the quantile (times eta) as the leaf value.
// First pass: n rows, W fixed-point weight.  Unweighted: alpha <= 1/(n+1) -> min, alpha >= n/(n+1) -> max, else with
// x = alpha (n+1), j = floor(x) - 1, d = (x - 1) - j the order statistics j, j+1 (0-based) and
// q = fp32(v_j + d fp32(v_{j+1} - v_j)).  Weighted: the first row in ascending order whose cumulative weight reaches
// ceil(alpha W) (the minimum when that is 0).
__global__ void __launch_bounds__(kQScanThreads)
quantile_scan_kernel(int pass, const int32_t* __restrict__ n_leaves, int max_leaves, int weighted, float alpha, float eta,
                     unsigned long long* __restrict__ hist, QSel* __restrict__ sel, const B2LeafDev* __restrict__ leaves,
                     float* __restrict__ leaf_value, float* __restrict__ tree_value) {
  using Scan = cub::BlockScan<unsigned long long, kQScanThreads>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ QSel st;
  __shared__ int pick[2];
  __shared__ unsigned long long before[2];
  const int leaf = blockIdx.x;
  if (leaf >= *n_leaves) return;
  const int t = threadIdx.x;
  const int shift = 24 - 8 * pass;
  const size_t L2 = (size_t)max_leaves * 2 * kQDigits;
  unsigned long long* cnt = hist + (size_t)leaf * 2 * kQDigits;
  unsigned long long* mass = hist + L2 + (size_t)leaf * 2 * kQDigits;
  if (t == 0) {
    if (pass == 0) { st.prefix[0] = st.prefix[1] = 0u; st.n = -1; }
    else st = sel[leaf];
  }
  __syncthreads();
  if (st.n == 0) return;
  const bool split = pass > 0 && st.prefix[0] != st.prefix[1];
  unsigned long long c[2], w[2];
  for (int s = 0; s < 2; ++s) {
    const int slot = (s == 1 && split) ? 1 : 0;
    c[s] = cnt[slot * kQDigits + t];
    w[s] = weighted ? mass[slot * kQDigits + t] : 0ull;
  }
  __syncthreads();   // every thread has read its digits before they are zeroed
  cnt[t] = 0ull; cnt[kQDigits + t] = 0ull;
  if (weighted) { mass[t] = 0ull; mass[kQDigits + t] = 0ull; }
  if (pass == 0) {
    unsigned long long tot_c, tot_w = 0ull, ignore;
    Scan(tmp).ExclusiveSum(c[0], ignore, tot_c);
    __syncthreads();
    if (weighted) { Scan(tmp).ExclusiveSum(w[0], ignore, tot_w); __syncthreads(); }
    if (t == 0) {
      const long long nn = (long long)tot_c;
      st.n = nn; st.frac = 0.0; st.by_mass = 0; st.rank[0] = st.rank[1] = 1;
      if (nn > 0) {
        if (weighted) {
          const long long target = (long long)ceil(__dmul_rn((double)alpha, (double)tot_w));
          if (target >= 1) { st.by_mass = 1; st.rank[0] = st.rank[1] = target; }
        } else {
          const double a = (double)alpha, n1 = (double)(nn + 1);
          if (a <= __ddiv_rn(1.0, n1)) {
            st.rank[0] = st.rank[1] = 1;
          } else if (a >= __ddiv_rn((double)nn, n1)) {
            st.rank[0] = st.rank[1] = nn;
          } else {
            const double x = __dmul_rn(a, n1);
            const long long j = (long long)floor(x) - 1;
            st.frac = __dsub_rn(__dsub_rn(x, 1.0), (double)j);
            st.rank[0] = j + 1; st.rank[1] = j + 2;
          }
        }
      }
    }
    __syncthreads();
    if (st.n == 0) { if (t == 0) sel[leaf] = st; return; }
  }
  for (int s = 0; s < 2; ++s) {
    const unsigned long long v = st.by_mass ? w[s] : c[s];
    unsigned long long ex, total;
    Scan(tmp).ExclusiveSum(v, ex, total);
    const unsigned long long target = (unsigned long long)st.rank[s];
    if (ex < target && ex + v >= target) { pick[s] = t; before[s] = ex; }
    __syncthreads();
  }
  if (t == 0) {
    for (int s = 0; s < 2; ++s) {
      st.prefix[s] |= (uint32_t)pick[s] << shift;
      st.rank[s] -= (long long)before[s];
    }
    sel[leaf] = st;
    if (pass == kQPasses - 1) {
      const float v0 = q_unkey(st.prefix[0]), v1 = q_unkey(st.prefix[1]);
      const float q = __double2float_rn(__dadd_rn((double)v0, __dmul_rn(st.frac, (double)__fadd_rn(v1, -v0))));
      const float val = __fmul_rn(q, eta);
      leaf_value[leaf] = val;
      if (tree_value) tree_value[leaves[leaf].nid] = val;
    }
  }
}

}  // namespace b2

static inline int q_grid(int64_t n, int num_sms) {
  int64_t g = (n + 255) / 256;
  const int64_t cap = (int64_t)num_sms * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

extern "C" {
size_t b2_quantile_hist_elems(int max_leaves) { return (size_t)max_leaves * 2 * b2::kQDigits * 2; }
size_t b2_quantile_sel_bytes(int max_leaves) { return (size_t)max_leaves * sizeof(b2::QSel); }

int b2_launch_gradient_quantile(int K, const float* alpha, const float* margin, const float* label, const float* weight,
                                int64_t n, float2* gh, uint32_t* absmax, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  b2::gradient_quantile_kernel<<<q_grid(n, num_sms), 256, 0, s>>>(K, alpha, margin, label, weight, n, gh, absmax);
  return (int)cudaGetLastError();
}

int b2_launch_quantile_metric(int K, const float* alpha, const float* margin, const float* label, const float* weight,
                              int64_t n, double* partial, double* out, int num_sms, cudaStream_t s) {
  if (n <= 0) return 0;
  const int g = q_grid(n, num_sms);
  b2::quantile_metric_kernel<<<g, 256, 0, s>>>(K, alpha, margin, label, weight, n, partial);
  return b2_launch_metric_sum(partial, g, out, s);
}

// one pass of the selection: count (hist_reduce, nullable, is called between count and scan to sum the histograms over
// the ranks), then scan.  hist holds b2_quantile_hist_elems(max_leaves) zeroed uint64 on entry and on return.
int b2_launch_quantile_count(int pass, const uint16_t* pos, const float* label, const float* margin, int K, int k,
                             const float2* gh, int64_t n, const int32_t* qexp, int weighted, const void* sel,
                             int max_leaves, unsigned long long* hist, int num_sms, cudaStream_t s) {
  const size_t smem = (size_t)max_leaves * b2::kQDigits * (weighted ? 12 : 4);
  const int use_smem = smem <= b2::kQSmemMax ? 1 : 0;
  int grid;
  if (use_smem) {
    static bool attr_set = false;
    if (!attr_set) {
      cudaError_t e = cudaFuncSetAttribute(b2::quantile_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)b2::kQSmemMax);
      if (e != cudaSuccess) return (int)e;
      attr_set = true;
    }
    const int64_t want = (n + b2::kQCountThreads * 8 - 1) / (b2::kQCountThreads * 8);
    grid = (int)(want < 1 ? 1 : (want > num_sms ? num_sms : want));
  } else {
    const int64_t want = (n + b2::kQCountThreads - 1) / b2::kQCountThreads;
    grid = (int)(want < 1 ? 1 : (want > 4 * num_sms ? 4 * num_sms : want));
  }
  if (n <= 0) return 0;
  b2::quantile_count_kernel<<<grid, b2::kQCountThreads, use_smem ? smem : 0, s>>>(
      pass, pos, label, margin, K, k, gh, n, qexp, weighted, reinterpret_cast<const b2::QSel*>(sel), max_leaves, use_smem, hist);
  return (int)cudaGetLastError();
}

int b2_launch_quantile_scan(int pass, const int32_t* n_leaves, int max_leaves, int weighted, float alpha, float eta,
                            unsigned long long* hist, void* sel, const B2LeafDev* leaves, float* leaf_value,
                            float* tree_value, cudaStream_t s) {
  b2::quantile_scan_kernel<<<max_leaves, b2::kQScanThreads, 0, s>>>(pass, n_leaves, max_leaves, weighted, alpha, eta, hist,
                                                                    reinterpret_cast<b2::QSel*>(sel), leaves, leaf_value,
                                                                    tree_value);
  return (int)cudaGetLastError();
}

int b2_quantile_passes() { return b2::kQPasses; }
}
