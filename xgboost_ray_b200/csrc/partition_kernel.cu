// partition_kernel.cu -- row partition (UpdatePosition), leaf sums and prediction-cache update.
//
// Replaces XGBoost's ApplySplit/UpdatePosition and UpdatePredictionCache stages reached through
// xgb.train() (xgboost_ray/main.py:745-752; SURVEY.md 8a rows a13, a14; Appendix A.8/A.9).
// Rows of a node live in a contiguous segment of a row-index list; a split rewrites the segment
// as [left rows | right rows] into the other (ping-pong) list.  Histogram sums are exact integers,
// so the order of rows inside a child segment is irrelevant to the model.
#include <stdlib.h>

#include "common.cuh"
#include "level_finalize.cuh"

namespace b2 {

constexpr int kPartThreads = 256;
constexpr int kPartChunk = 2048;  // rows per CTA work item

typedef B2SegWork SegWork;

// kCat = false: the matrix has no categorical feature; the row loop is then straight-line code whose 8 row-id loads
// and 8 bin-byte loads the compiler batches (48 registers).  With the category test in the body it software-pipelines
// only 2-3 deep, so numeric matrices keep their own
// instantiation.
// kMode 0: numeric only.  1: category set in shared memory.
constexpr int kSplitChunk = 8192;                       // rows per work item of the split-node kernels (partition, final assign)
constexpr int kSplitPasses = kSplitChunk / kPartChunk;  // a work item is processed as 4 register passes of 2048 rows

// One work item = 8192 consecutive rows of one split node.  The rows go through registers in 4 passes of 2048 (8 per
// thread: 8 row-id loads and 8 bin-byte loads in flight); row id + left flag are parked in shared memory, ONE 64-bit
// atomic claims the output ranges of the whole item, then the rows are written out.  Claiming per 2048 rows would put
// the counters of all nodes of a shallow level in one cache line and serialise the atomics of thousands of chunks in
// one L2 slice, a fixed cost per level however little data it moved.
template <int kMode, bool kRoot>
__global__ void __launch_bounds__(kPartThreads)
partition_kernel(const uint8_t* __restrict__ bins_col, int64_t col_stride, const int32_t* __restrict__ ridx_in,
                 int32_t* __restrict__ ridx_out, const B2SplitWork* __restrict__ work, const B2LevelCtl* __restrict__ ctl,
                 int32_t* counters /* [2*n_work]: low word lefts, high word rows claimed */, B2FinalizeArgs fin) {
  const int n_work = ctl->n_split, total_chunks = ctl->part_chunks;
  constexpr int kIters = kPartChunk / kPartThreads;                  // 8 rows per thread and pass
  constexpr int kWarps = kPartThreads / 32;
  constexpr int kCounts = kSplitPasses * kIters * kWarps;            // 256 per-warp left counts of a work item
  __shared__ uint32_t s_rid[kSplitChunk];                            // bit 31 = row goes left
  __shared__ int s_cnt[kCounts];                                     // index = (pass * kIters + it) * kWarps + warp (row order)
  __shared__ int s_base_left, s_base_right;
  __shared__ uint32_t s_cat[8];   // category set of the item's split (all zero for a numeric split)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int chunk = blockIdx.x; chunk < total_chunks; chunk += gridDim.x) {
    int lo = 0, hi = n_work - 1;
    while (lo < hi) {
      int mid = (lo + hi + 1) >> 1;
      if (__ldg(&work[mid].chunk_begin) <= chunk) lo = mid; else hi = mid - 1;
    }
    const B2SplitWork w = work[lo];
    const int row0 = (chunk - w.chunk_begin) * kSplitChunk;
    const int nrows = min(kSplitChunk, w.seg_count - row0);
    constexpr bool kCat = kMode != 0;
    if (kMode == 1) {
      if (threadIdx.x < 8) s_cat[threadIdx.x] = w.is_cat ? __ldg(&work[lo].cat_bits[threadIdx.x]) : 0u;
      __syncthreads();
    }
    const bool is_cat = kCat && w.is_cat != 0, has_missing = w.has_missing != 0, default_left = w.default_left != 0;
#pragma unroll 1
    for (int pass = 0; pass < kSplitPasses; ++pass) {
      const int pbase = pass * kPartChunk;
      if (pbase >= nrows) {   // nothing left in this item (uniform): its counts are zero
        if (threadIdx.x < kIters * kWarps) s_cnt[pass * kIters * kWarps + threadIdx.x] = 0;
        continue;
      }
      // two straight-line batches -- 8 row-id loads, then 8 bin-byte loads -- so that all of them are in flight together
      // (any branch between them, e.g. a test for the root's identity list, makes ptxas issue them as 8 dependent pairs)
      int rid[kIters]; bool left[kIters]; int bin[kIters];
      const int32_t* rsrc = kRoot ? nullptr : ridx_in + w.seg_begin + row0 + pbase + threadIdx.x;
#pragma unroll
      for (int it = 0; it < kIters; ++it) {
        const int r = pbase + it * kPartThreads + threadIdx.x;
        rid[it] = kRoot ? (r < nrows ? w.seg_begin + row0 + r : 0) : (r < nrows ? __ldg(rsrc + it * kPartThreads) : 0);
      }
      const uint8_t* col = bins_col + (int64_t)w.feature * col_stride;
#pragma unroll
      for (int it = 0; it < kIters; ++it) bin[it] = (int)__ldg(col + rid[it]);   // row 0 for lanes past the end: harmless
#pragma unroll
      for (int it = 0; it < kIters; ++it) {
        const int r = pbase + it * kPartThreads + threadIdx.x;
        const bool valid = r < nrows;
        const int b = bin[it];
        bool l;
        if (kCat) {
          const uint32_t word = s_cat[b >> 5];
          const bool in_set = ((word >> (b & 31)) & 1u) != 0u;                     // category in the set -> right
          const bool go_left = is_cat ? !in_set : (b <= w.split_bin);
          l = (has_missing && b == B2_MISSING_BIN) ? default_left : go_left;
        } else {
          l = (w.has_missing && b == B2_MISSING_BIN) ? (w.default_left != 0) : (b <= w.split_bin);
        }
        left[it] = valid && l;
      }
#pragma unroll
      for (int it = 0; it < kIters; ++it) {
        const unsigned bal = __ballot_sync(0xffffffffu, left[it]);
        if (lane == 0) s_cnt[(pass * kIters + it) * kWarps + warp] = __popc(bal);
        s_rid[pbase + it * kPartThreads + threadIdx.x] = (uint32_t)rid[it] | (left[it] ? 0x80000000u : 0u);
      }
    }
    __syncthreads();
    // exclusive prefix of the 256 counts in row order (warp 0: 8 consecutive counts per lane), then one atomic
    if (warp == 0) {
      int c[kCounts / 32], sum = 0;
#pragma unroll
      for (int k = 0; k < kCounts / 32; ++k) { c[k] = s_cnt[lane * (kCounts / 32) + k]; sum += c[k]; }
      int incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
      int run = incl - sum;
#pragma unroll
      for (int k = 0; k < kCounts / 32; ++k) { s_cnt[lane * (kCounts / 32) + k] = run; run += c[k]; }
      if (lane == 31) {
        // low word = left rows so far (what finalize_level reads as the left child's size), high word = rows so far
        const unsigned long long old = atomicAdd(reinterpret_cast<unsigned long long*>(counters + 2 * lo),
                                                 ((unsigned long long)(unsigned)nrows << 32) | (unsigned long long)(unsigned)incl);
        s_base_left = (int)(unsigned)(old & 0xffffffffull);
        s_base_right = (int)(unsigned)(old >> 32) - s_base_left;
      }
    }
    __syncthreads();
    const int base_l = s_base_left, base_r = s_base_right;
#pragma unroll 1
    for (int pass = 0; pass < kSplitPasses; ++pass) {
      const int pbase = pass * kPartChunk;
      if (pbase >= nrows) break;
#pragma unroll
      for (int it = 0; it < kIters; ++it) {
        const int r = pbase + it * kPartThreads + threadIdx.x;
        const uint32_t v = s_rid[r];
        const bool l = (v & 0x80000000u) != 0u;
        const unsigned bal = __ballot_sync(0xffffffffu, l);
        if (r < nrows) {
          const int lrank = s_cnt[(pass * kIters + it) * kWarps + warp] + __popc(bal & ((1u << lane) - 1u));
          if (l) ridx_out[w.seg_begin + base_l + lrank] = (int32_t)(v & 0x7fffffffu);
          else {
            const int rrank = r - lrank;  // rights before this row inside the item
            ridx_out[w.seg_begin + w.seg_count - 1 - (base_r + rrank)] = (int32_t)v;
          }
        }
      }
    }
    __syncthreads();
  }
  // The last CTA to finish finalises the level (no separate single-CTA launch).  Its counter resets itself, so the
  // next level and every replay of the captured tree start from zero.
  __shared__ FinalizeScratch<kPartThreads> s_fin;
  __shared__ bool s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();   // this CTA's counter atomics and row-id stores before its arrival
    const unsigned prev = atomicAdd(fin.done, 1u);
    s_last = prev == gridDim.x - 1;
    if (s_last) { __threadfence(); *fin.done = 0u; }
  }
  __syncthreads();
  if (!s_last) return;
  finalize_level_block<kPartThreads>(s_fin, ctl, work, counters, fin);
}

// ---- leaf refinement: 40-bit fixed-point sums of the fp32 gradients per leaf (exact int64)
// sums == nullptr: only record the leaf index of every row (pos); leaf_accumulate_kernel sums the leaves afterwards.
__global__ void __launch_bounds__(256)
leaf_sums_kernel(const float2* __restrict__ gh, const int32_t* __restrict__ ridx0, const int32_t* __restrict__ ridx1,
                 const SegWork* __restrict__ work, const B2LevelCtl* __restrict__ ctl, const int32_t* __restrict__ qexp,
                 int leaf_bits, long long* __restrict__ sums /* nullable: [n_leaves][2] */,
                 uint16_t* __restrict__ pos /* nullable: row -> leaf index, read by margin_update_kernel */) {
  const int n_work = ctl->hist_n_work, total_chunks = ctl->hist_total_chunks;
  __shared__ long long sg[8], sh[8];
  const double kg = ldexp(1.0, leaf_bits - qexp[0]), kh = ldexp(1.0, leaf_bits - qexp[1]);
  for (int chunk = blockIdx.x; chunk < total_chunks; chunk += gridDim.x) {
    int lo = 0, hi = n_work - 1;
    while (lo < hi) {
      int mid = (lo + hi + 1) >> 1;
      if (__ldg(&work[mid].chunk_begin) <= chunk) lo = mid; else hi = mid - 1;
    }
    const SegWork w = work[lo];
    const int32_t* ridx = w.pad0 ? nullptr : (w.buf ? ridx1 : ridx0);   // pad0: the leaf is the root (rows = identity)
    const int row0 = (chunk - w.chunk_begin) * kPartChunk;
    const int nrows = min(kPartChunk, w.seg_count - row0);
    if (!sums) {   // uniform
      for (int r = threadIdx.x; r < nrows; r += blockDim.x)
        pos[ridx ? __ldg(ridx + w.seg_begin + row0 + r) : (w.seg_begin + row0 + r)] = (uint16_t)w.id;
      continue;
    }
    long long ag = 0, ah = 0;
    for (int r = threadIdx.x; r < nrows; r += blockDim.x) {
      const int row = ridx ? __ldg(ridx + w.seg_begin + row0 + r) : (w.seg_begin + row0 + r);
      if (pos) pos[row] = (uint16_t)w.id;
      const float2 v = __ldg(gh + row);
      ag += __double2ll_rn(__dmul_rn((double)v.x, kg));
      ah += __double2ll_rn(__dmul_rn((double)v.y, kh));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { ag += __shfl_xor_sync(0xffffffffu, ag, o); ah += __shfl_xor_sync(0xffffffffu, ah, o); }
    if ((threadIdx.x & 31) == 0) { sg[threadIdx.x >> 5] = ag; sh[threadIdx.x >> 5] = ah; }
    __syncthreads();
    if (threadIdx.x == 0) {
      long long tg = 0, th = 0;
      for (int i = 0; i < 8; ++i) { tg += sg[i]; th += sh[i]; }
      atomicAdd((unsigned long long*)&sums[2 * w.id], (unsigned long long)tg);
      atomicAdd((unsigned long long*)&sums[2 * w.id + 1], (unsigned long long)th);
    }
    __syncthreads();
  }
}

// margin[row*K + k] += leaf_value[leaf]
__global__ void __launch_bounds__(256)
pred_update_kernel(float* __restrict__ margin, int K, int k, const int32_t* __restrict__ ridx0,
                   const int32_t* __restrict__ ridx1, const SegWork* __restrict__ work, const B2LevelCtl* __restrict__ ctl,
                   const float* __restrict__ leaf_value) {
  const int n_work = ctl->hist_n_work, total_chunks = ctl->hist_total_chunks;
  for (int chunk = blockIdx.x; chunk < total_chunks; chunk += gridDim.x) {
    int lo = 0, hi = n_work - 1;
    while (lo < hi) {
      int mid = (lo + hi + 1) >> 1;
      if (__ldg(&work[mid].chunk_begin) <= chunk) lo = mid; else hi = mid - 1;
    }
    const SegWork w = work[lo];
    const int32_t* ridx = w.pad0 ? nullptr : (w.buf ? ridx1 : ridx0);
    const int row0 = (chunk - w.chunk_begin) * kPartChunk;
    const int nrows = min(kPartChunk, w.seg_count - row0);
    const float v = __ldg(leaf_value + w.id);
    for (int r = threadIdx.x; r < nrows; r += blockDim.x) {
      const int64_t row = ridx ? __ldg(ridx + w.seg_begin + row0 + r) : (w.seg_begin + row0 + r);
      margin[row * K + k] += v;
    }
  }
}

// ---- last split level (d = max_depth - 1): the children are leaves, so their rows need no ordered index list any
// more.  Instead of partition -> finalize -> leaf_sums -> pred_update (three scattered passes over all rows) one pass
// decides left/right, adds the row's fp32 gradient pair to the 40-bit fixed-point sums of the child LEAF and records
// the leaf index of the row; the margin is then updated by a streaming kernel (margin_update_kernel).
// Leaf index of child `side` of split j: leaf_base + 2 j + side -- exactly the index decide_kernel gives the node at
// the next level (leaves are numbered in node order; leaf_base = leaves that existed before this level's children).
// kSums = false (the default whenever the per-leaf accumulators fit in shared memory): only pos is written, and
// leaf_accumulate_kernel sums the gradient pairs afterwards in row order.  Gathering gh[rid] here costs a 32-byte
// sector per 8-byte pair at the last level, where a node's rows are spread over the whole matrix.
template <bool kCat, bool kRoot, bool kSums>
__global__ void __launch_bounds__(kPartThreads)
final_assign_kernel(const uint8_t* __restrict__ bins_col, int64_t col_stride, const int32_t* __restrict__ ridx_in,
                    const B2SplitWork* __restrict__ work, const B2LevelCtl* __restrict__ ctl, const float2* __restrict__ gh,
                    const int32_t* __restrict__ qexp, int leaf_bits, long long* __restrict__ sums,
                    uint16_t* __restrict__ pos) {
  const int n_work = ctl->n_split, total_chunks = ctl->part_chunks, leaf_base = ctl->leaf_base_next;
  __shared__ long long s_acc[kPartThreads / 32][4];
  const double kg = kSums ? ldexp(1.0, leaf_bits - qexp[0]) : 0.0, kh = kSums ? ldexp(1.0, leaf_bits - qexp[1]) : 0.0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int chunk = blockIdx.x; chunk < total_chunks; chunk += gridDim.x) {
    int lo = 0, hi = n_work - 1;
    while (lo < hi) {
      int mid = (lo + hi + 1) >> 1;
      if (__ldg(&work[mid].chunk_begin) <= chunk) lo = mid; else hi = mid - 1;
    }
    const B2SplitWork w = work[lo];
    const int row0 = (chunk - w.chunk_begin) * kSplitChunk;
    const int nrows = min(kSplitChunk, w.seg_count - row0);
    const bool is_cat = kCat && w.is_cat != 0;
    const int leaf_l = leaf_base + 2 * lo;
    long long lg = 0, lh = 0, rg = 0, rh = 0;
    // batches of 4 rows per thread: 4 row-id loads, then 4 bin bytes + 4 gradient pairs, all in flight together
    // (8 rows when no gradient pair is loaded).  Row ids and bin bytes are streamed with the evict-first hint (__ldcs), so that L2
    // keeps the partly written 32-byte sectors of pos until their other rows have been stored
    constexpr int kBatch = kSums ? 4 : 8;
    const uint8_t* col = bins_col + (int64_t)w.feature * col_stride;
    for (int r0 = threadIdx.x; r0 < nrows; r0 += kBatch * kPartThreads) {
      int rid[kBatch]; int bin[kBatch]; float2 v[kBatch];
#pragma unroll
      for (int k = 0; k < kBatch; ++k) {
        const int r = r0 + k * kPartThreads;
        rid[k] = r < nrows ? (kRoot ? w.seg_begin + row0 + r : __ldcs(ridx_in + w.seg_begin + row0 + r)) : -1;
      }
#pragma unroll
      for (int k = 0; k < kBatch; ++k) {
        bin[k] = (int)__ldcs(col + (rid[k] < 0 ? 0 : rid[k]));
        if (kSums) v[k] = __ldg(gh + (rid[k] < 0 ? 0 : rid[k]));
      }
#pragma unroll
      for (int k = 0; k < kBatch; ++k) {
        if (rid[k] < 0) continue;
        const int b = bin[k];
        bool go_left = b <= w.split_bin;
        if (kCat && is_cat) go_left = ((__ldg(&work[lo].cat_bits[b >> 5]) >> (b & 31)) & 1u) == 0u;   // category in the set -> right
        const bool l = (w.has_missing && b == B2_MISSING_BIN) ? (w.default_left != 0) : go_left;
        if (kSums) {
          const long long qg = __double2ll_rn(__dmul_rn((double)v[k].x, kg)), qh = __double2ll_rn(__dmul_rn((double)v[k].y, kh));
          if (l) { lg += qg; lh += qh; } else { rg += qg; rh += qh; }
        }
        pos[rid[k]] = (uint16_t)(leaf_l + (l ? 0 : 1));
      }
    }
    if (!kSums) continue;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lg += __shfl_xor_sync(0xffffffffu, lg, o); lh += __shfl_xor_sync(0xffffffffu, lh, o);
      rg += __shfl_xor_sync(0xffffffffu, rg, o); rh += __shfl_xor_sync(0xffffffffu, rh, o);
    }
    if (lane == 0) { s_acc[warp][0] = lg; s_acc[warp][1] = lh; s_acc[warp][2] = rg; s_acc[warp][3] = rh; }
    __syncthreads();
    if (threadIdx.x < 4) {
      long long t = 0;
      for (int i = 0; i < kPartThreads / 32; ++i) t += s_acc[i][threadIdx.x];
      atomicAdd((unsigned long long*)&sums[2 * leaf_l + threadIdx.x], (unsigned long long)t);   // [leaf_l][g,h], [leaf_l+1][g,h]
    }
    __syncthreads();
  }
}

// margin[row*K + k] += leaf_value[pos[row]] -- streaming, rows in natural order
__global__ void __launch_bounds__(256)
margin_update_kernel(float* __restrict__ margin, int K, int k, const uint16_t* __restrict__ pos,
                     const float* __restrict__ leaf_value, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    margin[i * K + k] += __ldg(leaf_value + pos[i]);
}

// ---- leaf sums in natural row order: sums[pos[i]] += fixed(gh[i]).  pos and gh stream (10 bytes per row) instead of
// being gathered per leaf.  The values are the same 40-bit fixed-point integers leaf_sums_kernel / final_assign_kernel
// add, so the sums are bit-identical in any order.
// Every CTA keeps its sums in shared memory as two 32-bit words per int64 and adds with native 32-bit shared atomics:
// the carry out of the low word is known from the value the atomic returns, so low += lo; high += hi + carry is exact
// modulo 2^64, like an int64 add.  (A 64-bit shared atomic is a compare-and-swap loop on sm_90, and lanes of a warp
// that hit the same popular leaf retry one after another.)  Lanes spread over `copies` copies of the table
// (lane % copies), so that a popular leaf is not one shared-memory word for the whole warp.  At the end the copies are
// added up and every non-empty leaf costs one global atomic per CTA.
constexpr int kLeafAccThreads = 512;
constexpr int kLeafAccMaxDepth = 11;            // 2^11 leaves x 16 bytes = 32 KB of shared memory per CTA
constexpr int kLeafAccSmem = 32 * 1024;         // copies of the table: as many as fit here, at most 8
__device__ __forceinline__ void acc_add64(uint32_t* lo, uint32_t* hi, long long q) {
  const uint32_t l = (uint32_t)(unsigned long long)q, h = (uint32_t)((unsigned long long)q >> 32);
  const uint32_t old = atomicAdd(lo, l);
  const uint32_t hadd = h + ((uint32_t)(old + l) < old ? 1u : 0u);
  if (hadd != 0u) atomicAdd(hi, hadd);
}
__global__ void __launch_bounds__(kLeafAccThreads)
leaf_accumulate_kernel(const float2* __restrict__ gh, const uint16_t* __restrict__ pos, int64_t n, int n_acc, int log2_copies,
                       const int32_t* __restrict__ qexp, int leaf_bits, long long* __restrict__ sums /* [n_leaves][2] */) {
  extern __shared__ uint32_t s_acc[];   // 4 planes (g lo, g hi, h lo, h hi) of [n_acc][copies]
  const int copies = 1 << log2_copies, plane = n_acc << log2_copies;
  for (int i = threadIdx.x; i < 4 * plane; i += blockDim.x) s_acc[i] = 0u;
  __syncthreads();
  uint32_t *glo = s_acc, *ghi = s_acc + plane, *hlo = s_acc + 2 * plane, *hhi = s_acc + 3 * plane;
  const int copy = threadIdx.x & (copies - 1);
  const double kg = ldexp(1.0, leaf_bits - qexp[0]), kh = ldexp(1.0, leaf_bits - qexp[1]);
  constexpr int kBatch = 4;   // 4 leaf indices + 4 gradient pairs in flight per thread
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + (kBatch - 1) * stride < n; i += kBatch * stride) {
    int leaf[kBatch]; float2 v[kBatch];
#pragma unroll
    for (int b = 0; b < kBatch; ++b) { leaf[b] = pos[i + b * stride]; v[b] = __ldg(gh + i + b * stride); }
#pragma unroll
    for (int b = 0; b < kBatch; ++b) {
      const int a = (leaf[b] << log2_copies) + copy;
      acc_add64(glo + a, ghi + a, __double2ll_rn(__dmul_rn((double)v[b].x, kg)));
      acc_add64(hlo + a, hhi + a, __double2ll_rn(__dmul_rn((double)v[b].y, kh)));
    }
  }
  for (; i < n; i += stride) {
    const int a = ((int)pos[i] << log2_copies) + copy;
    const float2 v = __ldg(gh + i);
    acc_add64(glo + a, ghi + a, __double2ll_rn(__dmul_rn((double)v.x, kg)));
    acc_add64(hlo + a, hhi + a, __double2ll_rn(__dmul_rn((double)v.y, kh)));
  }
  __syncthreads();
  for (int j = threadIdx.x; j < 2 * n_acc; j += blockDim.x) {   // j = 2 * leaf + (0: g, 1: h)
    const uint32_t* lo = (j & 1) ? hlo : glo;
    const uint32_t* hi = (j & 1) ? hhi : ghi;
    unsigned long long t = 0ull;
    for (int c = 0; c < copies; ++c) {
      const int a = ((j >> 1) << log2_copies) + c;
      t += ((unsigned long long)hi[a] << 32) | (unsigned long long)lo[a];
    }
    if (t != 0ull) atomicAdd((unsigned long long*)&sums[j], t);
  }
}

__global__ void iota_kernel(int32_t* out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = (int32_t)i;
}

}  // namespace b2

extern "C" {
int b2_part_chunk_rows() { return b2::kPartChunk; }     // leaf-segment work items (leaf_sums / pred_update)
int b2_split_chunk_rows() { return b2::kSplitChunk; }   // split-node work items (partition / final_assign)

// partition + finalize of a level: `fin` is what the last CTA writes (level_finalize.cuh)
int b2_launch_partition(const uint8_t* bins_col, int64_t col_stride, const int32_t* ridx_in, int32_t* ridx_out,
                        const B2SplitWork* work, const B2LevelCtl* ctl, int max_chunks, int32_t* counters, int any_categorical,
                        B2FinalizeArgs fin, int num_sms, cudaStream_t stream) {
  if (max_chunks <= 0) max_chunks = 1;   // the last CTA finalises the level, so even an empty level launches one
  int grid = max_chunks < num_sms * 6 ? max_chunks : num_sms * 6;   // 6 CTAs per SM are resident (33 KB of shared memory, 48 registers)
#define B2_PART_LAUNCH(MODE)                                                                                                  \
  do {                                                                                                                        \
    if (ridx_in) b2::partition_kernel<MODE, false><<<grid, b2::kPartThreads, 0, stream>>>(bins_col, col_stride, ridx_in, ridx_out, work, ctl, counters, fin); \
    else b2::partition_kernel<MODE, true><<<grid, b2::kPartThreads, 0, stream>>>(bins_col, col_stride, ridx_in, ridx_out, work, ctl, counters, fin);    \
  } while (0)
  if (any_categorical) B2_PART_LAUNCH(1);
  else B2_PART_LAUNCH(0);
#undef B2_PART_LAUNCH
  return (int)cudaGetLastError();
}
int b2_launch_leaf_sums(const float2* gh, const int32_t* ridx0, const int32_t* ridx1, const void* work, const B2LevelCtl* ctl,
                        int max_chunks, const int32_t* qexp, int leaf_bits, long long* sums, uint16_t* pos, int num_sms,
                        cudaStream_t stream) {
  if (max_chunks <= 0) return 0;
  int grid = max_chunks < num_sms * 8 ? max_chunks : num_sms * 8;
  b2::leaf_sums_kernel<<<grid, 256, 0, stream>>>(gh, ridx0, ridx1, (const b2::SegWork*)work, ctl, qexp, leaf_bits, sums, pos);
  return (int)cudaGetLastError();
}
int b2_launch_final_assign(const uint8_t* bins_col, int64_t col_stride, const int32_t* ridx_in, const B2SplitWork* work,
                           const B2LevelCtl* ctl, int max_chunks, const float2* gh, const int32_t* qexp, int leaf_bits,
                           long long* sums, uint16_t* pos, int any_categorical, int num_sms, cudaStream_t stream) {
  if (max_chunks <= 0) return 0;
  int grid = max_chunks < num_sms * 8 ? max_chunks : num_sms * 8;
  // sums == nullptr: pos only (the leaves are summed by leaf_accumulate_kernel)
#define B2_FA_LAUNCH(CAT, ROOT)                                                                                               \
  do {                                                                                                                        \
    if (sums) b2::final_assign_kernel<CAT, ROOT, true><<<grid, b2::kPartThreads, 0, stream>>>(bins_col, col_stride, ridx_in, work, ctl, gh, qexp, leaf_bits, sums, pos); \
    else b2::final_assign_kernel<CAT, ROOT, false><<<grid, b2::kPartThreads, 0, stream>>>(bins_col, col_stride, ridx_in, work, ctl, gh, qexp, leaf_bits, sums, pos);    \
  } while (0)
  if (any_categorical) { if (ridx_in) B2_FA_LAUNCH(true, false); else B2_FA_LAUNCH(true, true); }
  else { if (ridx_in) B2_FA_LAUNCH(false, false); else B2_FA_LAUNCH(false, true); }
#undef B2_FA_LAUNCH
  return (int)cudaGetLastError();
}
int b2_leaf_acc_max_depth() { return b2::kLeafAccMaxDepth; }
int b2_launch_leaf_accumulate(const float2* gh, const uint16_t* pos, int64_t n, int max_depth, const int32_t* qexp, int leaf_bits,
                              long long* sums, int num_sms, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (max_depth > b2::kLeafAccMaxDepth) return (int)cudaErrorInvalidValue;
  const int n_acc = 1 << max_depth;
  int log2_copies = 0;
  while (log2_copies < 3 && ((size_t)n_acc * 16 << (log2_copies + 1)) <= (size_t)b2::kLeafAccSmem) ++log2_copies;
  const size_t smem = (size_t)n_acc * 16 << log2_copies;
  const int64_t want = (n + b2::kLeafAccThreads - 1) / b2::kLeafAccThreads;
  const int grid = (int)(want < (int64_t)num_sms * 2 ? want : (int64_t)num_sms * 2);
  b2::leaf_accumulate_kernel<<<grid, b2::kLeafAccThreads, smem, stream>>>(gh, pos, n, n_acc, log2_copies, qexp, leaf_bits, sums);
  return (int)cudaGetLastError();
}
int b2_launch_margin_update(float* margin, int K, int k, const uint16_t* pos, const float* leaf_value, int64_t n, int num_sms,
                            cudaStream_t stream) {
  if (n <= 0) return 0;
  int64_t want = (n + 255) / 256;
  int grid = (int)(want < (int64_t)num_sms * 16 ? want : (int64_t)num_sms * 16);
  b2::margin_update_kernel<<<grid, 256, 0, stream>>>(margin, K, k, pos, leaf_value, n);
  return (int)cudaGetLastError();
}
int b2_launch_pred_update(float* margin, int K, int k, const int32_t* ridx0, const int32_t* ridx1, const void* work,
                          const B2LevelCtl* ctl, int max_chunks, const float* leaf_value, int num_sms, cudaStream_t stream) {
  if (max_chunks <= 0) return 0;
  int grid = max_chunks < num_sms * 8 ? max_chunks : num_sms * 8;
  b2::pred_update_kernel<<<grid, 256, 0, stream>>>(margin, K, k, ridx0, ridx1, (const b2::SegWork*)work, ctl, leaf_value);
  return (int)cudaGetLastError();
}
int b2_launch_iota(int32_t* out, int64_t n, cudaStream_t stream) {
  if (n <= 0) return 0;
  int grid = (int)((n + 1023) / 1024);
  if (grid > 4096) grid = 4096;
  b2::iota_kernel<<<grid, 256, 0, stream>>>(out, n);
  return (int)cudaGetLastError();
}
}
