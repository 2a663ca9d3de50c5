// hist_kernel.cu -- feature x bin gradient/hessian histogram build for sm_90a.
//
// Replaces the BuildHist stage that the reference reaches through xgb.train()
// (xgboost_ray/main.py:745-752; SURVEY.md 8a row a10).  Bandwidth-bound scatter-reduce:
// no tensor cores.  Design (DESIGN.md "Histogram kernel"):
//
//  * A CTA owns ONE feature group (<= 32 features -> 32 "slots") of ONE node at a time and keeps
//    its histogram in shared memory as two int32 planes [256 bins][32 slots] (g and h): 64 KiB, so
//    three CTAs are resident per SM.  Because a bin row is exactly 32 words, the bank of an update
//    is its SLOT and does not depend on the bin value.
//  * A lane loads 16 bin bytes of one row (LDG.128 straight to registers; staging rows through
//    shared memory would spend the shared-memory bandwidth that the atomics are bound by).  Two
//    lanes cover the 32-byte group slice of a row, 16 rows per warp.  Lane l pre-rotates its bytes
//    by (l>>1) so that at step j the 32 lanes of a warp touch 32 DIFFERENT slots: every ATOMS.ADD
//    is bank-conflict free for any data, one wavefront per instruction.
//  * Sums are exact integers (fixed-point gradients), so the result is independent of the order
//    of rows, CTAs and GPUs.  A CTA flushes its planes to the global int64 histogram when it moves
//    to another node; every `window_rows` = 2^(30-qbits) rows it flushes just the cells that reached
//    2^30 (none for well spread bins), which is what keeps the int32 cells from overflowing.
//  * Rows of a node are addressed through the row-index segment list (gather) except at the root.
#include <stdlib.h>

#include "hist_common.cuh"

#ifndef B2_HIST_DEFAULT_VARIANT
#define B2_HIST_DEFAULT_VARIANT 3
#endif

namespace b2 {

// kGPC = feature groups per CTA.  1: 64 KiB of histogram, two lanes per row, 16 rows per warp step.
// 2: 128 KiB (one 1024-thread CTA per SM); FOUR lanes read 64 contiguous bytes of a row (one L1 wavefront
// instead of two) and the row id / gradient pair loads are shared by both groups, which removes about a
// quarter of the L1TEX wavefronts per row.
template <bool kGather, int kThreads, int kMinBlocks, int kGPC>
__global__ void __launch_bounds__(kThreads, kMinBlocks)
hist_build_kernel(const uint8_t* __restrict__ bins, int row_stride, const int2* __restrict__ gpair,
                  const int32_t* __restrict__ ridx, const B2HistWork* __restrict__ work, int n_work,
                  int total_chunks, int chunk_rows, int window_rows, int n_groups, long long* __restrict__ hist,
                  const B2LevelCtl* __restrict__ ctl, int log2_shards, int node_cap, int debug_mode) {
  constexpr int kLanesPerRow = 2 * kGPC;
  constexpr int kRowsPerWarp = 32 / kLanesPerRow;
  HistTarget target; target.base = (unsigned long long*)hist; target.log2_shards = log2_shards; target.node_cap = node_cap;
  target.n_groups = n_groups;
  if (ctl) { n_work = ctl->hist_n_work; total_chunks = ctl->hist_total_chunks; chunk_rows = ctl->hist_chunk_rows; }
  extern __shared__ __align__(16) int32_t s_hist[];  // [kGPC][256][2][32]
  const int n_cta_groups = (n_groups + kGPC - 1) / kGPC;
  const int group0 = (blockIdx.x % n_cta_groups) * kGPC;
  const int stream = blockIdx.x / n_cta_groups;
  const int n_streams = gridDim.x / n_cta_groups;
  if (total_chunks <= 0) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  // lane -> (row of the warp step, group of the CTA, 16-byte half of the group slice).  rot is distinct for the
  // 16 (row, group) pairs of a warp, so at every step the 32 lanes hit 32 different banks (bank = slot).
  const int sub = lane / kLanesPerRow, gsel = (lane % kLanesPerRow) >> 1, half = lane & 1;
  const int rot = sub * kGPC + gsel;
  const bool active = group0 + gsel < n_groups;
  const int lane_byte_off = (group0 + gsel) * 32 + half * 16;
  const uint32_t smem_g = (uint32_t)__cvta_generic_to_shared(s_hist) + gsel * (B2_GROUP_ELEMS * 4);

  for (int e = threadIdx.x; e < kGPC * B2_GROUP_ELEMS; e += blockDim.x) s_hist[e] = 0;
  __syncthreads();

  int cur = -1;          // work index whose partial sums are in shared memory
  int rows_in_window = 0;
  // A stream takes a CONTIGUOUS range of the chunk list, so consecutive chunks of a CTA mostly belong to the same
  // node and the 2 x 16K-cell node flush happens once per node per CTA instead of once per chunk (with the strided
  // assignment of round 1 every chunk of a deep level was a node change: levels 6-7 cost 1.5x the root per row).
  // debug_mode bit 2 (B2_HIST_DEBUG_MODE=4) restores the strided assignment for A/B timing.
  const bool strided = (debug_mode & 4) != 0;
  debug_mode &= 3;
  const int c_begin = strided ? stream : (int)(((long long)stream * total_chunks) / n_streams);
  const int c_end = strided ? total_chunks : (int)(((long long)(stream + 1) * total_chunks) / n_streams);
  const int c_step = strided ? n_streams : 1;
  for (int chunk = c_begin; chunk < c_end; chunk += c_step) {
    // locate the node of this chunk (uniform across the CTA): last w with chunk_begin <= chunk
    int lo = 0, hi = n_work - 1;
    while (lo < hi) {
      int mid = (lo + hi + 1) >> 1;
      if (__ldg(&work[mid].chunk_begin) <= chunk) lo = mid; else hi = mid - 1;
    }
    const int w = lo;
    const int seg_begin = __ldg(&work[w].seg_begin), seg_count = __ldg(&work[w].seg_count);
    const int row0 = (chunk - __ldg(&work[w].chunk_begin)) * chunk_rows;
    const int nrows = min(chunk_rows, seg_count - row0);
    if (cur >= 0 && w != cur) {
      // node change: add the partial sums to the global int64 histogram
      __syncthreads();
#pragma unroll
      for (int gs = 0; gs < kGPC; ++gs)
        if (group0 + gs < n_groups) flush_planes(s_hist + gs * B2_GROUP_ELEMS, target, __ldg(&work[cur].hist_index), group0 + gs);
      __syncthreads();
      rows_in_window = 0;
    } else if (cur >= 0 && rows_in_window + nrows > window_rows) {
      // same node, overflow guard interval reached: flush only the (rare) cells at or above 2^30
      // (flushing all cells with RED.64 every window, or a CTA-private int64 scratch with plain read-modify-write,
      // would move far more data than the few saturated cells)
      __syncthreads();
#pragma unroll
      for (int gs = 0; gs < kGPC; ++gs)
        if (group0 + gs < n_groups) flush_large_cells(s_hist + gs * B2_GROUP_ELEMS, target, __ldg(&work[cur].hist_index), group0 + gs);
      __syncthreads();
      rows_in_window = 0;
    }
    cur = w;
    rows_in_window += nrows;
    const int64_t pos0 = (int64_t)seg_begin + row0;
    const int iter_rows = n_warps * kRowsPerWarp;
    // 3-stage register pipeline: while stage k is accumulated, the loads of the next two
    // iterations are in flight, and (gather) the row ids of three more iterations behind them,
    // so no load waits on the ridx -> bins dependency.
    const int rbase = warp * kRowsPerWarp;
    const int r0 = rbase + sub;
    const int lim = active ? nrows : 0;   // lanes of a group past the last one (odd group count) load nothing
    int64_t id0 = fetch_rid<kGather>(ridx, pos0, r0, lim);
    int64_t id1 = fetch_rid<kGather>(ridx, pos0, r0 + iter_rows, lim);
    int64_t id2 = fetch_rid<kGather>(ridx, pos0, r0 + 2 * iter_rows, lim);
    unsigned sink = 0;
#define B2_LOAD(id) (debug_mode == 2 ? fake_row(id) : load_row_id(bins, gpair, id, row_stride, lane_byte_off))
    RowData s0 = B2_LOAD(id0);
    id0 = fetch_rid<kGather>(ridx, pos0, r0 + 3 * iter_rows, lim);
    RowData s1 = B2_LOAD(id1);
    id1 = fetch_rid<kGather>(ridx, pos0, r0 + 4 * iter_rows, lim);
    RowData s2 = B2_LOAD(id2);
    id2 = fetch_rid<kGather>(ridx, pos0, r0 + 5 * iter_rows, lim);
    for (int r = rbase; r < nrows; r += 3 * iter_rows) {   // warp-uniform trip count
      if (kGPC == 1 || active) accumulate_row(s0, smem_g, rot, half, debug_mode, &sink);
      s0 = B2_LOAD(id0);
      id0 = fetch_rid<kGather>(ridx, pos0, r + sub + 6 * iter_rows, lim);
      if (r + iter_rows < nrows && (kGPC == 1 || active)) accumulate_row(s1, smem_g, rot, half, debug_mode, &sink);
      s1 = B2_LOAD(id1);
      id1 = fetch_rid<kGather>(ridx, pos0, r + sub + 7 * iter_rows, lim);
      if (r + 2 * iter_rows < nrows && (kGPC == 1 || active)) accumulate_row(s2, smem_g, rot, half, debug_mode, &sink);
      s2 = B2_LOAD(id2);
      id2 = fetch_rid<kGather>(ridx, pos0, r + sub + 8 * iter_rows, lim);
    }
#undef B2_LOAD
    if (sink == 0x9e3779b9u) s_hist[threadIdx.x] = (int)sink;
  }
  if (cur >= 0) {
    __syncthreads();
#pragma unroll
    for (int gs = 0; gs < kGPC; ++gs)
      if (group0 + gs < n_groups) flush_planes(s_hist + gs * B2_GROUP_ELEMS, target, __ldg(&work[cur].hist_index), group0 + gs);
  }
}

// ================================================================ v3: group pairs with a narrow last group
// F = 32 a + r features are laid out as `a` full groups plus, when 0 < r <= 16, one NARROW group of w = pow2ceil(r)
// slots (engine.cu setup_groups).  A full group costs 2 shared-atomic wavefronts per row (32 slots x 2 planes / 32
// lanes); the r leftover features used to cost as much as a full group of 32 (F = 100 spent 22 % of its atomics on
// padding slots).  A narrow group keeps 32 / w replicas of its w slots side by side in its 64 KiB plane pair:
// lane l adds to replica l / w and walks the slots rotated by l % w, so one lane handles one ROW and the 32 lanes of
// a warp still hit 32 different banks -- w steps for 32 rows, i.e. w / 16 wavefronts per row.
// A CTA type = one pair of groups; types get CTAs in proportion to their cost (B2HistPlan), every type walks the
// whole chunk list with its own number of streams.

template <int W>
struct NarrowBytes {   // the W bin bytes of one row, rotated so that step j reads byte j
  uint32_t w[W >= 4 ? W / 4 : 1];
};
template <int W>
__device__ __forceinline__ NarrowBytes<W> load_narrow(const uint8_t* __restrict__ p, int rot) {
  NarrowBytes<W> r;
  if constexpr (W == 16) {
    uint4 v = rotate_bytes(ldg_nc_v4(p), rot);
    r.w[0] = v.x; r.w[1] = v.y; r.w[2] = v.z; r.w[3] = v.w;
  } else if constexpr (W == 8) {
    uint2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
    uint32_t a = v.x, b = v.y;
    if (rot & 4) { uint32_t t = a; a = b; b = t; }
    const int bs = (rot & 3) * 8;
    r.w[0] = __funnelshift_r(a, b, bs); r.w[1] = __funnelshift_r(b, a, bs);
  } else if constexpr (W == 4) {
    const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(p));
    r.w[0] = __funnelshift_r(v, v, (rot & 3) * 8);
  } else if constexpr (W == 2) {
    const uint32_t v = __ldg(reinterpret_cast<const uint16_t*>(p));
    r.w[0] = (rot & 1) ? ((v >> 8) | ((v & 0xffu) << 8)) : v;
  } else {
    r.w[0] = __ldg(p);
  }
  return r;
}

// one narrow group, rows [0, nrows) of a chunk: lane = row, W steps
template <bool kGather, int W>
__device__ __forceinline__ void narrow_pass(const uint8_t* __restrict__ bins, int row_stride, const int2* __restrict__ gpair,
                                            const int32_t* __restrict__ ridx, int64_t pos0, int nrows, int byte_off,
                                            uint32_t smem_g, int lane, int warp, int n_warps) {
  const int rot = lane & (W - 1), rep = lane / W;
  const uint32_t base = smem_g + (uint32_t)(rep * W) * 4u;
  // two-stage register pipeline over the warp's rows (warp-uniform trip count)
  int r = warp * 32 + lane;
  int64_t rid = r < nrows ? (kGather ? (int64_t)__ldg(ridx + pos0 + r) : pos0 + r) : -1;
  NarrowBytes<W> cur; int2 gp = make_int2(0, 0);
#pragma unroll
  for (int k = 0; k < (W >= 4 ? W / 4 : 1); ++k) cur.w[k] = 0;
  if (rid >= 0) { cur = load_narrow<W>(bins + rid * row_stride + byte_off, rot); gp = __ldg(gpair + rid); }
  for (int r0 = warp * 32; r0 < nrows; r0 += n_warps * 32) {
    const int rn = r0 + n_warps * 32 + lane;
    const int64_t rid_n = rn < nrows ? (kGather ? (int64_t)__ldg(ridx + pos0 + rn) : pos0 + rn) : -1;
    NarrowBytes<W> nxt; int2 gpn = make_int2(0, 0);
#pragma unroll
    for (int k = 0; k < (W >= 4 ? W / 4 : 1); ++k) nxt.w[k] = 0;
    if (rid_n >= 0) { nxt = load_narrow<W>(bins + rid_n * row_stride + byte_off, rot); gpn = __ldg(gpair + rid_n); }
    if (rid >= 0) {
#pragma unroll
      for (int j = 0; j < W; ++j) {
        const uint32_t bin256 = __byte_perm(cur.w[j >> 2], 0u, 0x4404u | ((uint32_t)(j & 3) << 4));
        const uint32_t a = base + bin256 + (((uint32_t)(j + rot)) & (uint32_t)(W - 1)) * 4u;
        red_shared_add(a, gp.x);
        red_shared_add(a + B2_GROUP_SLOTS * 4, gp.y);
      }
    }
    rid = rid_n; cur = nxt; gp = gpn;
  }
}

// full groups of a CTA, rows [0, nrows) of a chunk: kGPC = 2 -> four lanes cover the 64 contiguous bytes of the pair,
// kGPC = 1 -> two lanes cover the 32 bytes of the single group (the register pipeline of hist_build_kernel)
template <bool kGather, int kGPC, bool kAligned>
__device__ __forceinline__ void full_pass(const uint8_t* __restrict__ bins, int row_stride, const int2* __restrict__ gpair,
                                          const int32_t* __restrict__ ridx, int64_t pos0, int nrows, int group0,
                                          uint32_t smem_base, int lane, int warp, int n_warps) {
  constexpr int kLanesPerRow = 2 * kGPC;
  constexpr int kRowsPerWarp = 32 / kLanesPerRow;
  const int sub = lane / kLanesPerRow, gsel = (lane % kLanesPerRow) >> 1, half = lane & 1;
  const int rot = sub * kGPC + gsel;
  const int lane_byte_off = (group0 + gsel) * 32 + half * 16;
  const uint32_t smem_g = smem_base + gsel * (B2_GROUP_ELEMS * 4);
  const int iter_rows = n_warps * kRowsPerWarp;
  const int rbase = warp * kRowsPerWarp;
  const int r0 = rbase + sub;
  int64_t id0 = fetch_rid<kGather>(ridx, pos0, r0, nrows);
  int64_t id1 = fetch_rid<kGather>(ridx, pos0, r0 + iter_rows, nrows);
  int64_t id2 = fetch_rid<kGather>(ridx, pos0, r0 + 2 * iter_rows, nrows);
  RowData s0 = load_row_id(bins, gpair, id0, row_stride, lane_byte_off);
  id0 = fetch_rid<kGather>(ridx, pos0, r0 + 3 * iter_rows, nrows);
  RowData s1 = load_row_id(bins, gpair, id1, row_stride, lane_byte_off);
  id1 = fetch_rid<kGather>(ridx, pos0, r0 + 4 * iter_rows, nrows);
  RowData s2 = load_row_id(bins, gpair, id2, row_stride, lane_byte_off);
  id2 = fetch_rid<kGather>(ridx, pos0, r0 + 5 * iter_rows, nrows);
#define B2_ACC(S) do { if (kAligned) accumulate_row_aligned(S, smem_g, rot, half); else accumulate_row(S, smem_g, rot, half); } while (0)
  for (int r = rbase; r < nrows; r += 3 * iter_rows) {   // warp-uniform trip count
    B2_ACC(s0);
    s0 = load_row_id(bins, gpair, id0, row_stride, lane_byte_off);
    id0 = fetch_rid<kGather>(ridx, pos0, r + sub + 6 * iter_rows, nrows);
    if (r + iter_rows < nrows) B2_ACC(s1);
    s1 = load_row_id(bins, gpair, id1, row_stride, lane_byte_off);
    id1 = fetch_rid<kGather>(ridx, pos0, r + sub + 7 * iter_rows, nrows);
    if (r + 2 * iter_rows < nrows) B2_ACC(s2);
    s2 = load_row_id(bins, gpair, id2, row_stride, lane_byte_off);
    id2 = fetch_rid<kGather>(ridx, pos0, r + sub + 8 * iter_rows, nrows);
  }
#undef B2_ACC
}

template <bool kGather>
__device__ __forceinline__ void narrow_dispatch(int w, const uint8_t* __restrict__ bins, int row_stride, const int2* __restrict__ gpair,
                                                const int32_t* __restrict__ ridx, int64_t pos0, int nrows, int byte_off,
                                                uint32_t smem_g, int lane, int warp, int n_warps) {
  switch (w) {
    case 16: narrow_pass<kGather, 16>(bins, row_stride, gpair, ridx, pos0, nrows, byte_off, smem_g, lane, warp, n_warps); break;
    case 8: narrow_pass<kGather, 8>(bins, row_stride, gpair, ridx, pos0, nrows, byte_off, smem_g, lane, warp, n_warps); break;
    case 4: narrow_pass<kGather, 4>(bins, row_stride, gpair, ridx, pos0, nrows, byte_off, smem_g, lane, warp, n_warps); break;
    case 2: narrow_pass<kGather, 2>(bins, row_stride, gpair, ridx, pos0, nrows, byte_off, smem_g, lane, warp, n_warps); break;
    default: narrow_pass<kGather, 1>(bins, row_stride, gpair, ridx, pos0, nrows, byte_off, smem_g, lane, warp, n_warps); break;
  }
}

// kAligned: the dynamic shared memory is 64 KiB larger than the two group histograms and the histograms start at the
// first 64 KiB boundary inside it (accumulate_row_aligned)
template <bool kGather, bool kAligned>
__global__ void __launch_bounds__(1024, 1)
hist_build_kernel_v3(const uint8_t* __restrict__ bins, int row_stride, const int2* __restrict__ gpair,
                     const int32_t* __restrict__ ridx, const B2HistWork* __restrict__ work, int n_work,
                     int total_chunks, int chunk_rows, int window_rows, int n_groups, long long* __restrict__ hist,
                     const B2LevelCtl* __restrict__ ctl, int log2_shards, int node_cap, B2HistPlan plan) {
  HistTarget target; target.base = (unsigned long long*)hist; target.log2_shards = log2_shards; target.node_cap = node_cap;
  target.n_groups = n_groups;
  if (ctl) { n_work = ctl->hist_n_work; total_chunks = ctl->hist_total_chunks; chunk_rows = ctl->hist_chunk_rows; }
  extern __shared__ __align__(16) int32_t s_raw[];  // [2][256][2][32] (+ up to 64 KiB of alignment slack)
  int32_t* s_hist = s_raw;
  if (kAligned) {
    const uint32_t raw0 = (uint32_t)__cvta_generic_to_shared(s_raw);
    s_hist = s_raw + ((((raw0 + 65535u) & ~65535u) - raw0) >> 2);
  }
  int type = 0, cta0 = 0, cta1 = plan.cta_begin[1];
#pragma unroll
  for (int t = 1; t < B2_HIST_MAX_TYPES; ++t)   // constant indices: the plan stays in the parameter bank
    if (t < plan.n_types && (int)blockIdx.x >= plan.cta_begin[t]) { type = t; cta0 = plan.cta_begin[t]; cta1 = plan.cta_begin[t + 1]; }
  const int stream = (int)blockIdx.x - cta0;
  const int n_streams = cta1 - cta0;
  if (total_chunks <= 0 || n_streams <= 0) return;
  const int g0 = 2 * type, g1 = g0 + 1;
  const bool has1 = g1 < n_groups;
  const bool narrow0 = plan.narrow_w > 0 && g0 == n_groups - 1;            // the pair is the narrow group alone
  const bool narrow1 = has1 && plan.narrow_w > 0 && g1 == n_groups - 1;    // full group + narrow group
  const int mask0 = narrow0 ? plan.narrow_w - 1 : 31, mask1 = narrow1 ? plan.narrow_w - 1 : 31;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  const uint32_t smem0 = (uint32_t)__cvta_generic_to_shared(s_hist);

  for (int e = threadIdx.x; e < 2 * B2_GROUP_ELEMS; e += blockDim.x) s_hist[e] = 0;
  __syncthreads();

  int cur = -1;          // work index whose partial sums are in shared memory
  int rows_in_window = 0;
  const int c_begin = (int)(((long long)stream * total_chunks) / n_streams);
  const int c_end = (int)(((long long)(stream + 1) * total_chunks) / n_streams);
  for (int chunk = c_begin; chunk < c_end; ++chunk) {
    int lo = 0, hi = n_work - 1;
    while (lo < hi) {
      int mid = (lo + hi + 1) >> 1;
      if (__ldg(&work[mid].chunk_begin) <= chunk) lo = mid; else hi = mid - 1;
    }
    const int w = lo;
    const int seg_begin = __ldg(&work[w].seg_begin), seg_count = __ldg(&work[w].seg_count);
    const int row0 = (chunk - __ldg(&work[w].chunk_begin)) * chunk_rows;
    const int nrows = min(chunk_rows, seg_count - row0);
    if (cur >= 0 && w != cur) {
      __syncthreads();
      flush_planes(s_hist, target, __ldg(&work[cur].hist_index), g0, mask0);
      if (has1) flush_planes(s_hist + B2_GROUP_ELEMS, target, __ldg(&work[cur].hist_index), g1, mask1);
      __syncthreads();
      rows_in_window = 0;
    } else if (cur >= 0 && rows_in_window + nrows > window_rows) {
      __syncthreads();
      flush_large_cells(s_hist, target, __ldg(&work[cur].hist_index), g0, mask0);
      if (has1) flush_large_cells(s_hist + B2_GROUP_ELEMS, target, __ldg(&work[cur].hist_index), g1, mask1);
      __syncthreads();
      rows_in_window = 0;
    }
    cur = w;
    rows_in_window += nrows;
    const int64_t pos0 = (int64_t)seg_begin + row0;
    if (has1 && !narrow1) {
      full_pass<kGather, 2, kAligned>(bins, row_stride, gpair, ridx, pos0, nrows, g0, smem0, lane, warp, n_warps);
    } else {
      if (!narrow0) full_pass<kGather, 1, kAligned>(bins, row_stride, gpair, ridx, pos0, nrows, g0, smem0, lane, warp, n_warps);
      if (narrow0 || narrow1)
        narrow_dispatch<kGather>(plan.narrow_w, bins, row_stride, gpair, ridx, pos0, nrows, (narrow0 ? g0 : g1) * 32,
                                 smem0 + (narrow0 ? 0u : (uint32_t)(B2_GROUP_ELEMS * 4)), lane, warp, n_warps);
    }
  }
  if (cur >= 0) {
    __syncthreads();
    flush_planes(s_hist, target, __ldg(&work[cur].hist_index), g0, mask0);
    if (has1) flush_planes(s_hist + B2_GROUP_ELEMS, target, __ldg(&work[cur].hist_index), g1, mask1);
  }
}

// ---------------------------------------------------------------- v4: every CTA builds ALL feature groups of its rows
// v3 is expected to be bound by the shared-atomic pipe (one wavefront per clock per SM), not by DRAM, so the way down
// is fewer wavefronts per row.  F = 100 in the even
// layout pays for 128 slots.  v4 serves 96 < F <= 112 (and F = 96): three full groups (192 KiB of int32 cells) plus the
// <= 16 leftover features as a narrow group in a 32 KiB [256 bins][2 planes][16 slots] block = 224 KiB, ONE CTA type, so
// a row is read once by one CTA (no lock-step problem between types, see B2_HIST_NARROW in v3) and costs
// 3 x 2 + w / 8 wavefronts instead of 8.  Lane pair p = lane >> 1 owns a row (16 rows per warp step), lane & 1 selects
// the 16-byte half of each group; the three register stages of the pipeline are the three groups of the row.

// one narrow group in the 16-slot layout, rows [0, nrows) of a chunk: lane = row, W steps; lanes l and l + 16 share banks
template <bool kGather, int W>
__device__ __forceinline__ void narrow_pass16(const uint8_t* __restrict__ bins, int row_stride, const int2* __restrict__ gpair,
                                              const int32_t* __restrict__ ridx, int64_t pos0, int nrows, int byte_off,
                                              uint32_t smem_n, int lane, int warp, int n_warps) {
  const int rot = lane & (W - 1), rep = (lane / W) & (16 / W - 1);
  const uint32_t base = smem_n + (uint32_t)(rep * W) * 4u;
  int r = warp * 32 + lane;
  int64_t rid = r < nrows ? (kGather ? (int64_t)__ldg(ridx + pos0 + r) : pos0 + r) : -1;
  NarrowBytes<W> cur; int2 gp = make_int2(0, 0);
#pragma unroll
  for (int k = 0; k < (W >= 4 ? W / 4 : 1); ++k) cur.w[k] = 0;
  if (rid >= 0) { cur = load_narrow<W>(bins + rid * row_stride + byte_off, rot); gp = __ldg(gpair + rid); }
  for (int r0 = warp * 32; r0 < nrows; r0 += n_warps * 32) {
    const int rn = r0 + n_warps * 32 + lane;
    const int64_t rid_n = rn < nrows ? (kGather ? (int64_t)__ldg(ridx + pos0 + rn) : pos0 + rn) : -1;
    NarrowBytes<W> nxt; int2 gpn = make_int2(0, 0);
#pragma unroll
    for (int k = 0; k < (W >= 4 ? W / 4 : 1); ++k) nxt.w[k] = 0;
    if (rid_n >= 0) { nxt = load_narrow<W>(bins + rid_n * row_stride + byte_off, rot); gpn = __ldg(gpair + rid_n); }
    if (rid >= 0) {
#pragma unroll
      for (int j = 0; j < W; ++j) {
        const uint32_t bin128 = __byte_perm(cur.w[j >> 2], 0u, 0x4404u | ((uint32_t)(j & 3) << 4)) >> 1;
        const uint32_t a = base + bin128 + (((uint32_t)(j + rot)) & (uint32_t)(W - 1)) * 4u;
        red_shared_add(a, gp.x);
        red_shared_add(a + 64u, gp.y);
      }
    }
    rid = rid_n; cur = nxt; gp = gpn;
  }
}
template <bool kGather>
__device__ __forceinline__ void narrow_dispatch16(int w, const uint8_t* __restrict__ bins, int row_stride, const int2* __restrict__ gpair,
                                                  const int32_t* __restrict__ ridx, int64_t pos0, int nrows, int byte_off,
                                                  uint32_t smem_n, int lane, int warp, int n_warps) {
  switch (w) {
    case 16: narrow_pass16<kGather, 16>(bins, row_stride, gpair, ridx, pos0, nrows, byte_off, smem_n, lane, warp, n_warps); break;
    case 8: narrow_pass16<kGather, 8>(bins, row_stride, gpair, ridx, pos0, nrows, byte_off, smem_n, lane, warp, n_warps); break;
    case 4: narrow_pass16<kGather, 4>(bins, row_stride, gpair, ridx, pos0, nrows, byte_off, smem_n, lane, warp, n_warps); break;
    case 2: narrow_pass16<kGather, 2>(bins, row_stride, gpair, ridx, pos0, nrows, byte_off, smem_n, lane, warp, n_warps); break;
    default: narrow_pass16<kGather, 1>(bins, row_stride, gpair, ridx, pos0, nrows, byte_off, smem_n, lane, warp, n_warps); break;
  }
}
// 16-slot narrow block -> global histogram; large_only = the lazy window flush
__device__ __forceinline__ void flush_narrow16(int32_t* s_n, const HistTarget& t, int node_slot, int group, int narrow_w, bool large_only) {
  for (int i = threadIdx.x; i < B2_BINS * 2 * 16; i += blockDim.x) {
    const int v = s_n[i];
    if (v == 0 || (large_only && v < (1 << 30) && v > -(1 << 30))) continue;
    const int bin = i >> 5, plane = (i >> 4) & 1, slot = i & 15 & (narrow_w - 1);
    atomicAdd(t.base + target_index(t, node_slot, group, bin * 64 + plane * 32 + slot), (unsigned long long)(long long)v);
    s_n[i] = 0;
  }
}

__device__ __forceinline__ void accumulate_bins(uint4 v, int2 gp, uint32_t smem_g, int rot, int half) {
  RowData d; d.bins = v; d.gp = gp;
  accumulate_row(d, smem_g, rot, half);
}
// everything a lane needs of one row: its 16-byte half of the three full groups, (even lane only) the first four bytes
// of the narrow group, the gradient pair.  The loads of a row are issued TOGETHER: the four 32-byte sectors of the
// 128-byte row are then requested at the same time and DRAM serves them as one line (staggered over the iteration, a
// 32-byte piece is served as part of a 64-byte burst whose other half is fetched again later).
struct RowRegs {
  uint4 g0, g1, g2;
  uint32_t nb;
  int2 gp;
};
__device__ __forceinline__ RowRegs load_row_regs(const uint8_t* __restrict__ bins, const int2* __restrict__ gpair, int rid,
                                                 int row_stride, int off, bool narrow_lane) {
  RowRegs r;
  r.g0 = r.g1 = r.g2 = make_uint4(0, 0, 0, 0); r.nb = 0; r.gp = make_int2(0, 0);
  if (rid >= 0) {
    const uint8_t* p = bins + (int64_t)rid * row_stride;
    r.g0 = ldg_nc_v4(p + off);
    r.g1 = ldg_nc_v4(p + off + 32);
    r.g2 = ldg_nc_v4(p + off + 64);
    if (narrow_lane) r.nb = __ldg(reinterpret_cast<const uint32_t*>(p + 96));
    r.gp = __ldg(gpair + rid);
  }
  return r;
}
// rows [0, nrows) of a chunk, all groups: lane pair = row (16 rows per warp step), one row of look-ahead in registers.
// narrow_w in {0, 1, 2, 4}: the even lane of the pair also adds the narrow group's features (16 lanes, 4 replicas x 4
// slots = 16 banks of the [256][2][16] block).
template <bool kGather>
__device__ __forceinline__ void row_pass_v4(const uint8_t* __restrict__ bins, int row_stride, const int2* __restrict__ gpair,
                                            const int32_t* __restrict__ ridx, int64_t pos0, int nrows, uint32_t smem_base,
                                            uint32_t smem_n, int narrow_w, int lane, int warp, int n_warps) {
  const int sub = lane >> 1, half = lane & 1, rot = sub;
  const int off = half * 16;
  const int iter_rows = n_warps * 16;
  const int rbase = warp * 16;
  const bool narrow_lane = narrow_w > 0 && half == 0;
  const int nmask = narrow_w - 1;
  const int nrot = sub & nmask;
  const uint32_t nbase = smem_n + (uint32_t)(narrow_w > 0 ? (((sub / narrow_w) & (16 / narrow_w - 1)) * narrow_w) : 0) * 4u;
  int id = (int)fetch_rid<kGather>(ridx, pos0, rbase + sub, nrows);
  RowRegs cur = load_row_regs(bins, gpair, id, row_stride, off, narrow_lane);
  int id_n = (int)fetch_rid<kGather>(ridx, pos0, rbase + sub + iter_rows, nrows);
  int id_nn = (int)fetch_rid<kGather>(ridx, pos0, rbase + sub + 2 * iter_rows, nrows);
  for (int r = rbase; r < nrows; r += iter_rows) {   // warp-uniform trip count
    const RowRegs nxt = load_row_regs(bins, gpair, id_n, row_stride, off, narrow_lane);
    id_n = id_nn;
    if (id_n >= 0) {   // the row after the next one: pull its line (one 64-byte half per lane of the pair) and its gradient pair into L2
      const uint8_t* pf = bins + (int64_t)id_n * row_stride + half * 64;
      asm volatile("prefetch.global.L2 [%0];" ::"l"(pf));
      if (half == 0) asm volatile("prefetch.global.L2 [%0];" ::"l"(gpair + id_n));
    }
    id_nn = (int)fetch_rid<kGather>(ridx, pos0, r + sub + 3 * iter_rows, nrows);
    accumulate_bins(cur.g0, cur.gp, smem_base, rot, half);
    accumulate_bins(cur.g1, cur.gp, smem_base + B2_GROUP_ELEMS * 4, rot, half);
    accumulate_bins(cur.g2, cur.gp, smem_base + 2 * B2_GROUP_ELEMS * 4, rot, half);
    if (narrow_lane) {
      for (int j = 0; j < narrow_w; ++j) {
        const int idx = (j + nrot) & nmask;
        const uint32_t bin = (cur.nb >> (idx * 8)) & 0xffu;
        const uint32_t a = nbase + bin * 128u + (uint32_t)idx * 4u;
        red_shared_add(a, cur.gp.x);
        red_shared_add(a + 64u, cur.gp.y);
      }
    }
    cur = nxt;
  }
}

template <bool kGather>
__global__ void __launch_bounds__(512, 1)
hist_build_kernel_v4(const uint8_t* __restrict__ bins, int row_stride, const int2* __restrict__ gpair,
                     const int32_t* __restrict__ ridx, const B2HistWork* __restrict__ work, int n_work,
                     int total_chunks, int chunk_rows, int window_rows, int n_groups, long long* __restrict__ hist,
                     const B2LevelCtl* __restrict__ ctl, int log2_shards, int node_cap, int narrow_w) {
  HistTarget target; target.base = (unsigned long long*)hist; target.log2_shards = log2_shards; target.node_cap = node_cap;
  target.n_groups = n_groups;
  if (ctl) { n_work = ctl->hist_n_work; total_chunks = ctl->hist_total_chunks; chunk_rows = ctl->hist_chunk_rows; }
  extern __shared__ __align__(16) int32_t s_hist[];  // [3][256][2][32] then the narrow block [256][2][16]
  int32_t* s_narrow = s_hist + 3 * B2_GROUP_ELEMS;
  if (total_chunks <= 0) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  const uint32_t smem0 = (uint32_t)__cvta_generic_to_shared(s_hist);
  const uint32_t smem_n = smem0 + 3u * B2_GROUP_ELEMS * 4u;
  const int inline_w = narrow_w <= 4 ? narrow_w : 0;     // wider leftovers: their own pass over the chunk
  for (int e = threadIdx.x; e < 3 * B2_GROUP_ELEMS + B2_BINS * 32; e += blockDim.x) s_hist[e] = 0;
  __syncthreads();
  int cur = -1, rows_in_window = 0;
  const int stream = blockIdx.x, n_streams = gridDim.x;
  const int c_begin = (int)(((long long)stream * total_chunks) / n_streams);
  const int c_end = (int)(((long long)(stream + 1) * total_chunks) / n_streams);
  for (int chunk = c_begin; chunk < c_end; ++chunk) {
    int lo = 0, hi = n_work - 1;
    while (lo < hi) {
      int mid = (lo + hi + 1) >> 1;
      if (__ldg(&work[mid].chunk_begin) <= chunk) lo = mid; else hi = mid - 1;
    }
    const int w = lo;
    const int seg_begin = __ldg(&work[w].seg_begin), seg_count = __ldg(&work[w].seg_count);
    const int row0 = (chunk - __ldg(&work[w].chunk_begin)) * chunk_rows;
    const int nrows = min(chunk_rows, seg_count - row0);
    const bool node_change = cur >= 0 && w != cur;
    if (node_change || (cur >= 0 && rows_in_window + nrows > window_rows)) {
      const int node = __ldg(&work[cur].hist_index);
      __syncthreads();
      for (int g = 0; g < 3; ++g) {
        if (node_change) flush_planes(s_hist + g * B2_GROUP_ELEMS, target, node, g);
        else flush_large_cells(s_hist + g * B2_GROUP_ELEMS, target, node, g);
      }
      if (narrow_w > 0) flush_narrow16(s_narrow, target, node, 3, narrow_w, !node_change);
      __syncthreads();
      rows_in_window = 0;
    }
    cur = w;
    rows_in_window += nrows;
    const int64_t pos0 = (int64_t)seg_begin + row0;
    row_pass_v4<kGather>(bins, row_stride, gpair, ridx, pos0, nrows, smem0, smem_n, inline_w, lane, warp, n_warps);
    if (narrow_w > 4) narrow_dispatch16<kGather>(narrow_w, bins, row_stride, gpair, ridx, pos0, nrows, 96, smem_n, lane, warp, n_warps);
  }
  if (cur >= 0) {
    const int node = __ldg(&work[cur].hist_index);
    __syncthreads();
    for (int g = 0; g < 3; ++g) flush_planes(s_hist + g * B2_GROUP_ELEMS, target, node, g);
    if (narrow_w > 0) flush_narrow16(s_narrow, target, node, 3, narrow_w, false);
  }
}

// ---------------------------------------------------------------- sibling = parent - built
__global__ void hist_subtract_kernel(const long long* __restrict__ parent_level, long long* __restrict__ level,
                                     const int32_t* __restrict__ triples, int n_pairs, int64_t node_elems,
                                     const B2LevelCtl* __restrict__ ctl) {
  if (ctl) n_pairs = ctl->n_pairs;
  // triples[3*p] = parent slot (prev level), built slot, sibling slot (this level)
  const int p = blockIdx.y;
  if (p >= n_pairs) return;
  const long long* par = parent_level + (size_t)triples[3 * p] * node_elems;
  const long long* built = level + (size_t)triples[3 * p + 1] * node_elems;
  long long* sib = level + (size_t)triples[3 * p + 2] * node_elems;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < node_elems; i += (int64_t)gridDim.x * blockDim.x)
    sib[i] = par[i] - built[i];
}

}  // namespace b2

extern "C" {

// the configured kernel variant (B2_HIST_VARIANT); engine.cu picks the bin-matrix layout that suits it
int b2_hist_variant() {
  const char* e = getenv("B2_HIST_VARIANT");
  int v = e ? atoi(e) : B2_HIST_DEFAULT_VARIANT;
  return (v < 0 || v > 4) ? B2_HIST_DEFAULT_VARIANT : v;
}

// Launch on `stream`.  grid = n_groups * n_streams persistent CTAs; returns the cudaError.
int b2_launch_hist(const uint8_t* bins, int row_stride, const int2* gpair, const int32_t* ridx,
                   const B2HistWork* work, int n_work, int total_chunks, int chunk_rows, int window_rows,
                   int n_groups, long long* hist, const B2LevelCtl* ctl, int log2_shards, int node_cap, int narrow_w,
                   int num_sms, cudaStream_t stream) {
  static bool attr_set = false;
  static int debug_mode = -1, variant_cfg = -1;
  if (debug_mode < 0) { const char* e = getenv("B2_HIST_DEBUG_MODE"); debug_mode = e ? atoi(e) : 0; }
  // variants (B2_HIST_VARIANT): 0 = 256 threads x 3 CTAs/SM, one group per CTA
  //                             1 = 512 threads x 2 CTAs/SM, one group per CTA
  //                             2 = 1024 threads x 1 CTA/SM, two groups per CTA
  //                             3 = group pairs with a narrow last group, CTAs per pair by cost (default)
  if (variant_cfg < 0) {
    const char* e = getenv("B2_HIST_VARIANT");
    variant_cfg = e ? atoi(e) : B2_HIST_DEFAULT_VARIANT;
    const char* t = getenv("B2_HIST_THREADS");   // older spelling of variant_cfg 0
    if (!e && t && atoi(t) == 256) variant_cfg = 0;
    if (variant_cfg < 0 || variant_cfg > 4) variant_cfg = B2_HIST_DEFAULT_VARIANT;
  }
  int variant = variant_cfg;
  if (variant == 4 && ((n_groups == 3 && narrow_w == 0) || (n_groups == 4 && narrow_w > 0))) {
    // ---- all groups of a row in one CTA: three full groups + the narrow leftover (96 <= F <= 112)
    static bool attr4 = false;
    const int smem4 = (3 * B2_GROUP_ELEMS + B2_BINS * 32) * (int)sizeof(int32_t);   // 224 KiB
    if (!attr4) {
      cudaFuncSetAttribute(b2::hist_build_kernel_v4<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem4);
      cudaFuncSetAttribute(b2::hist_build_kernel_v4<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem4);
      attr4 = true;
    }
    if (!ctl && (total_chunks <= 0 || n_work <= 0)) return 0;
    if (!ctl && chunk_rows > window_rows) return (int)cudaErrorInvalidValue;
    int n_ctas = num_sms;
    if (!ctl && n_ctas > total_chunks) n_ctas = total_chunks;
    if (ridx) b2::hist_build_kernel_v4<true><<<n_ctas, 512, smem4, stream>>>(bins, row_stride, gpair, ridx, work, n_work, total_chunks, chunk_rows,
                                                                              window_rows, n_groups, hist, ctl, log2_shards, node_cap, narrow_w);
    else b2::hist_build_kernel_v4<false><<<n_ctas, 512, smem4, stream>>>(bins, row_stride, gpair, ridx, work, n_work, total_chunks, chunk_rows,
                                                                            window_rows, n_groups, hist, ctl, log2_shards, node_cap, narrow_w);
    return (int)cudaGetLastError();
  }
  if (variant == 4) variant = 3;   // other feature counts: group pairs
  // more groups than the pair plan holds (F > 32 * 2 * B2_HIST_MAX_TYPES = 512): one group per CTA, 512 threads
  if (variant == 3 && (n_groups + 1) / 2 > B2_HIST_MAX_TYPES) variant = 1;
  if (variant == 3) {
    // ---- group pairs with a narrow last group: CTAs per type in proportion to the atomic wavefronts per row
    static bool attr3 = false;
    static int aligned = -1;   // B2_HIST_ALIGNED=1: 64 KiB-aligned histograms, one PRMT forms the cell address
    if (aligned < 0) { const char* e = getenv("B2_HIST_ALIGNED"); aligned = (e && atoi(e) != 0) ? 1 : 0; }
    if (!attr3) {
      cudaFuncSetAttribute(b2::hist_build_kernel_v3<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, B2_GROUP_ELEMS * 8);
      cudaFuncSetAttribute(b2::hist_build_kernel_v3<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, B2_GROUP_ELEMS * 8);
      cudaFuncSetAttribute(b2::hist_build_kernel_v3<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, B2_GROUP_ELEMS * 8 + 65536);
      cudaFuncSetAttribute(b2::hist_build_kernel_v3<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, B2_GROUP_ELEMS * 8 + 65536);
      attr3 = true;
    }
    if (!ctl && (total_chunks <= 0 || n_work <= 0)) return 0;
    if (!ctl && chunk_rows > window_rows) return (int)cudaErrorInvalidValue;
    B2HistPlan plan;
    plan.n_types = (n_groups + 1) / 2; plan.narrow_w = narrow_w;
    if (plan.n_types > B2_HIST_MAX_TYPES) return (int)cudaErrorInvalidValue;
    int cost[B2_HIST_MAX_TYPES], total_cost = 0;
    for (int t = 0; t < plan.n_types; ++t) {
      cost[t] = 0;
      for (int g = 2 * t; g < 2 * t + 2 && g < n_groups; ++g) cost[t] += (narrow_w > 0 && g == n_groups - 1) ? narrow_w : 32;
      total_cost += cost[t];
    }
    int n_ctas = num_sms, assigned = 0, biggest = 0;
    if (n_ctas < plan.n_types) n_ctas = plan.n_types;
    int streams[B2_HIST_MAX_TYPES];
    for (int t = 0; t < plan.n_types; ++t) {
      // even layout: every type gets the SAME number of streams, also when the last type holds a single group (odd group
      // count) -- the types then walk the chunk list in lock step and a row's halves are fetched together (an idle tail
      // on the cheap type costs less than the 2.8x DRAM traffic measured when the types drift apart).  Only the narrow
      // layout splits the CTAs by cost.
      streams[t] = narrow_w > 0 ? (int)(((long long)n_ctas * cost[t] + total_cost / 2) / total_cost) : n_ctas / plan.n_types;
      if (streams[t] < 1) streams[t] = 1;
      if (!ctl && streams[t] > total_chunks) streams[t] = total_chunks;
      assigned += streams[t];
      if (cost[t] > cost[biggest]) biggest = t;
    }
    if (narrow_w > 0 && (ctl || assigned > n_ctas)) {   // cost-proportional split: make the persistent grid exactly one CTA per SM
      streams[biggest] += n_ctas - assigned;
      if (streams[biggest] < 1) streams[biggest] = 1;
    }
    plan.cta_begin[0] = 0;
    for (int t = 0; t < plan.n_types; ++t) plan.cta_begin[t + 1] = plan.cta_begin[t] + streams[t];
    for (int t = plan.n_types + 1; t <= B2_HIST_MAX_TYPES; ++t) plan.cta_begin[t] = plan.cta_begin[plan.n_types];
    dim3 grid3(plan.cta_begin[plan.n_types]), block3(1024);
    const int smem3 = 2 * B2_GROUP_ELEMS * (int)sizeof(int32_t) + (aligned ? 65536 : 0);
#define B2_V3_ARGS bins, row_stride, gpair, ridx, work, n_work, total_chunks, chunk_rows, window_rows, n_groups, hist, ctl, log2_shards, node_cap, plan
    if (aligned) {
      if (ridx) b2::hist_build_kernel_v3<true, true><<<grid3, block3, smem3, stream>>>(B2_V3_ARGS);
      else b2::hist_build_kernel_v3<false, true><<<grid3, block3, smem3, stream>>>(B2_V3_ARGS);
    } else {
      if (ridx) b2::hist_build_kernel_v3<true, false><<<grid3, block3, smem3, stream>>>(B2_V3_ARGS);
      else b2::hist_build_kernel_v3<false, false><<<grid3, block3, smem3, stream>>>(B2_V3_ARGS);
    }
#undef B2_V3_ARGS
    return (int)cudaGetLastError();
  }
  const int gpc = variant == 2 ? 2 : 1;
  const int smem = gpc * B2_GROUP_ELEMS * (int)sizeof(int32_t);  // 64 KiB per group
  if (!attr_set) {
    cudaFuncSetAttribute(b2::hist_build_kernel<true, 256, 3, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, B2_GROUP_ELEMS * 4);
    cudaFuncSetAttribute(b2::hist_build_kernel<false, 256, 3, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, B2_GROUP_ELEMS * 4);
    cudaFuncSetAttribute(b2::hist_build_kernel<true, 512, 2, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, B2_GROUP_ELEMS * 4);
    cudaFuncSetAttribute(b2::hist_build_kernel<false, 512, 2, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, B2_GROUP_ELEMS * 4);
    cudaFuncSetAttribute(b2::hist_build_kernel<true, 1024, 1, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, B2_GROUP_ELEMS * 8);
    cudaFuncSetAttribute(b2::hist_build_kernel<false, 1024, 1, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, B2_GROUP_ELEMS * 8);
    attr_set = true;
  }
  // with ctl the work list / chunk counts live in device memory (sync-free level loop) and the grid is the
  // full persistent grid; without it they are host values
  if (!ctl && (total_chunks <= 0 || n_work <= 0)) return 0;
  if (!ctl && chunk_rows > window_rows) return (int)cudaErrorInvalidValue;  // a chunk must fit one int32 window
  const int ctas_per_sm = variant == 0 ? 3 : variant == 1 ? 2 : 1;
  const int n_cta_groups = (n_groups + gpc - 1) / gpc;
  int n_streams = (num_sms * ctas_per_sm) / n_cta_groups;
  if (n_streams < 1) n_streams = 1;
  if (!ctl && n_streams > total_chunks) n_streams = total_chunks;
  dim3 grid(n_cta_groups * n_streams), block(variant == 0 ? 256 : variant == 1 ? 512 : 1024);
#define B2_HIST_ARGS bins, row_stride, gpair, ridx, work, n_work, total_chunks, chunk_rows, window_rows, n_groups, hist, ctl, log2_shards, \
                     node_cap, debug_mode
  if (variant == 2) {
    if (ridx) b2::hist_build_kernel<true, 1024, 1, 2><<<grid, block, smem, stream>>>(B2_HIST_ARGS);
    else b2::hist_build_kernel<false, 1024, 1, 2><<<grid, block, smem, stream>>>(B2_HIST_ARGS);
  } else if (variant == 1) {
    if (ridx) b2::hist_build_kernel<true, 512, 2, 1><<<grid, block, smem, stream>>>(B2_HIST_ARGS);
    else b2::hist_build_kernel<false, 512, 2, 1><<<grid, block, smem, stream>>>(B2_HIST_ARGS);
  } else {
    if (ridx) b2::hist_build_kernel<true, 256, 3, 1><<<grid, block, smem, stream>>>(B2_HIST_ARGS);
    else b2::hist_build_kernel<false, 256, 3, 1><<<grid, block, smem, stream>>>(B2_HIST_ARGS);
  }
#undef B2_HIST_ARGS
  return (int)cudaGetLastError();
}

int b2_launch_hist_subtract(const long long* parent_level, long long* level, const int32_t* triples, int n_pairs,
                            int64_t node_elems, const B2LevelCtl* ctl, cudaStream_t stream) {
  if (n_pairs <= 0) return 0;   // with ctl: n_pairs is the upper bound, the real count is read on the device
  int bx = (int)((node_elems + 256 * 8 - 1) / (256 * 8));
  if (bx < 1) bx = 1;
  dim3 grid(bx, n_pairs);
  b2::hist_subtract_kernel<<<grid, 256, 0, stream>>>(parent_level, level, triples, n_pairs, node_elems, ctl);
  return (int)cudaGetLastError();
}
}
