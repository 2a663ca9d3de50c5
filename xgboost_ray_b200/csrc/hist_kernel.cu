// hist_kernel.cu -- feature x bin gradient/hessian histogram build for sm_90a.
//
// Replaces the BuildHist stage that the reference reaches through xgb.train()
// (xgboost_ray/main.py:745-752; SURVEY.md 8a row a10).  Bandwidth-bound scatter-reduce:
// no tensor cores.  Design (DESIGN.md "Histogram kernel"):
//
//  * A feature group is <= 32 features -> 32 "slots".  A CTA keeps the histogram of each of its groups for ONE node at
//    a time in shared memory as two int32 planes [256 bins][32 slots] (g and h): 64 KiB per group.  Because a bin row
//    is exactly 32 words, the bank of an update is its SLOT and does not depend on the bin value.
//  * Up to kMaxPairGroups groups (F <= 512) hist_build_kernel_v3 runs: a CTA owns a PAIR of groups (128 KiB, one
//    1024-thread CTA per SM).  Wider matrices run hist_build_kernel: one group per CTA (64 KiB, 512 threads, two CTAs
//    per SM).
//  * A lane loads 16 bin bytes of one row (LDG.128 straight to registers; staging rows through
//    shared memory would spend the shared-memory bandwidth that the atomics are bound by).  Two
//    lanes cover the 32-byte group slice of a row.  Lane l pre-rotates its bytes so that at step j the
//    32 lanes of a warp touch 32 DIFFERENT slots: every ATOMS.ADD is bank-conflict free for any data,
//    one wavefront per instruction.
//  * Sums are exact integers (fixed-point gradients), so the result is independent of the order
//    of rows, CTAs and GPUs.  A CTA flushes its planes to the global int64 histogram when it moves
//    to another node; every `window_rows` = 2^(30-qbits) rows it flushes just the cells that reached
//    2^30 (none for well spread bins), which is what keeps the int32 cells from overflowing.
//  * Rows of a node are addressed through the row-index segment list (gather) except at the root.
#include "hist_common.cuh"
#include "launch.h"

namespace b2 {

// Feature groups up to which one CTA type owns a pair of groups (hist_build_kernel_v3); above it, one group per CTA.
constexpr int kMaxPairGroups = 16;

// rows [0, nrows) of a chunk for the kGPC full groups of a CTA: kGPC = 2 -> FOUR lanes read the 64 contiguous bytes of
// the pair (one L1 wavefront instead of two) and the row id / gradient pair loads are shared by both groups; kGPC = 1 ->
// two lanes cover the 32 bytes of the single group, 16 rows per warp step.
template <bool kGather, int kGPC>
__device__ __forceinline__ void full_pass(const uint8_t* __restrict__ bins, int row_stride, const int2* __restrict__ gpair,
                                          const int32_t* __restrict__ ridx, int64_t pos0, int nrows, int group0,
                                          uint32_t smem_base, int lane, int warp, int n_warps) {
  constexpr int kLanesPerRow = 2 * kGPC;
  constexpr int kRowsPerWarp = 32 / kLanesPerRow;
  // lane -> (row of the warp step, group of the CTA, 16-byte half of the group slice).  rot is distinct for the
  // 16 (row, group) pairs of a warp, so at every step the 32 lanes hit 32 different banks (bank = slot).
  const int sub = lane / kLanesPerRow, gsel = (lane % kLanesPerRow) >> 1, half = lane & 1;
  const int rot = sub * kGPC + gsel;
  const int lane_byte_off = (group0 + gsel) * 32 + half * 16;
  const uint32_t smem_g = smem_base + gsel * (B2_GROUP_ELEMS * 4);
  const int iter_rows = n_warps * kRowsPerWarp;
  // 3-stage register pipeline: while stage k is accumulated, the loads of the next two
  // iterations are in flight, and (gather) the row ids of three more iterations behind them,
  // so no load waits on the ridx -> bins dependency.
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
  for (int r = rbase; r < nrows; r += 3 * iter_rows) {   // warp-uniform trip count
    accumulate_row(s0, smem_g, rot, half);
    s0 = load_row_id(bins, gpair, id0, row_stride, lane_byte_off);
    id0 = fetch_rid<kGather>(ridx, pos0, r + sub + 6 * iter_rows, nrows);
    if (r + iter_rows < nrows) accumulate_row(s1, smem_g, rot, half);
    s1 = load_row_id(bins, gpair, id1, row_stride, lane_byte_off);
    id1 = fetch_rid<kGather>(ridx, pos0, r + sub + 7 * iter_rows, nrows);
    if (r + 2 * iter_rows < nrows) accumulate_row(s2, smem_g, rot, half);
    s2 = load_row_id(bins, gpair, id2, row_stride, lane_byte_off);
    id2 = fetch_rid<kGather>(ridx, pos0, r + sub + 8 * iter_rows, nrows);
  }
}

// one group per CTA (n_groups > kMaxPairGroups): CTA b builds group b % n_groups, stream b / n_groups
template <bool kGather>
__global__ void __launch_bounds__(512, 2)
hist_build_kernel(const uint8_t* __restrict__ bins, int row_stride, const int2* __restrict__ gpair,
                  const int32_t* __restrict__ ridx, const B2HistWork* __restrict__ work, int n_work,
                  int total_chunks, int chunk_rows, int window_rows, int n_groups, long long* __restrict__ hist,
                  const B2LevelCtl* __restrict__ ctl, int log2_shards, int node_cap) {
  HistTarget target; target.base = (unsigned long long*)hist; target.log2_shards = log2_shards; target.node_cap = node_cap;
  target.n_groups = n_groups;
  if (ctl) { n_work = ctl->hist_n_work; total_chunks = ctl->hist_total_chunks; chunk_rows = ctl->hist_chunk_rows; }
  extern __shared__ __align__(16) int32_t s_hist[];  // [256][2][32]
  const int group = blockIdx.x % n_groups;
  const int stream = blockIdx.x / n_groups;
  const int n_streams = gridDim.x / n_groups;
  if (total_chunks <= 0) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  const uint32_t smem0 = (uint32_t)__cvta_generic_to_shared(s_hist);

  for (int e = threadIdx.x; e < B2_GROUP_ELEMS; e += blockDim.x) s_hist[e] = 0;
  __syncthreads();

  int cur = -1;          // work index whose partial sums are in shared memory
  int rows_in_window = 0;
  // A stream takes a CONTIGUOUS range of the chunk list, so consecutive chunks of a CTA mostly belong to the same
  // node and the 2 x 16K-cell node flush happens once per node per CTA instead of once per chunk (with a strided
  // assignment every chunk of a deep level was a node change: levels 6-7 cost 1.5x the root per row).
  const int c_begin = (int)(((long long)stream * total_chunks) / n_streams);
  const int c_end = (int)(((long long)(stream + 1) * total_chunks) / n_streams);
  for (int chunk = c_begin; chunk < c_end; ++chunk) {
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
      flush_planes(s_hist, target, __ldg(&work[cur].hist_index), group);
      __syncthreads();
      rows_in_window = 0;
    } else if (cur >= 0 && rows_in_window + nrows > window_rows) {
      // same node, overflow guard interval reached: flush only the (rare) cells at or above 2^30
      // (flushing all cells with RED.64 every window, or a CTA-private int64 scratch with plain read-modify-write,
      // would move far more data than the few saturated cells)
      __syncthreads();
      flush_large_cells(s_hist, target, __ldg(&work[cur].hist_index), group);
      __syncthreads();
      rows_in_window = 0;
    }
    cur = w;
    rows_in_window += nrows;
    const int64_t pos0 = (int64_t)seg_begin + row0;
    full_pass<kGather, 1>(bins, row_stride, gpair, ridx, pos0, nrows, group, smem0, lane, warp, n_warps);
  }
  if (cur >= 0) {
    __syncthreads();
    flush_planes(s_hist, target, __ldg(&work[cur].hist_index), group);
  }
}

// ================================================================ v3: group pairs
// n_groups <= kMaxPairGroups: CTA type t owns groups 2t and 2t + 1 (the last type of an odd group count holds one).
// Every type gets the SAME number of streams, also when the last type holds a single group: the types then walk the
// chunk list in lock step and a row's halves are fetched together (an idle tail on the cheap type costs less than the
// 2.8x DRAM traffic measured when the types drift apart).  CTA b is type b / n_streams, stream b % n_streams.
template <bool kGather>
__global__ void __launch_bounds__(1024, 1)
hist_build_kernel_v3(const uint8_t* __restrict__ bins, int row_stride, const int2* __restrict__ gpair,
                     const int32_t* __restrict__ ridx, const B2HistWork* __restrict__ work, int n_work,
                     int total_chunks, int chunk_rows, int window_rows, int n_groups, long long* __restrict__ hist,
                     const B2LevelCtl* __restrict__ ctl, int log2_shards, int node_cap, int n_streams) {
  HistTarget target; target.base = (unsigned long long*)hist; target.log2_shards = log2_shards; target.node_cap = node_cap;
  target.n_groups = n_groups;
  if (ctl) { n_work = ctl->hist_n_work; total_chunks = ctl->hist_total_chunks; chunk_rows = ctl->hist_chunk_rows; }
  extern __shared__ __align__(16) int32_t s_hist[];  // [2][256][2][32]
  const int type = (int)blockIdx.x / n_streams;
  const int stream = (int)blockIdx.x % n_streams;
  if (total_chunks <= 0) return;
  const int g0 = 2 * type, g1 = g0 + 1;
  const bool has1 = g1 < n_groups;
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
      flush_planes(s_hist, target, __ldg(&work[cur].hist_index), g0);
      if (has1) flush_planes(s_hist + B2_GROUP_ELEMS, target, __ldg(&work[cur].hist_index), g1);
      __syncthreads();
      rows_in_window = 0;
    } else if (cur >= 0 && rows_in_window + nrows > window_rows) {
      __syncthreads();
      flush_large_cells(s_hist, target, __ldg(&work[cur].hist_index), g0);
      if (has1) flush_large_cells(s_hist + B2_GROUP_ELEMS, target, __ldg(&work[cur].hist_index), g1);
      __syncthreads();
      rows_in_window = 0;
    }
    cur = w;
    rows_in_window += nrows;
    const int64_t pos0 = (int64_t)seg_begin + row0;
    if (has1) full_pass<kGather, 2>(bins, row_stride, gpair, ridx, pos0, nrows, g0, smem0, lane, warp, n_warps);
    else full_pass<kGather, 1>(bins, row_stride, gpair, ridx, pos0, nrows, g0, smem0, lane, warp, n_warps);
  }
  if (cur >= 0) {
    __syncthreads();
    flush_planes(s_hist, target, __ldg(&work[cur].hist_index), g0);
    if (has1) flush_planes(s_hist + B2_GROUP_ELEMS, target, __ldg(&work[cur].hist_index), g1);
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

// the CSR build's per-node row totals [node_cap][2]; the dense build needs no scratch
size_t b2_hist_scratch_elems(B2BinRows src, int node_cap) { return src.ebins ? 2 * (size_t)node_cap : 0; }

// Launch on `stream`: a persistent grid of n_types * n_streams group-pair CTAs (n_groups <= kMaxPairGroups) or
// n_groups * n_streams one-group CTAs; returns the cudaError.
int b2_launch_hist(B2BinRows src, const int32_t* group_size, const int2* gpair, const int32_t* ridx, const B2HistWork* work,
                   int n_work, int total_chunks, int chunk_rows, int window_rows, int n_groups, long long* hist,
                   long long* scratch, const B2LevelCtl* ctl, int log2_shards, int node_cap, int num_sms, cudaStream_t stream) {
  if (src.ebins)
    return b2::launch_hist_csr(src, group_size, gpair, ridx, work, n_work, total_chunks, chunk_rows, n_groups, hist, scratch,
                               ctl, log2_shards, node_cap, num_sms, stream);
  const uint8_t* bins = src.bins; const int row_stride = src.row_stride;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(b2::hist_build_kernel_v3<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, B2_GROUP_ELEMS * 8);
    cudaFuncSetAttribute(b2::hist_build_kernel_v3<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, B2_GROUP_ELEMS * 8);
    cudaFuncSetAttribute(b2::hist_build_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, B2_GROUP_ELEMS * 4);
    cudaFuncSetAttribute(b2::hist_build_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, B2_GROUP_ELEMS * 4);
    attr_set = true;
  }
  // with ctl the work list / chunk counts live in device memory (sync-free level loop) and the grid is the
  // full persistent grid; without it they are host values
  if (!ctl && (total_chunks <= 0 || n_work <= 0)) return 0;
  if (!ctl && chunk_rows > window_rows) return (int)cudaErrorInvalidValue;  // a chunk must fit one int32 window
#define HIST_ARGS bins, row_stride, gpair, ridx, work, n_work, total_chunks, chunk_rows, window_rows, n_groups, hist, ctl, log2_shards, node_cap
  if (n_groups <= b2::kMaxPairGroups) {
    const int n_types = (n_groups + 1) / 2;
    const int n_ctas = num_sms < n_types ? n_types : num_sms;   // one 1024-thread CTA per SM
    int n_streams = n_ctas / n_types;
    if (!ctl && n_streams > total_chunks) n_streams = total_chunks;
    const int smem = 2 * B2_GROUP_ELEMS * (int)sizeof(int32_t);
    if (ridx) b2::hist_build_kernel_v3<true><<<n_types * n_streams, 1024, smem, stream>>>(HIST_ARGS, n_streams);
    else b2::hist_build_kernel_v3<false><<<n_types * n_streams, 1024, smem, stream>>>(HIST_ARGS, n_streams);
  } else {
    int n_streams = (num_sms * 2) / n_groups;   // two 512-thread CTAs per SM
    if (n_streams < 1) n_streams = 1;
    if (!ctl && n_streams > total_chunks) n_streams = total_chunks;
    const int smem = B2_GROUP_ELEMS * (int)sizeof(int32_t);
    if (ridx) b2::hist_build_kernel<true><<<n_groups * n_streams, 512, smem, stream>>>(HIST_ARGS);
    else b2::hist_build_kernel<false><<<n_groups * n_streams, 512, smem, stream>>>(HIST_ARGS);
  }
#undef HIST_ARGS
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
