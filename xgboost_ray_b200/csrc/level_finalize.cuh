// level_finalize.cuh -- what follows the partition of a level: child segments, build-child choice, next hist work list.
//
// Run by ONE CTA of kThreads threads: the last CTA of partition_kernel to finish (partition_kernel.cu).  The left-row
// counts of the split nodes were added by the other CTAs with atomics; the caller fences before it reads them here.
#pragma once

#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace b2 {

template <int kThreads>
struct FinalizeScratch {
  typedef cub::BlockScan<int, kThreads> Scan;
  typename Scan::TempStorage scan;
  long long rows;
  int chunk_rows;
};

template <int kThreads>
__device__ void finalize_level_block(FinalizeScratch<kThreads>& sm, const B2LevelCtl* __restrict__ ctl_cur,
                                     const B2SplitWork* __restrict__ split_work, const int32_t* counters,
                                     const B2FinalizeArgs& a) {
  typedef typename FinalizeScratch<kThreads>::Scan Scan;
  B2LevelCtl* ctl_nxt = a.ctl_nxt; B2NodeSeg* seg_nxt = a.seg_nxt; B2EvalNode* ev_nxt = a.ev_nxt;
  const int32_t* pair_parent_hist = a.pair_parent_hist; B2HistWork* hist_work = a.hist_work; int32_t* triples = a.triples;
  const int max_pairs = a.max_pairs, need_hist = a.need_hist, n_streams = a.n_streams, window_rows = a.window_rows;
  const int chunk_rows_override = a.chunk_rows_override;
  long long* stat_rows = a.stat_rows;
  const int ns = ctl_cur->n_split;
  if (threadIdx.x == 0) sm.rows = 0;
  __syncthreads();
  // pass 1: segments + total rows to build
  long long my_rows = 0;
  for (int j = threadIdx.x; j < ns; j += kThreads) {
    const B2SplitWork sw = split_work[j];
    const int cl = __ldcg(counters + 2 * j);   // written by the other CTAs' atomics: read at L2
    B2NodeSeg sl = seg_nxt[2 * j], sr = seg_nxt[2 * j + 1];
    sl.begin = sw.seg_begin; sl.count = cl;
    sr.begin = sw.seg_begin + cl; sr.count = sw.seg_count - cl;
    seg_nxt[2 * j] = sl; seg_nxt[2 * j + 1] = sr;
    if (need_hist) {
      const bool build_left = ev_nxt[2 * j].sum_h < ev_nxt[2 * j + 1].sum_h;   // smaller hessian (A.5)
      my_rows += build_left ? sl.count : sr.count;
    }
  }
  if (!need_hist) return;
  atomicAdd((unsigned long long*)&sm.rows, (unsigned long long)my_rows);
  __syncthreads();
  if (threadIdx.x == 0) {
    int c = chunk_rows_override;
    if (c <= 0) {
      // large levels: ~4 chunks per CTA stream for balance; small levels: ~1, because every extra
      // (CTA, node) pair costs a full 16K-cell flush
      const long long per_stream = sm.rows / n_streams;
      const long long target = per_stream >= 16384 ? per_stream / 4 : per_stream;
      c = 512;
      while (c < target && c < 8192) c <<= 1;
    }
    if (c > window_rows) c = window_rows;   // one chunk = one int32 window
    sm.chunk_rows = c;
    if (stat_rows) *stat_rows = sm.rows;
  }
  __syncthreads();
  const int chunk_rows = sm.chunk_rows;
  int carry = 0;
  for (int base = 0; base < ns; base += kThreads) {
    const int j = base + threadIdx.x;
    int chunks = 0, begin = 0, count = 0;
    if (j < ns) {
      const bool build_left = ev_nxt[2 * j].sum_h < ev_nxt[2 * j + 1].sum_h;
      const int b = build_left ? 2 * j : 2 * j + 1, s = b ^ 1;
      begin = seg_nxt[b].begin; count = seg_nxt[b].count;
      chunks = (count + chunk_rows - 1) / chunk_rows;
      ev_nxt[b].hist_index = j; ev_nxt[s].hist_index = max_pairs + j;
      triples[3 * j] = pair_parent_hist[j]; triples[3 * j + 1] = j; triples[3 * j + 2] = max_pairs + j;
    }
    int ex, total;
    Scan(sm.scan).ExclusiveSum(chunks, ex, total);
    __syncthreads();
    const int cb = carry + ex;
    carry += total;
    if (j < ns) { B2HistWork w; w.seg_begin = begin; w.seg_count = count; w.hist_index = j; w.chunk_begin = cb; hist_work[j] = w; }
  }
  if (threadIdx.x == 0) {
    ctl_nxt->hist_n_work = ns; ctl_nxt->hist_total_chunks = carry; ctl_nxt->hist_chunk_rows = chunk_rows;
    ctl_nxt->n_pairs = ns;
  }
}

}  // namespace b2
