// hist_csr_kernel.cu -- level histograms from the CSR bin layout (one bin per stored entry; DESIGN.md 2 item 26).
//
// The result is the int64 histogram hist_kernel.cu builds from the dense bins of the same matrix, cell for cell:
//  * hist_csr_build_kernel: every stored entry whose bin is below 255 adds its row's (qg, qh) to its (feature, bin)
//    cell with a global 64-bit atomic (a node of a wide matrix holds far more cells than shared memory), and every row
//    adds its pair to the node's total.  No int32 cell, so no overflow window.
//  * hist_csr_missing_kernel: bin 255 of a feature is the node's total minus the feature's bins 0..254.  In the dense
//    matrix every row has exactly one bin per feature, so this is what the dense kernel accumulates there: the rows
//    whose bin is the missing sentinel -- absent entries, stored NaN and stored `missing` -- or, for a column stored in
//    every row without a missing value, the rows whose real bin is 255.  An entry that binned to 255 is therefore never
//    added by the build kernel, and nothing is counted twice.  A padding slot of a group holds bin 0 in every dense row,
//    so its bin 0 is the node's total.
// The sums are exact integers, so the order of rows, CTAs and GPUs does not matter: the totals are per GPU, and the
// exchange adds the GPUs' histograms as it adds the dense ones.
#include "hist_common.cuh"

namespace b2 {

constexpr int kCsrHistThreads = 256;

// rows of a chunk: one thread per row, walking the row's stored entries
template <bool kGather>
__global__ void __launch_bounds__(kCsrHistThreads)
hist_csr_build_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const uint8_t* __restrict__ ebins,
                      const int32_t* __restrict__ feat_byte, const int2* __restrict__ gpair, const int32_t* __restrict__ ridx,
                      const B2HistWork* __restrict__ work, int n_work, int total_chunks, int chunk_rows, int n_groups,
                      long long* __restrict__ hist, long long* __restrict__ totals, const B2LevelCtl* __restrict__ ctl,
                      int log2_shards, int node_cap) {
  HistTarget target; target.base = (unsigned long long*)hist; target.log2_shards = log2_shards; target.node_cap = node_cap;
  target.n_groups = n_groups;
  if (ctl) { n_work = ctl->hist_n_work; total_chunks = ctl->hist_total_chunks; chunk_rows = ctl->hist_chunk_rows; }
  const int lane = threadIdx.x & 31;
  for (int chunk = blockIdx.x; chunk < total_chunks; chunk += gridDim.x) {
    int lo = 0, hi = n_work - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(&work[mid].chunk_begin) <= chunk) lo = mid; else hi = mid - 1;
    }
    const int seg_begin = __ldg(&work[lo].seg_begin), seg_count = __ldg(&work[lo].seg_count);
    const int node = __ldg(&work[lo].hist_index);
    const int row0 = (chunk - __ldg(&work[lo].chunk_begin)) * chunk_rows;
    const int nrows = min(chunk_rows, seg_count - row0);
    long long tg = 0, th = 0;
    for (int r = threadIdx.x; r < nrows; r += blockDim.x) {
      const int64_t p = (int64_t)seg_begin + row0 + r;
      const int64_t row = kGather ? (int64_t)__ldg(ridx + p) : p;
      const int2 gp = __ldg(gpair + row);
      tg += gp.x; th += gp.y;
      const int64_t e1 = __ldg(indptr + row + 1);
      for (int64_t e = __ldg(indptr + row); e < e1; ++e) {
        const int b = __ldg(ebins + e);
        if (b == B2_MISSING_BIN) continue;
        const int fb = __ldg(feat_byte + __ldg(indices + e));
        const int e_g = (b << 6) | (fb & 31);   // shared-cell numbering of hist_common.cuh: bin * 64 + plane * 32 + slot
        atomicAdd(target.base + target_index(target, node, fb >> 5, e_g), (unsigned long long)(long long)gp.x);
        atomicAdd(target.base + target_index(target, node, fb >> 5, e_g | 32), (unsigned long long)(long long)gp.y);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { tg += __shfl_xor_sync(0xffffffffu, tg, o); th += __shfl_xor_sync(0xffffffffu, th, o); }
    if (lane == 0 && (tg != 0 || th != 0)) {
      atomicAdd((unsigned long long*)totals + 2 * node, (unsigned long long)tg);
      atomicAdd((unsigned long long*)totals + 2 * node + 1, (unsigned long long)th);
    }
  }
}

// CTA (group, work item): 256 threads = 4 bin quarters x (2 planes x 32 slots)
__global__ void __launch_bounds__(256)
hist_csr_missing_kernel(const B2HistWork* __restrict__ work, int n_work, const int32_t* __restrict__ group_size, int n_groups,
                        long long* __restrict__ hist, const long long* __restrict__ totals, const B2LevelCtl* __restrict__ ctl,
                        int log2_shards, int node_cap) {
  HistTarget target; target.base = (unsigned long long*)hist; target.log2_shards = log2_shards; target.node_cap = node_cap;
  target.n_groups = n_groups;
  if (ctl) n_work = ctl->hist_n_work;
  const int w = blockIdx.y, group = blockIdx.x;
  if (w >= n_work) return;
  const int node = __ldg(&work[w].hist_index);
  const int ps = threadIdx.x & 63, quarter = threadIdx.x >> 6;   // ps = plane * 32 + slot
  __shared__ long long s_sum[4][64];
  long long sum = 0;
  const int b_end = quarter == 3 ? 255 : (quarter + 1) * 64;
  for (int b = quarter * 64; b < b_end; ++b) sum += (long long)target.base[target_index(target, node, group, (b << 6) | ps)];
  s_sum[quarter][ps] = sum;
  __syncthreads();
  if (threadIdx.x >= 64) return;
  const long long t = totals[2 * node + (ps >> 5)];
  const bool real = (ps & 31) < __ldg(group_size + group);
  const long long rest = s_sum[0][ps] + s_sum[1][ps] + s_sum[2][ps] + s_sum[3][ps];
  unsigned long long* cell = target.base + target_index(target, node, group, real ? ((B2_MISSING_BIN << 6) | ps) : ps);
  *cell = (unsigned long long)((long long)*cell + (real ? t - rest : t));
}

int launch_hist_csr(const B2BinRows& src, const int32_t* group_size, const int2* gpair, const int32_t* ridx,
                    const B2HistWork* work, int n_work, int total_chunks, int chunk_rows, int n_groups, long long* hist,
                    long long* totals, const B2LevelCtl* ctl, int log2_shards, int node_cap, int num_sms, cudaStream_t stream) {
  if (!ctl && (total_chunks <= 0 || n_work <= 0)) return 0;
  const cudaError_t e = cudaMemsetAsync(totals, 0, 2 * (size_t)node_cap * sizeof(long long), stream);
  if (e != cudaSuccess) return (int)e;
  int grid = num_sms * 8;
  if (!ctl && grid > total_chunks) grid = total_chunks;
  if (ridx) hist_csr_build_kernel<true><<<grid, kCsrHistThreads, 0, stream>>>(
      src.indptr, src.indices, src.ebins, src.feat_byte, gpair, ridx, work, n_work, total_chunks, chunk_rows, n_groups, hist,
      totals, ctl, log2_shards, node_cap);
  else hist_csr_build_kernel<false><<<grid, kCsrHistThreads, 0, stream>>>(
      src.indptr, src.indices, src.ebins, src.feat_byte, gpair, ridx, work, n_work, total_chunks, chunk_rows, n_groups, hist,
      totals, ctl, log2_shards, node_cap);
  const int nodes = ctl ? node_cap : n_work;
  hist_csr_missing_kernel<<<dim3(n_groups, nodes), 256, 0, stream>>>(work, n_work, group_size, n_groups, hist, totals, ctl,
                                                                     log2_shards, node_cap);
  return (int)cudaGetLastError();
}

}  // namespace b2
