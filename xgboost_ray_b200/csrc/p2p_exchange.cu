// p2p_exchange.cu -- histogram exchange fused with the sibling subtraction over NVLink peer memory.
//
// Replaces, for one tree level, what the reference gets from Rabit's allreduce inside xgb.train()
// (xgboost_ray/main.py:745-752; SURVEY.md 8a row a11, 8e) and what the NCCL path of this engine does with
// ncclReduceScatter + hist_subtract_kernel: ONE kernel
//   1. publishes "my partial histograms of this level are complete" to every rank (epoch flag, p2p.cuh),
//   2. waits for the same flag of every rank,
//   3. sums the W partial copies of the feature-slot slice this rank owns straight out of the peers' memory
//      (exact int64, so the order of ranks does not matter), stores the built child's slice into the level buffer and
//   4. derives the sibling's slice  parent - built  in the same pass (the parent level is local).
// The split candidates travel the other way: decide_kernel (control_kernel.cu) stores this rank's candidates into
// every peer's table before it decides.  No NCCL call is left inside a tree.
#include "p2p.cuh"
#include "launch.h"

namespace b2 {

// grid = (x, n_pairs upper bound); pair p: triples[3p] = parent slot (previous level buffer), [3p+1] = built slot,
// [3p+2] = sibling slot (this level buffer).  triples == nullptr: the root (one node, nothing to subtract).
__global__ void __launch_bounds__(256)
p2p_reduce_subtract_kernel(B2P2P pp, const long long* __restrict__ parent_level, long long* __restrict__ level,
                           const int32_t* __restrict__ triples, const B2LevelCtl* __restrict__ ctl, int node_cap,
                           int64_t slice_elems) {
  const uint32_t epoch = p2p_next_epoch(pp, kSlotHist);
  const unsigned n_ctas = gridDim.x * gridDim.y;
  if (blockIdx.x == 0 && blockIdx.y == 0) p2p_signal(pp, kSlotHist, epoch);
  const int n_pairs = triples ? ctl->n_pairs : 1;
  const int p = blockIdx.y;
  if (p < n_pairs) {
    p2p_wait(pp, kSlotHist, epoch);
    const int par_slot = triples ? triples[3 * p] : 0, built_slot = triples ? triples[3 * p + 1] : 0;
    const int sib_slot = triples ? triples[3 * p + 2] : 0;
    const size_t src = ((size_t)pp.rank * node_cap + built_slot) * (size_t)slice_elems;
    long long* built = level + (size_t)built_slot * slice_elems;
    long long* sib = level + (size_t)sib_slot * slice_elems;
    const long long* par = parent_level + (size_t)par_slot * slice_elems;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 2; i < slice_elems; i += (int64_t)gridDim.x * blockDim.x * 2) {
      unsigned long long a = 0, b = 0;
      for (int w = 0; w < pp.world; ++w) {
        const ulonglong2 v = ld_volatile_v2(pp.build[w] + src + i);
        a += v.x; b += v.y;
      }
      built[i] = (long long)a; built[i + 1] = (long long)b;
      if (triples) { sib[i] = par[i] - (long long)a; sib[i + 1] = par[i + 1] - (long long)b; }
    }
  }
  p2p_finish_grid(pp, kSlotHist, epoch, n_ctas);
}

// per-tree fixed-point scale: every rank stores its max|g|, max|h| bit patterns into every rank's misc table, then
// takes the maximum over the ranks (replaces ncclAllReduce(max) + quant_exponent_kernel)
__global__ void p2p_quant_exponent_kernel(B2P2P pp, const uint32_t* __restrict__ absmax, int32_t* __restrict__ qexp) {
  const uint32_t epoch = p2p_next_epoch(pp, kSlotAbsmax);
  if ((int)threadIdx.x < pp.world) {
    const long long v = (long long)(((unsigned long long)absmax[1] << 32) | (unsigned long long)absmax[0]);
    st_volatile_u64(pp.misc[threadIdx.x] + (size_t)pp.rank * pp.misc_stride, v);
  }
  __syncthreads();
  p2p_signal(pp, kSlotAbsmax, epoch);
  p2p_wait(pp, kSlotAbsmax, epoch);
  if (threadIdx.x == 0) {
    uint32_t mg = 0, mh = 0;
    for (int w = 0; w < pp.world; ++w) {
      const unsigned long long v = ld_volatile_u64(pp.misc[pp.rank] + (size_t)w * pp.misc_stride);
      const uint32_t g = (uint32_t)(v & 0xffffffffu), h = (uint32_t)(v >> 32);
      mg = g > mg ? g : mg; mh = h > mh ? h : mh;
    }
    qexp[0] = b2_frexp_exponent(mg);
    qexp[1] = b2_frexp_exponent(mh);
  }
  __syncthreads();
  p2p_finish_single(pp, kSlotAbsmax, epoch);
}

// leaf sums: every rank stores its [n_leaves][g, h][hi, lo] int64 limbs (common.cuh) into every rank's misc table
// (offset 2), then replaces its local limbs with the total over the ranks (replaces ncclAllReduce(sum) in front of
// leaf_values_kernel).  Limbs add limb by limb without wrapping, so the total is exact below 2^31 rows over all ranks.
__global__ void __launch_bounds__(1024)
p2p_leaf_sums_kernel(B2P2P pp, const int32_t* __restrict__ n_leaves, long long* __restrict__ sums) {
  const uint32_t epoch = p2p_next_epoch(pp, kSlotLeaf);
  const int n = 4 * *n_leaves;
  for (int w = 0; w < pp.world; ++w)
    for (int i = threadIdx.x; i < n; i += blockDim.x) st_volatile_u64(pp.misc[w] + (size_t)pp.rank * pp.misc_stride + 2 + i, sums[i]);
  __syncthreads();
  p2p_signal(pp, kSlotLeaf, epoch);
  p2p_wait(pp, kSlotLeaf, epoch);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    unsigned long long t = 0;
    for (int w = 0; w < pp.world; ++w) {
      t += ld_volatile_u64(pp.misc[pp.rank] + (size_t)w * pp.misc_stride + 2 + i);
    }
    sums[i] = (long long)t;
  }
  __syncthreads();
  p2p_finish_single(pp, kSlotLeaf, epoch);
}

// INTERLEAVED sharding without host-side amplification: every rank uploads ONE contiguous block of the driver's matrix
// (rows [start_w, start_w + count_w) on rank w, BATCH-style split) and then pulls the rows it owns -- global rows
// rank, rank + W, rank + 2W, ... -- out of the peers' blocks over NVLink.  One warp per row, coalesced float4 / float
// copies.
__global__ void __launch_bounds__(256)
gather_interleaved_rows_kernel(B2RowBlocks rb, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long j = warp; j < rb.n_mine; j += n_warps) {
    const long long i = rb.rank + j * rb.world;                 // global row
    int w = 0;
#pragma unroll
    for (int k = 1; k < B2_P2P_MAX_WORLD; ++k) if (k < rb.world && i >= rb.start[k]) w = k;
    const float* src = rb.base[w] + (i - rb.start[w]) * rb.n_cols;
    float* dst = out + j * rb.n_cols;
    for (int c = lane; c < rb.n_cols; c += 32) dst[c] = src[c];
  }
}

}  // namespace b2

extern "C" {
int b2_p2p_flag_words(int world) { return kP2PSlots * world; }
int b2_launch_p2p_reduce_subtract(const B2P2P* pp, const long long* parent_level, long long* level, const int32_t* triples,
                                  const B2LevelCtl* ctl, int max_pairs, int node_cap, int64_t slice_elems, int num_sms,
                                  cudaStream_t s) {
  if (max_pairs <= 0 || slice_elems <= 0) return 0;
  // enough CTAs to keep the NVLink reads of all peers in flight, few enough that the wait/finish overhead stays small
  int bx = (int)((slice_elems / 2 + 255) / 256);
  int cap = (4 * num_sms + max_pairs - 1) / max_pairs;
  if (cap < 1) cap = 1;
  if (bx > cap) bx = cap;
  if (bx < 1) bx = 1;
  dim3 grid(bx, max_pairs);
  b2::p2p_reduce_subtract_kernel<<<grid, 256, 0, s>>>(*pp, parent_level, level, triples, ctl, node_cap, slice_elems);
  return (int)cudaGetLastError();
}
int b2_launch_p2p_quant_exponent(const B2P2P* pp, const uint32_t* absmax, int32_t* qexp, cudaStream_t s) {
  b2::p2p_quant_exponent_kernel<<<1, 32, 0, s>>>(*pp, absmax, qexp);
  return (int)cudaGetLastError();
}
int b2_launch_p2p_leaf_sums(const B2P2P* pp, const int32_t* n_leaves, long long* sums, cudaStream_t s) {
  b2::p2p_leaf_sums_kernel<<<1, 1024, 0, s>>>(*pp, n_leaves, sums);
  return (int)cudaGetLastError();
}
int b2_launch_gather_interleaved_rows(const B2RowBlocks* blocks, float* out, int num_sms, cudaStream_t s) {
  const B2RowBlocks& rb = *blocks;
  if (rb.n_mine <= 0) return 0;
  long long want = (rb.n_mine * 32 + 255) / 256;
  int grid = (int)(want < (long long)num_sms * 16 ? want : (long long)num_sms * 16);
  b2::gather_interleaved_rows_kernel<<<grid, 256, 0, s>>>(rb, out);
  return (int)cudaGetLastError();
}
}
