// hist_common.cuh -- device helpers of the histogram kernels (hist_kernel.cu, hist_csr_kernel.cu): row loads, the
// conflict-free shared atomics and the flushes to the global int64 histogram.
#pragma once
#include "common.cuh"

namespace b2 {

// b2_launch_hist on the CSR bin layout (hist_csr_kernel.cu); totals: the [node_cap][2] scratch, zeroed here
int launch_hist_csr(const B2BinRows& src, const int32_t* group_size, const int2* gpair, const int32_t* ridx,
                    const B2HistWork* work, int n_work, int total_chunks, int chunk_rows, int n_groups, long long* hist,
                    long long* totals, const B2LevelCtl* ctl, int log2_shards, int node_cap, int num_sms, cudaStream_t stream);

__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void red_shared_add(uint32_t saddr, int v) {
  asm volatile("red.shared.add.s32 [%0], %1;" ::"r"(saddr), "r"(v) : "memory");
}

// result byte i = source byte (i + rot) & 15
__device__ __forceinline__ uint4 rotate_bytes(uint4 v, int rot) {
  uint32_t w0 = v.x, w1 = v.y, w2 = v.z, w3 = v.w;
  if (rot & 4) { uint32_t t = w0; w0 = w1; w1 = w2; w2 = w3; w3 = t; }
  if (rot & 8) { uint32_t t0 = w0, t1 = w1; w0 = w2; w1 = w3; w2 = t0; w3 = t1; }
  int bs = (rot & 3) * 8;
  uint4 r;
  r.x = __funnelshift_r(w0, w1, bs);
  r.y = __funnelshift_r(w1, w2, bs);
  r.z = __funnelshift_r(w2, w3, bs);
  r.w = __funnelshift_r(w3, w0, bs);
  return r;
}

struct RowData {
  uint4 bins;
  int2 gp;
};

// row id of chunk-row r (or -1 past the end of the chunk); root level: identity
template <bool kGather>
__device__ __forceinline__ int64_t fetch_rid(const int32_t* __restrict__ ridx, int64_t pos0, int r, int nrows) {
  if (r >= nrows) return -1;
  return kGather ? (int64_t)__ldg(ridx + pos0 + r) : pos0 + r;
}
__device__ __forceinline__ RowData load_row_id(const uint8_t* __restrict__ bins, const int2* __restrict__ gpair,
                                               int64_t rid, int row_stride, int lane_byte_off) {
  RowData d;
  d.bins = make_uint4(0, 0, 0, 0);
  d.gp = make_int2(0, 0);
  if (rid >= 0) {
    d.bins = ldg_nc_v4(bins + rid * row_stride + lane_byte_off);
    d.gp = __ldg(gpair + rid);
  }
  return d;
}

// 16 steps: one byte (= one feature slot) per step, two conflict-free shared atomics per step.
// Shared layout: int32 [256 bins][2 planes (g,h)][32 slots] = 256 B per bin, so bin*256 is the byte
// placed at byte position 1 by ONE prmt; the cell address is that plus a per-lane, per-step offset.
__device__ __forceinline__ void accumulate_row(const RowData& d, uint32_t smem_g, int rot, int half) {
  uint4 b = rotate_bytes(d.bins, rot);
  const uint32_t w[4] = {b.x, b.y, b.z, b.w};
  const uint32_t base = smem_g + half * 64;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const uint32_t bin256 = __byte_perm(w[j >> 2], 0u, 0x4404u | ((uint32_t)(j & 3) << 4));
    const uint32_t slot_off = ((uint32_t)(j + rot) & 15u) * 4u;
    const uint32_t a = base + bin256 + slot_off;
    red_shared_add(a, d.gp.x);
    red_shared_add(a + B2_GROUP_SLOTS * 4, d.gp.y);
  }
}

// shared cell e = bin*64 + plane*32 + slot  ->  global cell plane*8192 + bin*32 + slot
// Global histogram layout (feature-slot sharded for the reduce-scatter, DESIGN.md 5):
//   int64 [shards][node_cap][group][plane][256 bins][sp]   sp = 32 / shards, slot s lives on shard s % shards at s / shards.
// shards == 1 degenerates to [node][group][plane][bin][32].
struct HistTarget {
  unsigned long long* base;   // build buffer
  int log2_shards;            // shards = 1 << log2_shards
  int node_cap;               // node slots per shard in this launch's buffer
  int n_groups;
};
__device__ __forceinline__ size_t target_index(const HistTarget& t, int node_slot, int group, int e) {
  const int bin = e >> 6, plane = (e >> 5) & 1, slot = e & 31;
  const int shards = 1 << t.log2_shards, sp = B2_GROUP_SLOTS >> t.log2_shards;
  const int r = slot & (shards - 1), sl = slot >> t.log2_shards;
  const size_t slice_elems = (size_t)t.n_groups * 2 * B2_BINS * sp;
  return ((size_t)r * t.node_cap + node_slot) * slice_elems + ((size_t)(group * 2 + plane) * B2_BINS + bin) * sp + sl;
}

// lazy window flush: only cells whose magnitude reached 2^30 are moved to the global histogram.  Called
// (between barriers) at least every `window_rows` = 2^(30 - qbits) rows, during which a cell can grow by
// less than 2^30, so no int32 cell can overflow; for well spread bins nothing is flushed at all.
__device__ __forceinline__ void flush_large_cells(int32_t* s_hist, const HistTarget& t, int node_slot, int group) {
  for (int e = threadIdx.x * 4; e < B2_GROUP_ELEMS; e += blockDim.x * 4) {
    const int4 v = *reinterpret_cast<const int4*>(s_hist + e);
    const int vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (vv[k] >= (1 << 30) || vv[k] <= -(1 << 30)) {
        atomicAdd(t.base + target_index(t, node_slot, group, e + k), (unsigned long long)(long long)vv[k]);
        s_hist[e + k] = 0;
      }
    }
  }
}
// node flush: shared int32 partial sums -> global int64 histogram (RED.64), cells are left zeroed
__device__ __forceinline__ void flush_planes(int32_t* s_hist, const HistTarget& t, int node_slot, int group) {
  for (int e = threadIdx.x; e < B2_GROUP_ELEMS; e += blockDim.x) {
    const long long v = s_hist[e];
    if (v != 0) { atomicAdd(t.base + target_index(t, node_slot, group, e), (unsigned long long)v); s_hist[e] = 0; }
  }
}

}  // namespace b2
