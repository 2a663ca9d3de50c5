// engine.cu -- host side of libb2hist.so: C-ABI (include/b2hist.h), device memory, level loop,
// NCCL communicator.  One process drives one GPU (one Ray actor per GPU in the reference,
// xgboost_ray/main.py:862-892); row-sharded data parallel, model replicated, per-level
// histogram allreduce (SURVEY.md 8e).
//
// Mirrors, for the hot path only, what `xgboost` does underneath xgboost_ray/main.py:745-752:
//   gradient -> [per class tree] quantise -> root hist -> allreduce -> eval -> partition ->
//   smaller-child hist -> allreduce -> sibling subtraction -> ... -> leaf sums -> margin update.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <errno.h>
#include <sys/types.h>
#include <sys/uio.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <thread>
#include <vector>

#include "../../include/b2hist.h"
#include "common.cuh"
#include "sampling.cuh"

// ---------------------------------------------------------------- kernel launchers (other TUs)
extern "C" {
int b2_launch_hist(const uint8_t*, int, const int2*, const int32_t*, const B2HistWork*, int, int, int, int, int, long long*,
                   const B2LevelCtl*, int, int, int, int, cudaStream_t);
int b2_make_bins_tensor_map(void*, const uint8_t*, int64_t, int, int);
int b2_launch_hist_tma(const uint8_t*, int, const void*, const int2*, const int32_t*, const B2HistWork*, int, int, int, int, int, long long*,
                       const B2LevelCtl*, int, int, int64_t, int, cudaStream_t);
int b2_launch_hist_subtract(const long long*, long long*, const int32_t*, int, int64_t, const B2LevelCtl*, cudaStream_t);
int b2_launch_eval_splits(const long long*, int, const B2EvalNode*, int, const int32_t*, const int32_t*, const int32_t*,
                          const uint8_t*, const uint8_t*, const int32_t*, int, B2TrainParamDev, B2SplitCand*, int, const B2LevelCtl*,
                          int, int, B2ColSample, const B2NodeSeg*, B2SiblingSub, const B2DecideArgs*, uint32_t*, cudaStream_t);
int b2_eval_ctas_per_node(int, int, int);
int b2_eval_narrow_max_nodes();
int b2_launch_subsample(float2*, int64_t, uint32_t, uint32_t, uint32_t, double, int, cudaStream_t);
int b2_p2p_flag_words(int);
int b2_launch_p2p_reduce_subtract(const void*, const long long*, long long*, const int32_t*, const B2LevelCtl*, int, int, int64_t, int,
                                  cudaStream_t);
int b2_launch_p2p_quant_exponent(const void*, const uint32_t*, int32_t*, cudaStream_t);
int b2_launch_p2p_leaf_sums(const void*, const int32_t*, long long*, cudaStream_t);
int b2_hist_variant();
int b2_launch_p2p_close(const void*, cudaStream_t);
int b2_launch_gather_interleaved_rows(const void*, float*, int, cudaStream_t);
int b2_launch_final_assign(const uint8_t*, int64_t, const int32_t*, const B2SplitWork*, const B2LevelCtl*, int, const float2*,
                           const int32_t*, int, long long*, uint16_t*, int, int, cudaStream_t);
int b2_launch_margin_update(float*, int, int, const uint16_t*, const float*, int64_t, int, cudaStream_t);
int b2_leaf_acc_max_depth();
int b2_launch_leaf_accumulate(const float2*, const uint16_t*, int64_t, int, const int32_t*, int, long long*, int, cudaStream_t);
int b2_gradient_fused_max_classes();
int b2_launch_sum_fixed(const float2*, int64_t, const int32_t*, int, long long*, int, cudaStream_t);
int b2_cat_ctas();
int b2_launch_eval_cat_splits(const long long*, int, const B2EvalNode*, int, const int32_t*, int, const int32_t*, const int32_t*,
                              const int32_t*, int, B2TrainParamDev, B2SplitCand*, int, int, const B2LevelCtl*, int, int,
                              B2ColSample, const B2NodeSeg*, cudaStream_t);
int b2_launch_cat_stats(const float*, int64_t, int, float, const int32_t*, int, int32_t*, int, cudaStream_t);
int b2_launch_root_totals(const long long*, int, B2EvalNode*, const int32_t*, int, B2TrainParamDev, int, long long*, long long*,
                          cudaStream_t);
int b2_part_chunk_rows();
int b2_split_chunk_rows();
int b2_launch_partition(const uint8_t*, int64_t, const int32_t*, int32_t*, const B2SplitWork*, const B2LevelCtl*, int, int32_t*,
                        int, B2FinalizeArgs, int, cudaStream_t);
int b2_launch_leaf_sums(const float2*, const int32_t*, const int32_t*, const void*, const B2LevelCtl*, int, const int32_t*, int,
                        long long*, uint16_t*, int, cudaStream_t);
int b2_launch_pred_update(float*, int, int, const int32_t*, const int32_t*, const void*, const B2LevelCtl*, int, const float*, int,
                          cudaStream_t);
int b2_launch_decide(const B2DecideArgs*, const void*, cudaStream_t);
int b2_launch_leaf_plan(const B2LeafDev*, const int32_t*, B2SegWork*, B2LevelCtl*, cudaStream_t);
int b2_launch_leaf_values(const B2LeafDev*, const int32_t*, const long long*, const int32_t*, int, B2CtlParams, float*, B2TreeDev,
                          int32_t*, cudaStream_t);
int b2_launch_tree_init(B2TreeDev, B2LevelCtl*, B2NodeSeg*, B2EvalNode*, int32_t*, int, B2HistWork*, cudaStream_t);
int b2_launch_iota(int32_t*, int64_t, cudaStream_t);
int b2_launch_gradient(int, int, const float*, const float*, const float*, int64_t, float, float, float2*, uint32_t*, uint32_t*, int,
                       cudaStream_t);
int b2_launch_label_check(int, int, const float*, int64_t, uint32_t*, int, cudaStream_t);
int b2_launch_gradient_aft(int, double, const float*, const float*, const float*, const float*, int64_t, float2*, uint32_t*,
                           uint32_t*, int, cudaStream_t);
int b2_launch_aft_bounds_check(const float*, const float*, int64_t, uint32_t*, int, cudaStream_t);
int b2_launch_aft_metric(int, int, double, const float*, const float*, const float*, const float*, int64_t, double*, int,
                         cudaStream_t);
int b2_launch_pack_custom(const float*, const float*, int, int64_t, float2*, int, cudaStream_t);
int b2_launch_absmax(const float2*, int64_t, uint32_t*, int, cudaStream_t);
int b2_launch_quant_exponent(const uint32_t*, int32_t*, cudaStream_t);
int b2_launch_quantize(const float2*, int64_t, const int32_t*, int, int2*, int, cudaStream_t);
int b2_launch_metric(int, int, int, float, const float*, const float*, const float*, int64_t, double*, int, cudaStream_t);
int b2_launch_predict(const float*, int64_t, int, float, const B2TreeNodeDev*, const int32_t*, const uint32_t*, int, int, int, int,
                      float*, int, cudaStream_t);
int b2_launch_fill(float*, int64_t, float, int, cudaStream_t);
size_t b2_shap_contribs_smem(int, int, int);
int b2_launch_shap_contribs(const float*, int64_t, int64_t, int, float, const B2PathElem*, const B2PathInfo*, int, int,
                            const uint32_t*, int, const double*, const float*, float, double*, int, size_t, float*, int, cudaStream_t);
int b2_launch_shap_interactions(const float*, int64_t, int64_t, int, float, const B2PathElem*, const B2PathInfo*, int, int,
                                const uint32_t*, int, const double*, const float*, float, double*, float*, int, cudaStream_t);
int b2_launch_leaf_index(const float*, int64_t, int64_t, int, float, const B2TreeNodeDev*, const int32_t*, const uint32_t*, int, int,
                         float*, int, cudaStream_t);
int b2_rank_stage_rows();
size_t b2_rank_order_temp_bytes(int64_t, int64_t);
int b2_launch_rank_iota(int32_t*, int64_t, int, cudaStream_t);
int b2_rank_order(const float*, int64_t, const int64_t*, int64_t, const int32_t*, uint32_t*, uint32_t*, int32_t*, void*, size_t,
                  int, cudaStream_t);
int b2_launch_rank_disc(double*, int64_t, int, cudaStream_t);
int b2_launch_rank_inv_idcg(const int64_t*, int64_t, const uint32_t*, const double*, int, int, double*, int, cudaStream_t);
int b2_launch_rank_label_check(const float*, int64_t, int, uint32_t*, int, cudaStream_t);
int b2_launch_lambdarank_gradient(int, const int64_t*, int64_t, int64_t, const uint32_t*, const int32_t*, const float*,
                                  const double*, const double*, int, int, float*, float*, double*, float2*, uint32_t*, uint32_t*,
                                  int, cudaStream_t);
int b2_launch_rank_metric(int, int, int, int, const int64_t*, int64_t, const int32_t*, const float*, const uint32_t*,
                          const double*, double*, double*, int, cudaStream_t);
size_t b2_auc_temp_bytes(int64_t);
int b2_auc_binary(const float*, const float*, const float*, int64_t, void*, size_t, double*, int, cudaStream_t);
int b2_launch_transform(int, int, float*, int64_t, int, cudaStream_t);
int b2_extract_batch();
int b2_launch_extract_keys(const float*, int64_t, int, int, int, float, uint32_t*, int64_t, int, cudaStream_t);
size_t b2_sort_temp_bytes(int64_t);
int b2_sketch_column(const uint32_t*, const int32_t*, uint32_t*, int32_t*, long long*, int64_t, long long, void*, size_t, int32_t*,
                     int32_t*, float*, long long*, int32_t*, long long*, int, float*, int32_t*, float*, int32_t*, int, cudaStream_t);
int b2_launch_weight_absmax(const float*, int64_t, uint32_t*, int, cudaStream_t);
int b2_launch_weight_quantize(const float*, int64_t, int64_t, const uint32_t*, int32_t*, int, cudaStream_t);
int b2_launch_bin(const float*, int64_t, int, float, const int32_t*, const float*, const int32_t*, const uint8_t*, int, uint8_t*,
                  uint8_t*, int64_t, int, cudaStream_t);
}

namespace {

// ---------------------------------------------------------------- errors
thread_local std::string g_last_error;
struct B2Error { std::string msg; };
[[noreturn]] void fail(const char* fmt, ...) {
  char buf[1024];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
  throw B2Error{buf};
}
#define CUDA_CHECK(expr)                                                                       \
  do {                                                                                         \
    cudaError_t e_ = (expr);                                                                   \
    if (e_ != cudaSuccess) fail("CUDA error %s at %s:%d: %s", cudaGetErrorName(e_), __FILE__, __LINE__, cudaGetErrorString(e_)); \
  } while (0)
#define LAUNCH_CHECK(expr)                                                                     \
  do {                                                                                         \
    int e_ = (expr);                                                                           \
    if (e_ != 0) fail("kernel launch failed (%s) at %s:%d", cudaGetErrorString((cudaError_t)e_), __FILE__, __LINE__); \
  } while (0)
#define API_BEGIN try {
#define API_END                                            \
  }                                                        \
  catch (const B2Error& e) { g_last_error = e.msg; return -1; } \
  catch (const std::exception& e) { g_last_error = e.what(); return -1; } \
  return 0;

// ---------------------------------------------------------------- device context
struct Ctx {
  int device = -1;
  cudaStream_t stream = nullptr;
  int num_sms = 0;
};
std::mutex g_ctx_mu;
std::map<int, Ctx*> g_ctx;
Ctx* get_ctx(int device) {
  std::lock_guard<std::mutex> lk(g_ctx_mu);
  auto it = g_ctx.find(device);
  if (it != g_ctx.end()) { CUDA_CHECK(cudaSetDevice(device)); return it->second; }
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) fail("no CUDA device available (%s): libb2hist has no CPU fallback", cudaGetErrorString(e));
  if (device < 0 || device >= n) fail("invalid device %d (have %d)", device, n);
  CUDA_CHECK(cudaSetDevice(device));
  Ctx* c = new Ctx();
  c->device = device;
  CUDA_CHECK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  cudaDeviceProp prop;
  CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)   // sm_90a code loads on compute capability 9.0 only
    fail("device %d is sm_%d%d; this engine is built for sm_90a (H100) only", device, prop.major, prop.minor);
  c->num_sms = prop.multiProcessorCount;
  g_ctx[device] = c;
  return c;
}

// Device memory goes through a small caching pool: matrices and boosters allocate and free the same few large blocks
// over and over (every DMatrix, every sketch), cudaFree synchronises the device, and once a peer's buffers are mapped
// for the NVLink exchange every cudaMalloc also has to be mapped into the peers (measured: the second quantisation of
// a bench run took 0.28 s with peer mappings against 0.06 s without).  Freed blocks are kept per device and handed out
// again when their size fits (<= 25 % + 1 MiB slack); the cache is bounded by B2_POOL_MAX_GB (default 24, under a third
// of an 80 GB H100) and emptied when an allocation fails.
struct DevPool {
  std::mutex mu;
  std::multimap<size_t, void*> free_blocks;
  size_t cached = 0;
};
DevPool g_dev_pool[64];
size_t pool_cap_bytes() {
  static size_t cap = 0;
  if (!cap) { const char* e = getenv("B2_POOL_MAX_GB"); double gb = e ? atof(e) : 24.0; cap = (size_t)(gb < 0 ? 0 : gb * 1e9) + 1; }
  return cap;
}
void pool_trim(DevPool& pool, size_t keep) {   // caller holds pool.mu
  while (pool.cached > keep && !pool.free_blocks.empty()) {
    auto it = std::prev(pool.free_blocks.end());   // largest first
    cudaFree(it->second);
    pool.cached -= it->first;
    pool.free_blocks.erase(it);
  }
}
void* pool_alloc(size_t bytes, size_t* got, int* dev_out) {
  int dev = 0; cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  *dev_out = dev;
  bytes = (bytes + 511) & ~(size_t)511;
  DevPool& pool = g_dev_pool[dev];
  {
    std::lock_guard<std::mutex> lk(pool.mu);
    auto it = pool.free_blocks.lower_bound(bytes);
    if (it != pool.free_blocks.end() && it->first <= bytes + bytes / 4 + ((size_t)1 << 20)) {
      void* p = it->second; *got = it->first;
      pool.cached -= it->first;
      pool.free_blocks.erase(it);
      return p;
    }
  }
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) {   // out of memory: give the cached blocks back and try once more
    cudaGetLastError();
    { std::lock_guard<std::mutex> lk(pool.mu); pool_trim(pool, 0); }
    e = cudaMalloc(&p, bytes);
  }
  if (e != cudaSuccess) { cudaGetLastError(); fail("cudaMalloc of %zu bytes failed: %s", bytes, cudaGetErrorString(e)); }
  *got = bytes;
  return p;
}
void pool_free(void* p, size_t bytes, int dev) {
  if (!p) return;
  if (dev < 0 || dev >= 64) dev = 0;
  DevPool& pool = g_dev_pool[dev];
  std::lock_guard<std::mutex> lk(pool.mu);
  if (bytes > pool_cap_bytes()) { cudaFree(p); return; }
  pool.free_blocks.emplace(bytes, p);
  pool.cached += bytes;
  if (pool.cached > pool_cap_bytes()) pool_trim(pool, pool_cap_bytes() / 2);
}

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;          // elements the caller may use
  size_t block_bytes = 0;  // size of the pooled block behind p
  int dev = 0;
  void ensure(size_t n) {
    if (n <= cap) return;
    release();
    size_t got = 0;
    p = (T*)pool_alloc(n * sizeof(T), &got, &dev);
    block_bytes = got;
    cap = n;
  }
  void release() { if (p) pool_free(p, block_bytes, dev); p = nullptr; cap = 0; block_bytes = 0; }
  ~DevBuf() { release(); }
};

// ---------------------------------------------------------------- host -> device ingest
// Pageable host memory goes through the driver's single bounce buffer at ~10-13 GB/s.  Here T
// worker threads copy 16 MiB slices into their own pinned staging buffers and issue the DMA on
// their own streams, so host memcpy and PCIe transfers of different slices overlap (SURVEY.md 8f-3).
struct PinnedPool {
  static constexpr int kWorkers = 16, kSlots = 2;   // upper bound; B2_UPLOAD_WORKERS picks how many are used
  static constexpr size_t kSlice = (size_t)8 << 20;
  void* buf[kWorkers][kSlots] = {};
  cudaStream_t stream[kWorkers] = {};
  cudaEvent_t done[kWorkers][kSlots] = {};
  bool ready = false;
  std::mutex mu;
  int n_init = 0;
  void init(int n) {
    for (int w = n_init; w < n; ++w) {
      CUDA_CHECK(cudaStreamCreateWithFlags(&stream[w], cudaStreamNonBlocking));
      for (int k = 0; k < kSlots; ++k) {
        CUDA_CHECK(cudaMallocHost(&buf[w][k], kSlice));
        CUDA_CHECK(cudaEventCreateWithFlags(&done[w][k], cudaEventDisableTiming));
      }
      n_init = w + 1;
    }
  }
};
std::map<int, PinnedPool*> g_pools;

// Where the rows of an upload come from: this process (src) or ANOTHER process' memory (pid / remote_addr), row by row
// `row_stride` bytes apart -- the driver's matrix read with process_vm_readv straight into the pinned staging slices, so
// a shard never exists as a second host copy (matrix.py:471-484 puts every shard into the object store instead).
struct UploadSource {
  const void* src = nullptr;      // local, contiguous
  long long pid = 0;              // != 0: remote
  uint64_t remote_addr = 0;       // address of row 0 in process `pid`
  size_t row_bytes = 0, row_stride = 0;
};
// copy `len` bytes starting at byte offset `off` of the (virtually contiguous) source into dst; returns false on error
bool fetch_slice(const UploadSource& u, void* dst, size_t off, size_t len, std::string* err) {
  if (u.pid == 0) { memcpy(dst, (const char*)u.src + off, len); return true; }
  if (u.row_stride == u.row_bytes) {   // contiguous rows: one (or a few) big reads
    size_t done = 0;
    while (done < len) {
      struct iovec l = {(char*)dst + done, len - done}, r = {(void*)(uintptr_t)(u.remote_addr + off + done), len - done};
      const ssize_t got = process_vm_readv((pid_t)u.pid, &l, 1, &r, 1, 0);
      if (got <= 0) { if (err) *err = std::string("process_vm_readv: ") + strerror(errno); return false; }
      done += (size_t)got;
    }
    return true;
  }
  // strided rows (INTERLEAVED sharding: every W-th row of the driver's matrix).  One remote iovec per row costs the
  // kernel a page pin per 400-byte row (measured: 3 s for a 2 GB shard, 23 s with two actors contending); instead the
  // CONTIGUOUS span that covers a batch of rows is read with one iovec into a scratch buffer and the wanted rows are
  // picked out of it locally -- W times the bytes over the memory bus, two orders of magnitude fewer page pins.
  constexpr size_t kSpan = (size_t)4 << 20;
  static thread_local std::vector<char> scratch;
  if (scratch.size() < kSpan + u.row_stride) scratch.resize(kSpan + u.row_stride);
  const size_t rows_per_batch = std::max<size_t>(1, kSpan / u.row_stride);
  size_t done = 0;
  while (done < len) {
    const size_t pos = off + done, row0 = pos / u.row_bytes;
    const size_t last_byte = std::min(off + len, (row0 + rows_per_batch) * u.row_bytes) - 1;
    const size_t row1 = last_byte / u.row_bytes;                      // last row touched by this batch
    const size_t span = (row1 - row0) * u.row_stride + u.row_bytes;
    size_t got_total = 0;
    while (got_total < span) {
      struct iovec l = {scratch.data() + got_total, span - got_total};
      struct iovec r = {(void*)(uintptr_t)(u.remote_addr + row0 * u.row_stride + got_total), span - got_total};
      const ssize_t got = process_vm_readv((pid_t)u.pid, &l, 1, &r, 1, 0);
      if (got <= 0) { if (err) *err = std::string("process_vm_readv: ") + strerror(errno); return false; }
      got_total += (size_t)got;
    }
    for (size_t row = row0; row <= row1; ++row) {
      const size_t b0 = std::max(pos, row * u.row_bytes), b1 = std::min(off + len, (row + 1) * u.row_bytes);   // byte range of this row inside the slice
      memcpy((char*)dst + (b0 - off), scratch.data() + (row - row0) * u.row_stride + (b0 - row * u.row_bytes), b1 - b0);
    }
    done = std::min(off + len, (row1 + 1) * u.row_bytes) - off;
  }
  return true;
}

void upload_pipelined(Ctx* ctx, void* dst, const UploadSource& u, size_t bytes);
void upload_pipelined(Ctx* ctx, void* dst, const void* src, size_t bytes) {
  UploadSource u; u.src = src;
  upload_pipelined(ctx, dst, u, bytes);
}
void upload_pipelined(Ctx* ctx, void* dst, const UploadSource& u, size_t bytes) {
  const void* src = u.src;
  if (u.pid == 0 && bytes < ((size_t)64 << 20)) {
    if (bytes) CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return;
  }
  PinnedPool* pool;
  {
    std::lock_guard<std::mutex> lk(g_ctx_mu);
    PinnedPool*& p = g_pools[ctx->device];
    if (!p) p = new PinnedPool();
    pool = p;
  }
  std::lock_guard<std::mutex> lk(pool->mu);   // one bulk upload per device at a time
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));   // dst allocation / earlier work is complete
  const size_t n_slices = (bytes + PinnedPool::kSlice - 1) / PinnedPool::kSlice;
  static int n_workers = 0;
  if (n_workers == 0) {
    const char* e = getenv("B2_UPLOAD_WORKERS");
    n_workers = e ? atoi(e) : 8;
    if (n_workers < 1) n_workers = 1;
    if (n_workers > PinnedPool::kWorkers) n_workers = PinnedPool::kWorkers;
  }
  const int W = n_workers;
  pool->init(W);
  std::atomic<int> failed{0};
  std::mutex err_mu; std::string fetch_err;
  auto worker = [&](int w) {
    if (cudaSetDevice(ctx->device) != cudaSuccess) { failed = 1; return; }
    int use = 0;
    for (size_t i = w; i < n_slices; i += W, ++use) {
      const int k = use % PinnedPool::kSlots;
      const size_t off = i * PinnedPool::kSlice, len = std::min(PinnedPool::kSlice, bytes - off);
      if (use >= PinnedPool::kSlots && cudaEventSynchronize(pool->done[w][k]) != cudaSuccess) { failed = 1; return; }
      std::string e;
      if (!fetch_slice(u, pool->buf[w][k], off, len, &e)) { std::lock_guard<std::mutex> lk(err_mu); fetch_err = e; failed = 2; return; }
      if (cudaMemcpyAsync((char*)dst + off, pool->buf[w][k], len, cudaMemcpyHostToDevice, pool->stream[w]) != cudaSuccess ||
          cudaEventRecord(pool->done[w][k], pool->stream[w]) != cudaSuccess) { failed = 1; return; }
    }
    if (cudaStreamSynchronize(pool->stream[w]) != cudaSuccess) failed = 1;
  };
  std::vector<std::thread> th;
  for (int w = 0; w < W; ++w) th.emplace_back(worker, w);
  for (auto& t : th) t.join();
  if (failed.load() == 2) fail("reading the shard out of the driver process failed: %s", fetch_err.c_str());
  if (failed.load()) fail("pipelined host->device upload failed: %s", cudaGetErrorString(cudaGetLastError()));
}

// ---------------------------------------------------------------- NCCL (dlopen'ed)
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { kNcclSum = 0, kNcclMax = 2, kNcclMin = 3 };   // ncclRedOp_t
enum { kNcclUint8 = 1, kNcclInt32 = 2, kNcclUint32 = 3, kNcclInt64 = 4, kNcclUint64 = 5, kNcclFloat32 = 7, kNcclFloat64 = 8 };
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*ReduceScatter)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*CommAbort)(ncclComm_t) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
NcclApi* nccl() {
  static NcclApi api;
  static std::once_flag once;
  static std::string err;
  std::call_once(once, [] {
    const char* names[] = {"libnccl.so.2", "libnccl.so", "/usr/lib/x86_64-linux-gnu/libnccl.so.2"};
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);  // reuse torch's copy if loaded
    for (int i = 0; !h && i < 3; ++i) h = dlopen(names[i], RTLD_NOW | RTLD_GLOBAL);
    if (!h) { err = std::string("cannot load libnccl: ") + dlerror(); return; }
    api.lib = h;
#define LOAD(field, sym) *(void**)(&api.field) = dlsym(h, sym); if (!api.field) err = std::string("missing symbol ") + sym;
    LOAD(GetUniqueId, "ncclGetUniqueId") LOAD(CommInitRank, "ncclCommInitRank") LOAD(AllReduce, "ncclAllReduce")
    LOAD(AllGather, "ncclAllGather") LOAD(ReduceScatter, "ncclReduceScatter") LOAD(CommAbort, "ncclCommAbort") LOAD(CommDestroy, "ncclCommDestroy")
    LOAD(GetErrorString, "ncclGetErrorString")
#undef LOAD
  });
  if (!err.empty()) fail("%s", err.c_str());
  return &api;
}
#define NCCL_CHECK(expr)                                                                              \
  do {                                                                                                \
    int r_ = (expr);                                                                                  \
    if (r_ != 0) fail("NCCL error %d (%s) at %s:%d", r_, nccl()->GetErrorString(r_), __FILE__, __LINE__); \
  } while (0)

struct Comm {
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1, device = 0;
  std::atomic<bool> aborted{false};
  uint32_t* d_abort = nullptr;        // device word polled by the peer-memory waits (p2p.cuh); set by B2_CommAbort
  cudaStream_t abort_stream = nullptr;
};

void allreduce(Comm* c, void* buf, size_t count, int dtype, int op, cudaStream_t s) {
  if (!c || c->world <= 1 || count == 0) return;
  if (c->aborted.load()) fail("communicator aborted");
  NCCL_CHECK(nccl()->AllReduce(buf, buf, count, dtype, op, c->comm, s));
}

// ---------------------------------------------------------------- handles
enum HandleKind { kComm = 1, kMatrix = 2, kBooster = 3 };
struct HandleBase { int kind; };
template <typename T>
T* from_handle(B2Handle h, int kind, const char* what) {
  if (!h) fail("null %s handle", what);
  HandleBase* b = reinterpret_cast<HandleBase*>(h);
  if (b->kind != kind) fail("handle is not a %s", what);
  return reinterpret_cast<T*>(h);
}

struct CommH : HandleBase { Comm c; };

// ids of the matrices that are alive: a Booster's evaluation cache is keyed by the id, never by the address (a freed
// matrix and a new one of the same shape can share an address)
std::mutex g_matrix_mu;
std::set<uint64_t> g_live_matrices;
uint64_t g_next_matrix_uid = 1;

struct Matrix : HandleBase {
  uint64_t margin_version = 0;   // bumped when base_margin changes (cached evaluation margins start from it)
  uint64_t uid = 0;       // unique for the life of the process; 0 = not registered (stack temporaries)
  Ctx* ctx = nullptr;
  int64_t n = 0;
  int F = 0;
  float missing = NAN;
  DevBuf<float> raw;     // [n][F], optional
  bool has_raw = false;
  DevBuf<uint8_t> bins;  // [n][row_stride]
  alignas(64) unsigned char tmap_tile[128];   // TMA tensor map over bins, box {32 B, 64 rows}, for the contiguous root stage
  bool has_tmap = false;
  DevBuf<uint8_t> bins_col;  // [F][col_stride] feature-major copy for the row partition
  int64_t col_stride = 0;
  bool quantized = false;
  int n_groups = 0, row_stride = 0, max_bin = 0;
  int narrow_w = 0;                   // > 0: the last group is narrow (<= 16 features, width rounded up to a power of two)
  std::vector<int32_t> group_first, group_size, feat_byte;
  std::vector<int32_t> cut_ptrs;
  std::vector<float> cut_vals, min_vals;
  std::vector<uint8_t> has_missing;
  std::vector<int32_t> nbins;
  std::vector<uint8_t> is_cat;        // [F] 1 = categorical feature (B2_MatrixSetFeatureTypes); empty = all numeric
  std::vector<int32_t> cat_feats;     // ids of the categorical features
  DevBuf<int32_t> d_group_first, d_group_size, d_feat_byte, d_cut_ptrs, d_nbins, d_cat_feats;
  DevBuf<float> d_cut_vals;
  DevBuf<uint8_t> d_has_missing, d_is_cat;
  bool any_cat() const { return !cat_feats.empty(); }
  DevBuf<float> label, weight, base_margin;
  int64_t n_label = 0, n_weight = 0, n_base_margin = 0;
  DevBuf<float> lower, upper;          // survival label bounds (label_lower_bound / label_upper_bound), read by survival:aft
  int64_t n_lower = 0, n_upper = 0;
  bool has_bounds() const { return n_lower == n && n_upper == n; }
  // query groups (B2_MatrixSetGroups): group g is rows [qgroup_ptr[g], qgroup_ptr[g+1]); read by the rank objectives and
  // the ndcg / map / pre metrics.  rank_version changes with the groups and the labels (the 1/IDCG cache key)
  std::vector<int64_t> h_qgroup_ptr;
  DevBuf<int64_t> qgroup_ptr;
  int64_t n_qgroups = 0, max_qgroup = 0;
  uint64_t rank_version = 0;
  bool has_qgroups() const { return n_qgroups > 0; }
  std::vector<uint32_t> fwq;         // feature_weights in Q16 (empty = all 1.0)
  DevBuf<uint32_t> d_fwq;
};

// Feature -> (group, slot) layout of the bin matrix.  Default: the features are spread EVENLY over ceil(F / 32) groups, so
// that every CTA type of the histogram kernel (one pair of groups) costs the same and the types walk the chunk list in
// lock step -- the CTAs that read the two 64-byte halves of a row do it at the same time and the row is fetched from
// DRAM once.  B2_HIST_NARROW=1 selects the layout "a full groups + one NARROW group of the r = F mod 32 <= 16 leftover
// features" (one lane per row, pow2ceil(r) steps; hist_kernel.cu v3).  It removes the padding-slot atomics (F = 100:
// 6.25 instead of 8 wavefronts per row) but the CTA types then cost 4 : 2.25 and drift apart, so the two halves of a
// row are no longer read together and DRAM traffic grows.  Kept as an opt-in, parity-tested variant.
int g_hist_narrow = -1;   // -1: read B2_HIST_NARROW on first use; B2_SetOption("hist_narrow", ...) overrides it
void setup_groups(Matrix* m) {
  const int F = m->F;
  if (g_hist_narrow < 0) { const char* e = getenv("B2_HIST_NARROW"); g_hist_narrow = (e && atoi(e) != 0) ? 1 : 0; }
  const int narrow_on = g_hist_narrow;
  m->n_groups = (F + B2_GROUP_SLOTS - 1) / B2_GROUP_SLOTS;
  if (m->n_groups < 1) m->n_groups = 1;
  m->row_stride = m->n_groups * B2_GROUP_SLOTS;
  m->group_first.assign(m->n_groups, 0);
  m->group_size.assign(m->n_groups, 0);
  m->feat_byte.assign(F, 0);
  m->narrow_w = 0;
  const int r = F % B2_GROUP_SLOTS;
  // kernel v4 (all groups of a row in one CTA) wants three full groups + a narrow leftover group
  const bool v4_layout = b2_hist_variant() == 4 && F > 96 && F <= 112;
  const bool narrow = (narrow_on || v4_layout) && r > 0 && r <= 16;
  if (narrow) { m->narrow_w = 1; while (m->narrow_w < r) m->narrow_w <<= 1; }
  const int base = F / m->n_groups, rem = F % m->n_groups;
  int f = 0;
  for (int g = 0; g < m->n_groups; ++g) {
    const int sz = narrow ? (g + 1 < m->n_groups ? B2_GROUP_SLOTS : r) : base + (g < rem ? 1 : 0);
    m->group_first[g] = f; m->group_size[g] = sz;
    for (int s = 0; s < sz; ++s) m->feat_byte[f + s] = g * B2_GROUP_SLOTS + s;
    f += sz;
  }
}

template <typename T>
void upload(DevBuf<T>& d, const std::vector<T>& h, cudaStream_t s) {
  d.ensure(h.size() ? h.size() : 1);
  if (!h.empty()) CUDA_CHECK(cudaMemcpyAsync(d.p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, s));
}

void upload_cuts(Matrix* m) {
  cudaStream_t s = m->ctx->stream;
  m->nbins.resize(m->F);
  for (int f = 0; f < m->F; ++f) m->nbins[f] = m->cut_ptrs[f + 1] - m->cut_ptrs[f];
  upload(m->d_group_first, m->group_first, s); upload(m->d_group_size, m->group_size, s);
  upload(m->d_feat_byte, m->feat_byte, s); upload(m->d_cut_ptrs, m->cut_ptrs, s);
  upload(m->d_cut_vals, m->cut_vals, s); upload(m->d_nbins, m->nbins, s);
  upload(m->d_has_missing, m->has_missing, s);
  if (m->is_cat.empty()) m->is_cat.assign(m->F, 0);
  upload(m->d_is_cat, m->is_cat, s); upload(m->d_cat_feats, m->cat_feats, s);
  CUDA_CHECK(cudaStreamSynchronize(s));
}

// GPU sketch: exact global summary per feature -> cuts (sketch.cu).  No host round trip per feature.
// Multi-GPU: the column keys of every rank are allgathered (padded to the largest shard); feature f is
// sorted and pruned only by its owner rank f % world, and the cut tables are merged with one integer
// allreduce (non-owners contribute zeros), so every rank ends up with identical global cuts.
void make_cuts(Matrix* m, Comm* comm, int max_bin) {
  Ctx* ctx = m->ctx; cudaStream_t s = ctx->stream;
  if (max_bin < 2 || max_bin > 256) fail("max_bin must be in [2, 256] (uint8 bin matrix), got %d", max_bin);
  if (!m->has_raw) fail("matrix has no raw data to sketch");
  const int world = comm ? comm->world : 1, rank = comm ? comm->rank : 0;
  // largest shard and global row count
  DevBuf<long long> d_cnt; d_cnt.ensure(2);
  long long h_cnt[2] = {m->n, m->n};
  if (world > 1) {
    CUDA_CHECK(cudaMemcpyAsync(d_cnt.p, h_cnt, sizeof(h_cnt), cudaMemcpyHostToDevice, s));
    allreduce(comm, d_cnt.p, 1, kNcclInt64, kNcclMax, s);
    allreduce(comm, d_cnt.p + 1, 1, kNcclInt64, kNcclSum, s);
    CUDA_CHECK(cudaMemcpyAsync(h_cnt, d_cnt.p, sizeof(h_cnt), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
  }
  const int64_t n_pad = h_cnt[0], n_total = n_pad * world; const long long n_global = h_cnt[1];
  const int B = b2_extract_batch(); const int F = m->F;
  DevBuf<uint32_t> keys_local, keys_all, keys_sorted;
  DevBuf<int32_t> flags, idx, m_scratch; DevBuf<float> uval; DevBuf<long long> rmin, nvalid;
  DevBuf<int32_t> d_tab;   // [F*256 cut bits][F n_cuts][F min bits][F has_missing]
  DevBuf<uint8_t> temp;
  const size_t nt = (size_t)std::max<int64_t>(n_total, 1);
  keys_local.ensure((size_t)std::max<int64_t>(n_pad, 1) * B);
  if (world > 1) keys_all.ensure(nt);
  keys_sorted.ensure(nt); flags.ensure(nt); idx.ensure(nt); uval.ensure(nt); rmin.ensure(nt); m_scratch.ensure(1); nvalid.ensure(2);
  // sample weights make the sketch a weighted one (xgboost SketchContainer pushes info.weights_): quantise them to
  // integers with a global power-of-two scale so that the weighted ranks are exact and identical on every rank
  DevBuf<int32_t> wq_local, wq_all, wq_sorted; DevBuf<long long> wpre; DevBuf<uint32_t> d_wmax;
  const int32_t* wq = nullptr;
  {
    long long h_has[1] = {m->n_weight > 0 ? 1 : 0};
    if (world > 1) {   // a rank whose shard came without weights while others have them would desynchronise the collectives
      CUDA_CHECK(cudaMemcpyAsync(d_cnt.p, h_has, sizeof(h_has), cudaMemcpyHostToDevice, s));
      allreduce(comm, d_cnt.p, 1, kNcclInt64, kNcclMax, s);
      CUDA_CHECK(cudaMemcpyAsync(h_has, d_cnt.p, sizeof(h_has), cudaMemcpyDeviceToHost, s));
      CUDA_CHECK(cudaStreamSynchronize(s));
    }
    if (h_has[0]) {
      if (m->n_weight != m->n) fail("sample weights are set on some ranks only (this rank has %lld for %lld rows)", (long long)m->n_weight, (long long)m->n);
      d_wmax.ensure(2);
      CUDA_CHECK(cudaMemsetAsync(d_wmax.p, 0, 2 * sizeof(uint32_t), s));
      LAUNCH_CHECK(b2_launch_weight_absmax(m->weight.p, m->n, d_wmax.p, ctx->num_sms, s));
      allreduce(comm, d_wmax.p, 2, kNcclUint32, kNcclMax, s);
      uint32_t h_w[2];
      CUDA_CHECK(cudaMemcpyAsync(h_w, d_wmax.p, sizeof(h_w), cudaMemcpyDeviceToHost, s));
      CUDA_CHECK(cudaStreamSynchronize(s));
      if (h_w[1]) fail("sample weights must be finite and non-negative");
      wq_local.ensure((size_t)std::max<int64_t>(n_pad, 1));
      LAUNCH_CHECK(b2_launch_weight_quantize(m->weight.p, m->n, n_pad, d_wmax.p, wq_local.p, ctx->num_sms, s));
      wq = wq_local.p;
      if (world > 1) {
        wq_all.ensure(nt);
        NCCL_CHECK(nccl()->AllGather(wq_local.p, wq_all.p, (size_t)n_pad, kNcclInt32, comm->comm, s));
        wq = wq_all.p;
      }
      wq_sorted.ensure(nt); wpre.ensure(nt);
    }
  }
  const size_t temp_bytes = b2_sort_temp_bytes(n_total > 0 ? n_total : 1);
  temp.ensure(temp_bytes ? temp_bytes : 1);
  const size_t tab_n = (size_t)F * 256 + 3 * (size_t)F;
  d_tab.ensure(tab_n);
  CUDA_CHECK(cudaMemsetAsync(d_tab.p, 0, tab_n * sizeof(int32_t), s));
  float* d_cuts = (float*)d_tab.p; int32_t* d_ncuts = d_tab.p + (size_t)F * 256;
  float* d_mins = (float*)(d_ncuts + F); int32_t* d_hasmiss = d_ncuts + 2 * (size_t)F;
  if (m->is_cat.empty()) m->is_cat.assign(F, 0);
  for (int f0 = 0; f0 < F; f0 += B) {
    const int nf = std::min(B, F - f0);
    bool any_numeric = false;
    for (int j = 0; j < nf; ++j) any_numeric = any_numeric || !m->is_cat[f0 + j];
    if (!any_numeric) continue;
    LAUNCH_CHECK(b2_launch_extract_keys(m->raw.p, m->n, F, f0, nf, m->missing, keys_local.p, n_pad, ctx->num_sms, s));
    for (int j = 0; j < nf; ++j) {
      const int f = f0 + j;
      if (m->is_cat[f]) continue;   // categorical: cuts are the codes 0..max (below)
      const uint32_t* kin = keys_local.p + (size_t)j * n_pad;
      if (world > 1) {
        NCCL_CHECK(nccl()->AllGather(kin, keys_all.p, (size_t)n_pad, kNcclUint32, comm->comm, s));
        kin = keys_all.p;
        if (f % world != rank) continue;   // the owner rank sketches this feature
      }
      LAUNCH_CHECK(b2_sketch_column(kin, wq, keys_sorted.p, wq_sorted.p, wpre.p, n_total, n_global, temp.p, temp_bytes, flags.p, idx.p, uval.p, rmin.p,
                                    m_scratch.p, nvalid.p, max_bin, d_cuts + (size_t)f * 256, d_ncuts + f, d_mins + f,
                                    d_hasmiss + f, ctx->num_sms, s));
    }
  }
  // merge the per-owner tables: exact because every entry is written by exactly one rank (others hold 0 bits)
  allreduce(comm, d_tab.p, tab_n, kNcclInt32, kNcclSum, s);
  std::vector<int32_t> h_tab(tab_n);
  CUDA_CHECK(cudaMemcpyAsync(h_tab.data(), d_tab.p, tab_n * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  // categorical features: global max code / has-missing / invalid flags (allreduce max)
  const int n_cat = (int)m->cat_feats.size();
  std::vector<int32_t> h_cat((size_t)std::max(n_cat, 1) * 3, 0);
  DevBuf<int32_t> d_cat, d_catf;
  if (n_cat > 0) {
    for (int i = 0; i < n_cat; ++i) { h_cat[i * 3] = -1; h_cat[i * 3 + 1] = 0; h_cat[i * 3 + 2] = 0; }
    d_cat.ensure((size_t)n_cat * 3); d_catf.ensure((size_t)n_cat);
    CUDA_CHECK(cudaMemcpyAsync(d_cat.p, h_cat.data(), (size_t)n_cat * 3 * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    CUDA_CHECK(cudaMemcpyAsync(d_catf.p, m->cat_feats.data(), (size_t)n_cat * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    LAUNCH_CHECK(b2_launch_cat_stats(m->raw.p, m->n, F, m->missing, d_catf.p, n_cat, d_cat.p, ctx->num_sms, s));
    allreduce(comm, d_cat.p, (size_t)n_cat * 3, kNcclInt32, kNcclMax, s);
    CUDA_CHECK(cudaMemcpyAsync(h_cat.data(), d_cat.p, (size_t)n_cat * 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  }
  CUDA_CHECK(cudaStreamSynchronize(s));
  for (int i = 0; i < n_cat; ++i) {
    const int f = m->cat_feats[i], mx = h_cat[i * 3], miss = h_cat[i * 3 + 1];
    if (h_cat[i * 3 + 2] || (miss && mx > 254))
      fail("categorical feature %d: category codes must be integers in [0, %d]%s", f, miss ? 254 : 255,
           miss ? " (the feature has missing values; bin 255 is the missing sentinel)" : "");
    int32_t* t = h_tab.data();
    float* cuts_f = (float*)t + (size_t)f * 256;
    const int nc = mx < 0 ? 1 : mx + 1;
    for (int k = 0; k < nc; ++k) cuts_f[k] = (float)k;
    t[(size_t)F * 256 + f] = nc;
    ((float*)(t + (size_t)F * 256 + F))[f] = -1e-5f;
    t[(size_t)F * 256 + 2 * (size_t)F + f] = miss;
  }
  const float* h_cuts = (const float*)h_tab.data(); const int32_t* h_nc = h_tab.data() + (size_t)F * 256;
  const float* h_mins = (const float*)(h_nc + F); const int32_t* h_hm = h_nc + 2 * (size_t)F;
  m->cut_ptrs.assign(F + 1, 0);
  m->cut_vals.clear(); m->min_vals.assign(h_mins, h_mins + F); m->has_missing.assign(F, 0);
  for (int f = 0; f < F; ++f) {
    if (h_nc[f] < 1 || h_nc[f] > 256) fail("sketch produced %d cuts for feature %d", h_nc[f], f);
    m->cut_ptrs[f + 1] = m->cut_ptrs[f] + h_nc[f];
    m->cut_vals.insert(m->cut_vals.end(), h_cuts + (size_t)f * 256, h_cuts + (size_t)f * 256 + h_nc[f]);
    m->has_missing[f] = h_hm[f] ? 1 : 0;
  }
  m->max_bin = max_bin;
}

void bin_matrix(Matrix* m) {
  Ctx* ctx = m->ctx; cudaStream_t s = ctx->stream;
  setup_groups(m);
  upload_cuts(m);
  m->bins.ensure((size_t)std::max<int64_t>(m->n, 1) * m->row_stride);
  CUDA_CHECK(cudaMemsetAsync(m->bins.p, 0, (size_t)std::max<int64_t>(m->n, 1) * m->row_stride, s));
  m->col_stride = (std::max<int64_t>(m->n, 1) + 127) & ~(int64_t)127;
  m->bins_col.ensure((size_t)m->col_stride * m->F);
  LAUNCH_CHECK(b2_launch_bin(m->raw.p, m->n, m->F, m->missing, m->d_cut_ptrs.p, m->d_cut_vals.p, m->d_feat_byte.p,
                             m->any_cat() ? m->d_is_cat.p : nullptr, m->row_stride, m->bins.p, m->bins_col.p, m->col_stride,
                             ctx->num_sms, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  m->has_tmap = b2_make_bins_tensor_map(m->tmap_tile, m->bins.p, m->n, m->row_stride, 64) == 0;
  m->quantized = true;
}

// ---------------------------------------------------------------- booster
// objective ids, shared with objective_kernel.cu (the kernels take them as plain ints)
enum { kObjSquaredError = 0, kObjLogistic = 1, kObjSoftprob = 2, kObjRegLogistic = 3, kObjLogitRaw = 4, kObjSquaredLog = 5,
       kObjPseudoHuber = 6, kObjPoisson = 7, kObjGamma = 8, kObjTweedie = 9, kObjAft = 10, kObjRankPairwise = 11,
       kObjRankNdcg = 12 };
bool obj_log_link(int o) { return o == kObjPoisson || o == kObjGamma || o == kObjTweedie || o == kObjAft; }
bool obj_sigmoid(int o) { return o == kObjLogistic || o == kObjRegLogistic; }
bool obj_rank(int o) { return o == kObjRankPairwise || o == kObjRankNdcg; }
// objectives whose gradient kernel reports non-finite gradient pairs (gradient_param_kernel)
bool obj_checks_finite(int o) { return o >= kObjSquaredLog; }
struct Params {
  int objective = kObjSquaredError;
  std::string objective_name = "reg:squarederror";
  int num_class = 1;
  int num_parallel_tree = 1;   // trees grown per class and round from the SAME gradients (random forests); leaf values are scaled by eta / n
  int max_depth = 6;
  float eta = 0.3f, gamma = 0.0f, min_child_weight = 1.0f, lambda = 1.0f, alpha = 0.0f, base_score = 0.5f;
  int qbits = 18;
  int hist_chunk_rows = 0;  // 0 = auto
  int profile = 1;
  int num_feature = 0;
  int device = 0;
  int max_cat_to_onehot = 4, max_cat_threshold = 64;   // xgboost defaults (src/tree/param.h)
  float scale_pos_weight = 1.0f, max_delta_step = 0.0f;
  bool max_delta_step_set = false;             // false: count:poisson uses 0.7 (xgboost's Learner::ConfigureObjective)
  float huber_slope = 1.0f;                    // reg:pseudohubererror delta (also the mphe metric's)
  float tweedie_variance_power = 1.5f;         // reg:tweedie rho in [1, 2)
  int aft_dist = 0;                            // survival:aft distribution: 0 normal, 1 logistic, 2 extreme
  float aft_sigma = 1.0f;                      // survival:aft scale sigma > 0
  int rank_k = 32;                             // lambdarank_num_pair_per_sample (topk pairs: the first k model positions)
  bool ndcg_exp_gain = true;                   // ndcg gain 2^y - 1 (true) or y (rank:ndcg and the ndcg metrics)
  float subsample = 1.0f, colsample_bytree = 1.0f, colsample_bylevel = 1.0f, colsample_bynode = 1.0f;
  int seed = 0;
  bool base_score_set = false;   // false: estimated from the labels before the first tree (xgboost >= 2.0, A.3)
  bool use_cols() const { return colsample_bytree < 1.0f || colsample_bylevel < 1.0f || colsample_bynode < 1.0f; }
};

struct TreeHost {
  std::vector<int32_t> left, right, parent, feature, split_bin;
  std::vector<float> cond, value, base_weight, loss_chg;
  std::vector<double> sum_hess;
  std::vector<uint8_t> default_left;
  std::vector<uint8_t> split_type;        // 1 = categorical split
  std::vector<uint32_t> cat_bits;         // [n][8] categories that go right (all zero for numeric nodes)
  bool any_cat = false;
  int add(int par) {
    int id = (int)left.size();
    left.push_back(-1); right.push_back(-1); parent.push_back(par); feature.push_back(-1); split_bin.push_back(-1);
    cond.push_back(0.f); value.push_back(0.f); base_weight.push_back(0.f); loss_chg.push_back(0.f); sum_hess.push_back(0.0);
    default_left.push_back(0); split_type.push_back(0); cat_bits.insert(cat_bits.end(), 8, 0u);
    return id;
  }
  int size() const { return (int)left.size(); }
};


struct Timers {
  double hist_ms = 0, round_ms = 0;
  double shap_ms = 0;   // kernel time of pred_contribs / pred_interactions (CUDA events around the SHAP kernels)
  long long shap_rows = 0;
  double phase_ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // profile=2: quant, hist, allreduce, subtract, eval+decide, partition+finalize, leaf, other
  long long hist_launches = 0, hist_rows = 0, kernel_launches = 0, rounds = 0;
  double hist_bytes = 0, allreduce_bytes = 0;
  void reset() { *this = Timers(); }
};

struct EvalCache { DevBuf<float> margin; int n_trees_applied = 0; int64_t n = 0; uint64_t margin_version = 0; };

// per-group descending order of a row vector (rank_kernel.cu b2_rank_order): keys_sorted / rows hold, for every model
// position, the sort key (the value) and the row.  The buffers are pooled and kept, so a booster sorts its train margins
// every round without allocating.
struct RankOrder {
  DevBuf<int32_t> iota, rows; DevBuf<uint32_t> keys, keys_sorted; DevBuf<uint8_t> temp;
  int64_t n = -1, groups = -1; size_t temp_bytes = 0;
  void run(Matrix* m, const float* v, int num_sms, cudaStream_t s) {
    if (n != m->n || groups != m->n_qgroups) {
      const size_t rows_cap = (size_t)std::max<int64_t>(m->n, 1);
      iota.ensure(rows_cap); rows.ensure(rows_cap); keys.ensure(rows_cap); keys_sorted.ensure(rows_cap);
      temp_bytes = b2_rank_order_temp_bytes(m->n, m->n_qgroups);
      temp.ensure(std::max<size_t>(temp_bytes, 1));
      LAUNCH_CHECK(b2_launch_rank_iota(iota.p, m->n, num_sms, s));
      n = m->n; groups = m->n_qgroups;
    }
    LAUNCH_CHECK(b2_rank_order(v, m->n, m->qgroup_ptr.p, m->n_qgroups, iota.p, keys.p, keys_sorted.p, rows.p, temp.p,
                               temp_bytes, num_sms, s));
  }
};

struct Booster : HandleBase {
  Ctx* ctx = nullptr;
  Params p;
  Matrix* train = nullptr;
  int n_features = 0;
  Comm* comm = nullptr;
  std::vector<TreeHost> trees;
  std::atomic<bool> cancel{false};
  // device model cache for prediction
  DevBuf<B2TreeNodeDev> d_nodes; DevBuf<int32_t> d_tree_offset; int d_trees_synced = 0;
  std::vector<B2TreeNodeDev> h_nodes; std::vector<int32_t> h_tree_offset;
  DevBuf<uint32_t> d_cat_table; std::vector<uint32_t> h_cat_table;   // [categorical nodes][8]
  // TreeSHAP path table (build_paths), rebuilt when the tree set changes (paths_synced = trees it was built from, -1 = stale)
  DevBuf<B2PathElem> d_path_elems; DevBuf<B2PathInfo> d_paths; DevBuf<uint32_t> d_path_cats;
  std::vector<int32_t> tree_path_offset;   // [trees + 1]: paths of tree t are [offset[t], offset[t+1])
  std::vector<double> tree_expected;       // [trees] cover-weighted mean of the leaves (the tree's SHAP bias)
  int paths_synced = -1;
  // training state
  bool margin_ready = false;
  DevBuf<float> margin;          // [n][K]
  DevBuf<float2> gh;             // [K][n]
  DevBuf<float2> gh_round;       // copy of the round's gradients (num_parallel_tree > 1 with row sampling)
  DevBuf<int2> q;                // [n]
  DevBuf<int32_t> ridx[2];
  DevBuf<long long> hist[2];
  // Everything a peer maps lives in ONE allocation (one cudaIpc handle per peer instead of four): the build buffer, the
  // candidate table, the misc table and the flag words are views into it
  template <typename T> struct View { T* p = nullptr; };
  DevBuf<uint8_t> xarena;
  size_t xoff_cands = 0, xoff_misc = 0, xoff_flags = 0, x_misc_stride = 0;
  View<long long> hist_build;       // reduce-scatter send buffer [shards][node_cap][slice] (only when shards > 1)
  View<B2SplitCand> d_cands_all;    // candidates of all ranks [shards][nodes][cpn]
  int shards = 1, log2_shards = 0, sp = 32, cpn = 1;   // cpn = most candidates per node of a level (numeric CTAs + categorical CTAs)
  int cpn_num = 1;
  View<uint32_t> t_cat;                    // [max_nodes][8] category sets of the tree being grown (in t_block)
  DevBuf<uint8_t> d_col_masks;             // [max_depth][F] level feature sets of the tree being grown (column sampling)
  // NVLink peer-memory exchange (p2p.cuh, p2p_exchange.cu): on when every rank mapped its peers; B2_EXCHANGE=nccl keeps NCCL
  struct P2PState {
    bool enabled = false, tried = false;
    B2P2P pp;
    DevBuf<uint32_t> words;               // [kP2PSlots] epoch, [kP2PSlots] done, err, local abort stand-in (never mapped by peers)
    uint32_t* flags = nullptr;            // views into Booster::xarena
    long long* misc = nullptr;            // [world][misc_stride]
    std::vector<void*> opened;
    int cand_cap = 0;
  } p2p;
  // CUDA graphs of the per-tree launch sequence, one per class tree of a round (grow_tree is sync-free and its
  // arguments are the same for every tree, so the sequence is captured once and replayed)
  struct TreeGraph {
    cudaGraphExec_t exec = nullptr;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> hist_ev;   // owned; recorded by the graph (external event nodes)
    long long hist_launches = 0, kernel_launches = 0;
    double allreduce_bytes = 0;
  };
  std::map<int, TreeGraph> graphs;
  std::map<int, int> direct_trees;         // trees grown with direct launches per class slot (the first one allocates)
  bool graph_failed = false;
  bool absmax_fused = false;               // this round's gradient kernel already produced d_absmax[k]
  bool labels_checked = false;             // the train labels are inside the objective's domain (check_labels)
  bool gh_ready = false;                   // gh holds the gradient pairs of a round (B2_BoosterGetGradients)
  DevBuf<uint32_t> d_grad_err;             // set by the gradient kernel when a gradient pair is not finite
  uint32_t* h_grad_err = nullptr;          // pinned copy, written at the end of the round's stream work
  DevBuf<uint16_t> pos;                    // [n] leaf index of every row (final_assign / leaf_sums -> margin_update)
  size_t slice_elems = 0;
  size_t node_elems = 0;
  DevBuf<uint32_t> d_absmax; DevBuf<int32_t> d_qexp;
  // device-resident control tables of the sync-free level loop (control_kernel.cu)
  int ctl_depth = 0;                       // max_depth the tables are sized for
  // the tree being grown, laid out as its pinned read-back block (TreeLayout) so that one copy brings it back
  DevBuf<uint8_t> t_block;
  View<int32_t> t_i32;                     // 7 int32 arrays [max_nodes] + n_nodes + n_leaves
  View<float> t_f32;                       // loss_chg, leaf_weight, leaf_value [max_nodes]
  View<long long> t_i64;                   // sum_g, sum_h [max_nodes] + level_rows [max_depth+1]
  View<int32_t> t_qexp;                    // the tree's quantisation exponents (written by leaf_values_kernel)
  DevBuf<B2LevelCtl> d_ctl;                // [0],[1] level ping-pong, [2] leaf pass
  DevBuf<B2NodeSeg> d_seg[2]; DevBuf<B2EvalNode> d_ev[2];
  DevBuf<B2HistWork> d_hist_work; DevBuf<B2SplitWork> d_split_work; DevBuf<B2SegWork> d_seg_work;
  DevBuf<B2SplitCand> d_cands; DevBuf<int32_t> d_counters, d_triples, d_pair_parent;
  DevBuf<uint32_t> d_part_done;            // CTAs of a partition that finished (zero between launches: the last resets it)
  DevBuf<uint32_t> d_eval_done;            // CTAs of a split scan that finished when it decides the level (same rule)
  DevBuf<B2SplitCand> d_cand_best;         // [nodes of a level] decide's winner of every node
  DevBuf<B2LeafDev> d_leaves;
  DevBuf<long long> d_leaf_sums; DevBuf<float> d_leaf_values; DevBuf<double> d_metric;
  std::vector<void*> staging;              // pinned host copies of finished trees, one per class tree of a round
  size_t staging_bytes = 0;
  DevBuf<float> d_custom_g, d_custom_h;
  std::map<uint64_t, EvalCache*> eval_cache;   // keyed by Matrix::uid
  // learning to rank: the train margins' order (every round), the discount table ln2 / log(r + 2) (grown to the largest
  // group seen), 1/IDCG of the train groups (keyed by matrix, its rank_version, k and the gain) and the stage of the
  // groups larger than the gradient kernel's shared-memory stage
  RankOrder rank_order;
  DevBuf<double> rank_disc; int64_t rank_disc_len = 0;
  DevBuf<double> rank_inv_idcg; uint64_t idcg_uid = 0, idcg_version = 0; int idcg_k = -1, idcg_gain = -1;
  DevBuf<float> rank_scratch_m, rank_scratch_y; DevBuf<double> rank_scratch_p;
  // profiling
  Timers t;
  std::vector<cudaEvent_t> ev_pool; size_t ev_used = 0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> hist_events;
  std::vector<std::pair<int, cudaEvent_t>> phase_marks;   // (phase that ENDS at this event)
  cudaEvent_t round_start = nullptr, round_stop = nullptr;
  ~Booster() {
    for (auto& kv : graphs) {
      if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
      for (auto& pr : kv.second.hist_ev) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
    }
    // No barrier with the peers here: a peer touches this rank's arena only inside the exchange kernels of a round, and
    // every one of those accesses happens-before a flag that this rank waited for before ITS round completed -- once the
    // last round is synchronised the arena is quiescent.  (A barrier in the destructor made a rank whose peer keeps its
    // Booster alive -- the rank that returns the model -- spin until the peer-wait timeout: 23 s per train() call.)
    if (ctx) cudaStreamSynchronize(ctx->stream);
    for (void* q : p2p.opened) cudaIpcCloseMemHandle(q);
    for (auto e : ev_pool) cudaEventDestroy(e);
    if (round_start) cudaEventDestroy(round_start);
    if (round_stop) cudaEventDestroy(round_stop);
    for (auto& kv : eval_cache) delete kv.second;
    for (void* h : staging) cudaFreeHost(h);
    if (h_grad_err) cudaFreeHost(h_grad_err);
  }
};

cudaEvent_t get_event(Booster* b) {
  if (b->ev_used == b->ev_pool.size()) { cudaEvent_t e; CUDA_CHECK(cudaEventCreate(&e)); b->ev_pool.push_back(e); }
  return b->ev_pool[b->ev_used++];
}
void mark_phase(Booster* b, int phase) {
  if (b->p.profile < 2) return;
  cudaEvent_t e = get_event(b);
  CUDA_CHECK(cudaEventRecord(e, b->ctx->stream));
  b->phase_marks.push_back({phase, e});
}
void resolve_events(Booster* b) {
  for (size_t i = 1; i < b->phase_marks.size(); ++i) {
    float ms = 0.f;
    if (b->phase_marks[i].first >= 0 && cudaEventElapsedTime(&ms, b->phase_marks[i - 1].second, b->phase_marks[i].second) == cudaSuccess)
      b->t.phase_ms[b->phase_marks[i].first] += ms;
  }
  b->phase_marks.clear();
  for (auto& pr : b->hist_events) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, pr.first, pr.second) == cudaSuccess) b->t.hist_ms += ms;
  }
  b->hist_events.clear();
  b->ev_used = 0;
}

void parse_params(const char* text, Params* p, int* max_bin_out) {
  std::string s(text ? text : "");
  size_t pos = 0;
  while (pos < s.size()) {
    size_t nl = s.find('\n', pos);
    if (nl == std::string::npos) nl = s.size();
    std::string line = s.substr(pos, nl - pos);
    pos = nl + 1;
    size_t eq = line.find('=');
    if (eq == std::string::npos) continue;
    std::string k = line.substr(0, eq), v = line.substr(eq + 1);
    auto f = [&]() { return (float)atof(v.c_str()); };
    auto i = [&]() { return atoi(v.c_str()); };
    if (k == "objective") {
      p->objective_name = v;
      if (v == "reg:squarederror" || v == "reg:linear") p->objective = kObjSquaredError;
      else if (v == "binary:logistic") p->objective = kObjLogistic;
      else if (v == "multi:softprob" || v == "multi:softmax") p->objective = kObjSoftprob;
      else if (v == "reg:logistic") p->objective = kObjRegLogistic;
      else if (v == "binary:logitraw") p->objective = kObjLogitRaw;
      else if (v == "reg:squaredlogerror") p->objective = kObjSquaredLog;
      else if (v == "reg:pseudohubererror") p->objective = kObjPseudoHuber;
      else if (v == "count:poisson") p->objective = kObjPoisson;
      else if (v == "reg:gamma") p->objective = kObjGamma;
      else if (v == "reg:tweedie") p->objective = kObjTweedie;
      else if (v == "survival:aft") p->objective = kObjAft;
      else if (v == "rank:pairwise") p->objective = kObjRankPairwise;
      else if (v == "rank:ndcg") p->objective = kObjRankNdcg;
      else fail("unsupported objective '%s' (supported: reg:squarederror, reg:logistic, binary:logistic, binary:logitraw, "
                "reg:squaredlogerror, reg:pseudohubererror, count:poisson, reg:gamma, reg:tweedie, survival:aft, "
                "rank:pairwise, rank:ndcg, multi:softprob, multi:softmax)", v.c_str());
    } else if (k == "num_class") p->num_class = i();
    else if (k == "num_parallel_tree") p->num_parallel_tree = i();
    else if (k == "max_depth") p->max_depth = i();
    else if (k == "eta" || k == "learning_rate") p->eta = f();
    else if (k == "gamma" || k == "min_split_loss") p->gamma = f();
    else if (k == "min_child_weight") p->min_child_weight = f();
    else if (k == "lambda" || k == "reg_lambda") p->lambda = f();
    else if (k == "alpha" || k == "reg_alpha") p->alpha = f();
    else if (k == "base_score") { p->base_score = f(); p->base_score_set = true; }
    else if (k == "hist_qbits") p->qbits = i();
    else if (k == "hist_chunk_rows") p->hist_chunk_rows = i();
    else if (k == "profile") p->profile = i();
    else if (k == "num_feature") p->num_feature = i();
    else if (k == "device") p->device = i();
    else if (k == "subsample") p->subsample = f();
    else if (k == "colsample_bytree") p->colsample_bytree = f();
    else if (k == "colsample_bylevel") p->colsample_bylevel = f();
    else if (k == "colsample_bynode") p->colsample_bynode = f();
    else if (k == "seed" || k == "random_state") p->seed = i();
    else if (k == "scale_pos_weight") p->scale_pos_weight = f();
    else if (k == "max_delta_step") { p->max_delta_step = f(); p->max_delta_step_set = true; }
    else if (k == "huber_slope") p->huber_slope = f();
    else if (k == "tweedie_variance_power") p->tweedie_variance_power = f();
    else if (k == "aft_loss_distribution") {
      if (v == "normal") p->aft_dist = 0;
      else if (v == "logistic") p->aft_dist = 1;
      else if (v == "extreme") p->aft_dist = 2;
      else fail("aft_loss_distribution must be normal, logistic or extreme, got '%s'", v.c_str());
    }
    else if (k == "aft_loss_distribution_scale") p->aft_sigma = f();
    else if (k == "lambdarank_pair_method") {
      if (v != "topk") fail("lambdarank_pair_method='%s' is not supported (supported: topk; random pair sampling "
                            "(mean) is not implemented)", v.c_str());
    }
    else if (k == "lambdarank_num_pair_per_sample") {
      char* end = nullptr;
      const long long kv = strtoll(v.c_str(), &end, 10);
      if (v.empty() || *end != '\0' || kv < 1 || kv > INT32_MAX)
        fail("lambdarank_num_pair_per_sample must be an integer >= 1, got '%s'", v.c_str());
      p->rank_k = (int)kv;
    }
    else if (k == "lambdarank_unbiased" || k == "ndcg_exp_gain") {
      bool on;
      if (v == "1" || v == "true" || v == "True") on = true;
      else if (v == "0" || v == "false" || v == "False") on = false;
      else fail("%s must be a boolean, got '%s'", k.c_str(), v.c_str());
      if (k == "ndcg_exp_gain") p->ndcg_exp_gain = on;
      else if (on) fail("lambdarank_unbiased=true is not supported (position-bias estimation is not implemented)");
    }
    else if (k == "max_cat_to_onehot") p->max_cat_to_onehot = i();
    else if (k == "max_cat_threshold") p->max_cat_threshold = i();
    else if (k == "max_bin") { if (max_bin_out) *max_bin_out = i(); }
    // unknown keys (nthread, tree_method, verbosity, ...) are accepted and ignored, like xgboost
  }
  if (obj_rank(p->objective) && p->num_class > 1)
    fail("%s has one output per row: num_class must be 1, got %d", p->objective_name.c_str(), p->num_class);
  if (p->objective != kObjSoftprob) p->num_class = 1;
  if (p->objective == kObjSoftprob && p->num_class < 2) fail("multi:softprob needs num_class >= 2");
  if (p->max_depth < 1 || p->max_depth > 14) fail("max_depth must be in [1, 14], got %d", p->max_depth);
  if (p->num_parallel_tree < 1 || p->num_parallel_tree > 4096) fail("num_parallel_tree must be in [1, 4096], got %d", p->num_parallel_tree);
  if (p->qbits < 8 || p->qbits > 24) fail("hist_qbits must be in [8, 24], got %d", p->qbits);
  for (float v : {p->subsample, p->colsample_bytree, p->colsample_bylevel, p->colsample_bynode})
    if (!(v > 0.0f && v <= 1.0f)) fail("subsample / colsample_* must be in (0, 1], got %g", (double)v);
  if (p->max_cat_to_onehot < 1) fail("max_cat_to_onehot must be >= 1, got %d", p->max_cat_to_onehot);
  if (p->max_cat_threshold < 1) fail("max_cat_threshold must be >= 1, got %d", p->max_cat_threshold);
  if (p->objective == kObjPoisson) {
    if (!p->max_delta_step_set) p->max_delta_step = 0.7f;   // both the hessian's shift and the leaf-step clamp
    if (!(p->max_delta_step >= 0.0f)) fail("max_delta_step must be >= 0 for count:poisson, got %g", (double)p->max_delta_step);
  }
  if (p->objective == kObjPseudoHuber && !(p->huber_slope > 0.0f))
    fail("huber_slope must be > 0 for reg:pseudohubererror, got %g", (double)p->huber_slope);
  if (p->objective == kObjTweedie && !(p->tweedie_variance_power >= 1.0f && p->tweedie_variance_power < 2.0f))
    fail("tweedie_variance_power must be in [1, 2), got %g", (double)p->tweedie_variance_power);
  if (!(p->aft_sigma > 0.0f) || std::isinf(p->aft_sigma))
    fail("aft_loss_distribution_scale must be finite and > 0, got %g", (double)p->aft_sigma);
  // survival:aft fits no intercept: base_score defaults to 0.5 (margin log 0.5) and is never estimated
  if (p->objective == kObjAft && !p->base_score_set) { p->base_score = 0.5f; p->base_score_set = true; }
  // the rank objectives neither: their margin is the score itself (identity transform)
  if (obj_rank(p->objective) && !p->base_score_set) { p->base_score = 0.5f; p->base_score_set = true; }
  if (p->base_score_set) {
    if (p->objective == kObjRegLogistic && !(p->base_score > 0.0f && p->base_score < 1.0f))
      fail("base_score must be in (0, 1) for reg:logistic, got %g", (double)p->base_score);
    if (obj_log_link(p->objective) && !(p->base_score > 0.0f))
      fail("base_score must be > 0 for %s, got %g", p->objective_name.c_str(), (double)p->base_score);
  }
}

// the parameter that the gradient kernel of an objective takes (gradient_param_kernel)
float objective_param(const Params& p) {
  if (p.objective == kObjPseudoHuber) return p.huber_slope;
  if (p.objective == kObjPoisson) return p.max_delta_step;
  if (p.objective == kObjTweedie) return p.tweedie_variance_power;
  return 0.0f;
}

// margin of base_score (the inverse of the prediction transform), evaluated on the host with libm's logf
float base_margin_value(const Params& p) {
  if (obj_sigmoid(p.objective)) return -logf(1.0f / p.base_score - 1.0f);
  if (obj_log_link(p.objective)) return logf(p.base_score);
  return p.base_score;
}

// -- host replicas of the gain / weight formulas (A.6, A.7); same IEEE sequence as the kernels
double h_thr_l1(double g, double a) { if (g > a) return g - a; if (g < -a) return g + a; return 0.0; }
float h_calc_weight(const Params& p, double G, double H) {
  if (H < (double)p.min_child_weight || H <= 0.0) return 0.0f;
  double t = p.alpha == 0.0f ? G : h_thr_l1(G, (double)p.alpha);
  double dw = -t / (H + (double)p.lambda);
  if (p.max_delta_step != 0.0f && fabs(dw) > (double)p.max_delta_step) dw = copysign((double)p.max_delta_step, dw);
  return (float)dw;
}

int window_rows_for(int qbits) {
  // overflow-guard interval of the histogram kernel: |q| <= 2^qbits, so 2^(30-qbits) rows add less than 2^30
  // to a cell that was below 2^30 at the last check (hist_kernel.cu flush_large_cells)
  return 1 << (30 - qbits);
}

int pick_chunk_rows(Booster* b, int64_t rows) {
  if (b->p.hist_chunk_rows > 0) return b->p.hist_chunk_rows;
  const int n_streams = std::max(1, b->ctx->num_sms * 3 / b->train->n_groups);
  const int64_t per_stream = rows / n_streams;
  int64_t target = per_stream >= 16384 ? per_stream / 4 : per_stream;
  int c = 512;
  while (c < target && c < 8192) c <<= 1;
  const int w = window_rows_for(b->p.qbits);
  if (c > w) c = w;   // one chunk = one int32 window
  return c;
}

// layout of the per-tree read-back block (device t_* buffers are copied verbatim into one pinned block)
struct TreeLayout {
  size_t max_nodes, i32_count, f32_count, i64_count, bytes;
  size_t off_f32, off_i64, off_qexp, off_cat;
};
TreeLayout tree_layout(int max_depth) {
  TreeLayout L;
  L.max_nodes = ((size_t)1 << (max_depth + 1));
  L.i32_count = 7 * L.max_nodes + 2;
  L.f32_count = 3 * L.max_nodes;
  L.i64_count = 2 * L.max_nodes + (size_t)max_depth + 2;
  L.off_f32 = L.i32_count * 4;
  L.off_i64 = (L.off_f32 + L.f32_count * 4 + 7) & ~(size_t)7;
  L.off_qexp = L.off_i64 + L.i64_count * 8;
  L.off_cat = L.off_qexp + 16;
  L.bytes = L.off_cat + L.max_nodes * 8 * sizeof(uint32_t);
  return L;
}
B2TreeDev tree_dev(Booster* b) {
  const TreeLayout L = tree_layout(b->ctl_depth);
  B2TreeDev t;
  int32_t* i = b->t_i32.p; const size_t m = L.max_nodes;
  t.left = i; t.right = i + m; t.parent = i + 2 * m; t.feature = i + 3 * m; t.split_bin = i + 4 * m; t.default_left = i + 5 * m;
  t.split_type = i + 6 * m;
  t.n_nodes = i + 7 * m;
  t.cat_bits = b->t_cat.p;
  t.loss_chg = b->t_f32.p; t.leaf_weight = b->t_f32.p + m; t.leaf_value = b->t_f32.p + 2 * m;
  t.sum_g = b->t_i64.p; t.sum_h = b->t_i64.p + m;
  return t;
}

// Map every peer's build buffer, candidate table, misc table and flag array (cudaIpc) for the peer-memory exchange.
// All ranks take the same decision: one failed mapping anywhere leaves every rank on NCCL.
int p2p_timeout_seconds() {
  const char* e = getenv("B2_P2P_TIMEOUT_S");
  int v = e ? atoi(e) : 60;
  return v < 1 ? 1 : v;
}
void p2p_setup(Booster* b) {
  Booster::P2PState& st = b->p2p;
  if (st.tried || b->shards <= 1) return;
  st.tried = true;
  const char* env = getenv("B2_EXCHANGE");
  if (env && (strcmp(env, "nccl") == 0 || strcmp(env, "NCCL") == 0)) return;
  Comm* c = b->comm; cudaStream_t s = b->ctx->stream; const int W = c->world;
  if (W > B2_P2P_MAX_WORLD) return;
  const size_t misc_stride = b->x_misc_stride;
  const size_t n_flags = (size_t)b2_p2p_flag_words(W), n_words = 2 * (size_t)kP2PSlots + 2;
  st.words.ensure(n_words);
  CUDA_CHECK(cudaMemsetAsync(st.flags, 0, n_flags * sizeof(uint32_t), s));
  CUDA_CHECK(cudaMemsetAsync(st.words.p, 0, n_words * sizeof(uint32_t), s));
  CUDA_CHECK(cudaMemsetAsync(st.misc, 0, (size_t)W * misc_stride * sizeof(long long), s));
  cudaIpcMemHandle_t mine; int ok = 1;
  if (cudaIpcGetMemHandle(&mine, b->xarena.p) != cudaSuccess) { ok = 0; cudaGetLastError(); memset(&mine, 0, sizeof(mine)); }
  DevBuf<uint8_t> d_mine, d_all; d_mine.ensure(sizeof(mine)); d_all.ensure(sizeof(mine) * (size_t)W);
  CUDA_CHECK(cudaMemcpyAsync(d_mine.p, &mine, sizeof(mine), cudaMemcpyHostToDevice, s));
  NCCL_CHECK(nccl()->AllGather(d_mine.p, d_all.p, sizeof(mine), kNcclUint8, c->comm, s));   // also orders the memsets before any peer store
  std::vector<cudaIpcMemHandle_t> all((size_t)W);
  CUDA_CHECK(cudaMemcpyAsync(all.data(), d_all.p, sizeof(mine) * (size_t)W, cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  memset(&st.pp, 0, sizeof(st.pp));
  st.pp.world = W; st.pp.rank = c->rank; st.pp.cand_cap = st.cand_cap; st.pp.misc_stride = (int32_t)misc_stride;
  st.pp.epoch = st.words.p; st.pp.done = st.words.p + kP2PSlots; st.pp.err = st.words.p + 2 * kP2PSlots;
  st.pp.abort_flag = c->d_abort ? c->d_abort : st.words.p + 2 * kP2PSlots + 1;
  st.pp.spin_limit = (long long)p2p_timeout_seconds() * 1000000LL;
  for (int w = 0; w < W && ok; ++w) {
    uint8_t* base = b->xarena.p;
    if (w != c->rank) {
      void* q = nullptr;
      if (cudaIpcOpenMemHandle(&q, all[w], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { ok = 0; cudaGetLastError(); break; }
      st.opened.push_back(q);
      base = (uint8_t*)q;
    }
    st.pp.build[w] = (long long*)base; st.pp.cands[w] = (B2SplitCand*)(base + b->xoff_cands);
    st.pp.misc[w] = (long long*)(base + b->xoff_misc); st.pp.flags[w] = (uint32_t*)(base + b->xoff_flags);
  }
  // agree: max over ranks of "failed"
  DevBuf<int32_t> d_ok; d_ok.ensure(1);
  int32_t neg = ok ? 0 : 1;
  CUDA_CHECK(cudaMemcpyAsync(d_ok.p, &neg, sizeof(neg), cudaMemcpyHostToDevice, s));
  allreduce(c, d_ok.p, 1, kNcclInt32, kNcclMax, s);
  CUDA_CHECK(cudaMemcpyAsync(&neg, d_ok.p, sizeof(neg), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  if (neg) {
    for (void* q : st.opened) cudaIpcCloseMemHandle(q);
    st.opened.clear();
    if (getenv("B2_EXCHANGE")) fprintf(stderr, "[b2hist] peer mapping failed on some rank; histogram exchange stays on NCCL\n");
    return;
  }
  st.enabled = true;
}

void ensure_ctl_tables(Booster* b) {
  const int D = b->p.max_depth; const int G = b->train->n_groups;
  if (b->ctl_depth == D) return;
  if (b->ctl_depth != 0 && b->p2p.enabled) fail("max_depth cannot change while the peer-memory exchange is mapped");
  for (auto& kv : b->graphs) {   // captured launch sequences hold the old table addresses
    if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
    for (auto& pr : kv.second.hist_ev) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
  }
  b->graphs.clear(); b->direct_trees.clear();
  b->ctl_depth = D;
  const TreeLayout L = tree_layout(D);
  const size_t lcap = (size_t)1 << D, half = (size_t)1 << (D > 0 ? D - 1 : 0);
  b->t_block.ensure(L.bytes);
  b->t_i32.p = (int32_t*)b->t_block.p; b->t_f32.p = (float*)(b->t_block.p + L.off_f32);
  b->t_i64.p = (long long*)(b->t_block.p + L.off_i64); b->t_qexp.p = (int32_t*)(b->t_block.p + L.off_qexp);
  b->t_cat.p = (uint32_t*)(b->t_block.p + L.off_cat);
  b->d_ctl.ensure(3);
  for (int k = 0; k < 2; ++k) { b->d_seg[k].ensure(lcap); b->d_ev[k].ensure(lcap); }
  b->d_hist_work.ensure(half); b->d_split_work.ensure(half);
  b->d_counters.ensure(2 * half); b->d_triples.ensure(3 * half); b->d_pair_parent.ensure(half);
  if (!b->d_part_done.p) { b->d_part_done.ensure(1); CUDA_CHECK(cudaMemsetAsync(b->d_part_done.p, 0, sizeof(uint32_t), b->ctx->stream)); }
  if (!b->d_eval_done.p) { b->d_eval_done.ensure(1); CUDA_CHECK(cudaMemsetAsync(b->d_eval_done.p, 0, sizeof(uint32_t), b->ctx->stream)); }
  b->d_cand_best.ensure(half);
  b->d_leaves.ensure(L.max_nodes); b->d_seg_work.ensure(L.max_nodes);
  b->d_leaf_sums.ensure(2 * lcap); b->d_leaf_values.ensure(lcap);
  b->node_elems = (size_t)G * B2_GROUP_ELEMS;
  // feature-slot sharding of the histogram exchange: rank r owns slots s with s % shards == r (DESIGN.md 5)
  const int world = b->comm ? b->comm->world : 1;
  b->shards = (world > 1 && world <= 32 && (32 % world) == 0) ? world : 1;
  b->log2_shards = 0; while ((1 << b->log2_shards) < b->shards) b->log2_shards++;
  b->sp = B2_GROUP_SLOTS / b->shards;
  b->slice_elems = (size_t)G * 2 * B2_BINS * b->sp;
  b->cpn_num = b2_eval_ctas_per_node(G, b->log2_shards, 1);   // the most numeric candidates per node of any level
  b->cpn = b->cpn_num + (b->train->any_cat() ? b2_cat_ctas() : 0);
  b->hist[0].ensure(half * b->slice_elems); b->hist[1].ensure(half * b->slice_elems);
  if (b->shards > 1) {
    auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
    const size_t build_bytes = up(half * b->node_elems * sizeof(long long));
    const size_t cands_bytes = up(half * b->cpn * b->shards * sizeof(B2SplitCand));
    b->x_misc_stride = 2 + 2 * lcap;                                   // even: 16-byte aligned regions
    const size_t misc_bytes = up((size_t)b->shards * b->x_misc_stride * sizeof(long long));
    const size_t flag_bytes = up((size_t)b2_p2p_flag_words(b->shards) * sizeof(uint32_t));
    b->xoff_cands = build_bytes; b->xoff_misc = b->xoff_cands + cands_bytes; b->xoff_flags = b->xoff_misc + misc_bytes;
    b->xarena.ensure(b->xoff_flags + flag_bytes);
    b->hist_build.p = (long long*)b->xarena.p;
    b->d_cands_all.p = (B2SplitCand*)(b->xarena.p + b->xoff_cands);
    b->p2p.misc = (long long*)(b->xarena.p + b->xoff_misc);
    b->p2p.flags = (uint32_t*)(b->xarena.p + b->xoff_flags);
  }
  b->d_cands.ensure(half * b->cpn);
  CUDA_CHECK(cudaMemsetAsync(b->t_i64.p, 0, L.i64_count * 8, b->ctx->stream));
  b->p2p.cand_cap = (int)(half * b->cpn);
  p2p_setup(b);
}

// Launch bookkeeping of one tree: with direct launches it is applied right away, a captured tree keeps it with its
// graph and applies it on every replay.
struct TreeStats {
  long long hist_launches = 0, kernel_launches = 0;
  double allreduce_bytes = 0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> hist_ev;
  bool capturing = false;
};
void record_hist_launch(Booster* b, TreeStats& st, cudaEvent_t& e0, cudaEvent_t& e1, bool begin) {
  if (!b->p.profile) return;
  cudaStream_t s = b->ctx->stream;
  if (begin) {
    if (st.capturing) { CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1)); }   // owned by the graph
    else { e0 = get_event(b); e1 = get_event(b); }
    // inside a capture the record becomes an event-record node that every replay executes (external event)
    CUDA_CHECK(cudaEventRecordWithFlags(e0, s, st.capturing ? cudaEventRecordExternal : cudaEventRecordDefault));
  } else {
    CUDA_CHECK(cudaEventRecordWithFlags(e1, s, st.capturing ? cudaEventRecordExternal : cudaEventRecordDefault));
    st.hist_ev.push_back({e0, e1});
  }
}

bool use_tma_hist() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("B2_HIST_TMA"); v = (e && atoi(e) != 0) ? 1 : 0; }
  return v == 1;
}
bool env_flag(const char* name, bool dflt) {
  const char* e = getenv(name);
  return e ? atoi(e) != 0 : dflt;
}

// Where the histogram kernel of a level accumulates: the reduce-scatter / peer-read build buffer when the exchange
// is sharded by feature slot (shards == world), else the level buffer itself (single GPU, or in-place allreduce).
long long* build_target(Booster* b, long long* level_buf) { return b->shards > 1 ? b->hist_build.p : level_buf; }

// Histogram exchange of the nodes built for one level + sibling subtraction (parent - built).
//   peer memory : ONE kernel reads the W partial slices out of the peers' build buffers, stores built and sibling
//   NCCL        : reduce-scatter (shards == world) or in-place allreduce, then hist_subtract_kernel
// `triples` == nullptr: the root (nothing to subtract).
void exchange_and_subtract(Booster* b, TreeStats& st, const long long* parent_level, long long* level_buf, const int32_t* triples,
                           const B2LevelCtl* ctl_nxt, int nb, int node_cap) {
  cudaStream_t s = b->ctx->stream;
  const bool multi = b->comm && b->comm->world > 1;
  if (multi && b->comm->aborted.load()) fail("communicator aborted");
  if (multi && b->p2p.enabled) {
    LAUNCH_CHECK(b2_launch_p2p_reduce_subtract(&b->p2p.pp, parent_level, level_buf, triples, ctl_nxt, nb, node_cap,
                                               (int64_t)b->slice_elems, b->ctx->num_sms, s));
    st.allreduce_bytes += (double)nb * b->node_elems * 8 * (b->shards - 1) / b->shards;
    st.kernel_launches++;
    mark_phase(b, 2);
    return;
  }
  if (multi && b->shards > 1) {
    NCCL_CHECK(nccl()->ReduceScatter(b->hist_build.p, level_buf, (size_t)nb * b->slice_elems, kNcclInt64, kNcclSum, b->comm->comm, s));
    st.allreduce_bytes += (double)nb * b->node_elems * 8 * (b->shards - 1) / b->shards;
  } else if (multi) {
    NCCL_CHECK(nccl()->AllReduce(level_buf, level_buf, (size_t)nb * b->node_elems, kNcclInt64, kNcclSum, b->comm->comm, s));
    st.allreduce_bytes += (double)nb * b->node_elems * 8;
  }
  mark_phase(b, 2);
  if (triples) {
    LAUNCH_CHECK(b2_launch_hist_subtract(parent_level, level_buf, triples, nb, (int64_t)b->slice_elems, ctl_nxt, s));
    st.kernel_launches++;
  }
  mark_phase(b, 3);
}

// Grow one tree for class k from gh[k] (already on device); updates margin[:, k].  No host
// synchronisation: every data-dependent decision is taken by the control kernels, the host
// enqueues a fixed sequence and the finished tree is copied into pinned block `slot`.
// With st.capturing the stream is in capture mode: nothing here may allocate, touch pageable host memory or depend on
// host state that changes from tree to tree (run_tree decides when that holds).
void grow_tree(Booster* b, int k, int slot, TreeStats& st) {
  Matrix* m = b->train; Ctx* ctx = b->ctx; cudaStream_t s = ctx->stream; const Params& p = b->p;
  const int64_t n = m->n; const int K = p.num_class; const int G = m->n_groups; const int D = p.max_depth;
  const float2* gh = b->gh.p + (size_t)k * n;
  ensure_ctl_tables(b);
  const TreeLayout L = tree_layout(D);
  const bool multi = b->comm && b->comm->world > 1;
  const bool p2p = multi && b->p2p.enabled;
  static const bool leaf_fused = env_flag("B2_LEAF_FUSED", true);
  // leaf sums from a streaming pass over (pos, gh) in row order; needs one shared-memory accumulator per leaf
  const bool leaf_stream = leaf_fused && D >= 1 && D <= b2_leaf_acc_max_depth();
  // sibling subtraction inside eval_splits_kernel (no hist_subtract pass).  The peer-memory exchange subtracts while it
  // reduces, and the categorical scan reads the sibling slots itself, so both keep the stored siblings.
  const bool sub_in_scan = !p2p && !m->any_cat();
  mark_phase(b, -1);
  // ---- fixed-point quantisation (global scale via max over the ranks)
  const uint32_t tree_index = (uint32_t)b->trees.size() + (uint32_t)slot;   // position of this tree in the model (sampling seed)
  uint32_t* d_absmax = b->d_absmax.p + 2 * k;
  if (p.subsample < 1.0f) {
    LAUNCH_CHECK(b2_launch_subsample(b->gh.p + (size_t)k * n, n, (uint32_t)p.seed, tree_index, b->comm ? (uint32_t)b->comm->rank : 0u,
                                     (double)p.subsample, ctx->num_sms, s));
    st.kernel_launches++;
  }
  // column sampling: the tree's feature set and one nested set per level are drawn on the host (they depend on
  // (seed, tree, level) only, never on the data), the per-node subsets inside the split-scan kernels
  std::vector<int> n_level_feats(D > 0 ? D : 1, m->F);
  if (p.use_cols()) {
    const int F = m->F;
    const uint32_t* fwq = m->fwq.empty() ? nullptr : m->fwq.data();
    std::vector<uint8_t> mask_tree(F), masks((size_t)std::max(D, 1) * F);
    for (int f = 0; f < F; ++f)
      mask_tree[f] = b2_col_selected((uint32_t)p.seed, tree_index, B2_SCOPE_TREE, f, nullptr, fwq, F, b2_sample_count((double)p.colsample_bytree, F));
    int n_tree = 0; for (int f = 0; f < F; ++f) n_tree += mask_tree[f];
    for (int d = 0; d < D; ++d) {
      int cnt = 0;
      for (int f = 0; f < F; ++f) {
        masks[(size_t)d * F + f] = b2_col_selected((uint32_t)p.seed, tree_index, B2_SCOPE_LEVEL(d), f, mask_tree.data(), fwq, F,
                                                   b2_sample_count((double)p.colsample_bylevel, n_tree));
        cnt += masks[(size_t)d * F + f];
      }
      n_level_feats[d] = cnt;
    }
    b->d_col_masks.ensure(masks.size());
    CUDA_CHECK(cudaMemcpyAsync(b->d_col_masks.p, masks.data(), masks.size(), cudaMemcpyHostToDevice, s));   // pageable source: staged before return
  }
  if (!b->absmax_fused) {   // custom objective / row sampling / many classes: |g|,|h| maxima in their own pass
    CUDA_CHECK(cudaMemsetAsync(d_absmax, 0, 2 * sizeof(uint32_t), s));
    LAUNCH_CHECK(b2_launch_absmax(gh, n, d_absmax, ctx->num_sms, s));
    st.kernel_launches++;
  }
  if (p2p) LAUNCH_CHECK(b2_launch_p2p_quant_exponent(&b->p2p.pp, d_absmax, b->d_qexp.p, s));
  else {
    allreduce(b->comm, d_absmax, 2, kNcclUint32, kNcclMax, s);
    LAUNCH_CHECK(b2_launch_quant_exponent(d_absmax, b->d_qexp.p, s));
  }
  LAUNCH_CHECK(b2_launch_quantize(gh, n, b->d_qexp.p, p.qbits, b->q.p, ctx->num_sms, s));
  st.kernel_launches += 2;

  B2TrainParamDev dp;
  dp.min_child_weight = (double)p.min_child_weight; dp.lambda = (double)p.lambda; dp.alpha = (double)p.alpha;
  dp.inv_scale_g = dp.inv_scale_h = 1.0;
  dp.max_cat_to_onehot = p.max_cat_to_onehot; dp.max_cat_threshold = p.max_cat_threshold;
  dp.max_delta_step = (double)p.max_delta_step;
  B2CtlParams cp; cp.mcw = dp.min_child_weight; cp.lambda = dp.lambda; cp.alpha = dp.alpha; cp.max_delta_step = dp.max_delta_step; cp.gamma = p.gamma; cp.eta = p.eta / (float)p.num_parallel_tree;
  const B2TreeDev tree = tree_dev(b);
  int32_t* d_n_leaves = tree.n_nodes + 1;
  long long* d_level_rows = b->t_i64.p + 2 * L.max_nodes;
  B2LevelCtl* ctl = b->d_ctl.p;
  const int window = window_rows_for(p.qbits);
  const int n_streams = std::max(1, ctx->num_sms * 3 / G);
  const int pchunk = b2_split_chunk_rows(), lchunk = b2_part_chunk_rows();
  const int max_part_chunks_total = (int)((n + pchunk - 1) / pchunk);   // + nodes of the level: upper bound of the split work items
  const size_t lcap = (size_t)1 << D;
  const int max_leaf_chunks = (int)((n + lchunk - 1) / lchunk) + (int)lcap;

  LAUNCH_CHECK(b2_launch_tree_init(tree, ctl, b->d_seg[0].p, b->d_ev[0].p, d_n_leaves, (int)n, b->d_hist_work.p, s));
  CUDA_CHECK(cudaMemsetAsync(b->d_leaf_sums.p, 0, 2 * lcap * sizeof(long long), s));
  mark_phase(b, 0);
  // ---- root histogram (no gather; row count known on the host)
  const int sh = b->log2_shards;
  const int shard_rank = b->shards > 1 ? b->comm->rank : 0;
  CUDA_CHECK(cudaMemsetAsync(build_target(b, b->hist[0].p), 0, b->node_elems * sizeof(long long), s));
  {
    const int chunk_rows = pick_chunk_rows(b, n);
    const int chunks = (int)((n + chunk_rows - 1) / chunk_rows);
    if (n > 0) {
      cudaEvent_t e0 = nullptr, e1 = nullptr;
      record_hist_launch(b, st, e0, e1, true);
      if (use_tma_hist() && m->has_tmap)
        LAUNCH_CHECK(b2_launch_hist_tma(m->bins.p, m->row_stride, m->tmap_tile, b->q.p, nullptr, b->d_hist_work.p, 1, chunks, chunk_rows, window, G,
                                        build_target(b, b->hist[0].p), nullptr, sh, 1, n, ctx->num_sms, s));
      else
        LAUNCH_CHECK(b2_launch_hist(m->bins.p, m->row_stride, b->q.p, nullptr, b->d_hist_work.p, 1, chunks, chunk_rows, window, G,
                                    build_target(b, b->hist[0].p), nullptr, sh, 1, m->narrow_w, ctx->num_sms, s));
      record_hist_launch(b, st, e0, e1, false);
      st.hist_launches++; st.kernel_launches++;
    }
  }
  mark_phase(b, 1);
  exchange_and_subtract(b, st, nullptr, b->hist[0].p, nullptr, nullptr, 1, 1);
  LAUNCH_CHECK(b2_launch_root_totals(b->hist[0].p, G, b->d_ev[0].p, b->d_qexp.p, p.qbits, dp, sh, tree.sum_g, tree.sum_h, s));
  st.kernel_launches += 2;
  int hb = 0;  // hist buffer holding the current level
  for (int d = 0; d <= D; ++d) {
    const int cur = d & 1, nxt = cur ^ 1;
    const int max_nodes_level = 1 << d;
    const bool can_split = d < D;
    const bool last_split_level = d == D - 1;
    // candidates per node of this level: the scan's CTAs per node (its layout depends on the node count) + categorical
    const int cpn_num = b2_eval_ctas_per_node(G, sh, max_nodes_level);
    const int cpn = cpn_num + (m->any_cat() ? b2_cat_ctas() : 0);
    B2DecideArgs da;
    da.ctl_cur = ctl + cur; da.ctl_nxt = ctl + nxt; da.seg_cur = b->d_seg[cur].p; da.seg_nxt = b->d_seg[nxt].p;
    da.ev_cur = b->d_ev[cur].p; da.ev_nxt = b->d_ev[nxt].p;
    da.cands = b->d_cands.p; da.cand_best = b->d_cand_best.p; da.local_cands = b->d_cands.p;
    da.tree = tree; da.split_work = b->d_split_work.p; da.pair_parent_hist = b->d_pair_parent.p; da.leaves = b->d_leaves.p;
    da.n_leaves = d_n_leaves; da.has_missing = m->d_has_missing.p; da.qexp = b->d_qexp.p;
    da.part_counters = can_split ? b->d_counters.p : nullptr; da.p = cp;
    da.cands_per_node = cpn; da.cand_ranks = b->shards; da.cand_rank_stride = max_nodes_level * cpn;
    da.can_split = can_split ? 1 : 0; da.qbits = p.qbits;
    // one GPU, numeric features only, levels scanned by the narrow layout: the last CTA of the scan decides the level
    // (no decide launch)
    const bool fold_decide = can_split && !multi && !m->any_cat() && max_nodes_level <= b2_eval_narrow_max_nodes();
    if (can_split) {
      B2ColSample cs;
      cs.level_mask = p.use_cols() ? b->d_col_masks.p + (size_t)d * m->F : nullptr;
      cs.fwq = m->fwq.empty() ? nullptr : m->d_fwq.p;
      cs.bynode = (double)p.colsample_bynode; cs.n_level = n_level_feats[d]; cs.n_features = m->F;
      cs.seed = (uint32_t)p.seed; cs.tree = p.use_cols() ? tree_index : 0u;
      // siblings of this level: parent (previous level buffer) - built, formed in the scan; stored only when the next
      // level takes them as parents
      B2SiblingSub sub{nullptr, nullptr, nullptr, 0};
      if (sub_in_scan && d > 0) {
        sub.parent_level = b->hist[hb ^ 1].p; sub.triples = b->d_triples.p;
        sub.sib_out = d + 1 < D ? b->hist[hb].p : nullptr; sub.sib_base = max_nodes_level / 2;
      }
      LAUNCH_CHECK(b2_launch_eval_splits(b->hist[hb].p, G, b->d_ev[cur].p, max_nodes_level, m->d_group_first.p, m->d_group_size.p,
                                         m->d_nbins.p, m->d_has_missing.p, m->any_cat() ? m->d_is_cat.p : nullptr, b->d_qexp.p,
                                         p.qbits, dp, b->d_cands.p, cpn, ctl + cur, sh, shard_rank, cs, b->d_seg[cur].p, sub,
                                         fold_decide ? &da : nullptr, b->d_eval_done.p, s));
      st.kernel_launches++;
      if (m->any_cat()) {
        LAUNCH_CHECK(b2_launch_eval_cat_splits(b->hist[hb].p, G, b->d_ev[cur].p, max_nodes_level, m->d_cat_feats.p,
                                               (int)m->cat_feats.size(), m->d_feat_byte.p, m->d_nbins.p, b->d_qexp.p, p.qbits, dp,
                                               b->d_cands.p, cpn, cpn_num, ctl + cur, sh, shard_rank, cs, b->d_seg[cur].p, s));
        st.kernel_launches++;
      }
      if (p2p) {   // decide_kernel stores the candidates straight into the peers' tables and waits for theirs
        da.cands = b->d_cands_all.p;
        da.cand_rank_stride = b->p2p.cand_cap;
      } else if (b->shards > 1) {   // every rank scanned only its own slots: gather the per-node candidates
        const size_t bytes = (size_t)max_nodes_level * cpn * sizeof(B2SplitCand);
        NCCL_CHECK(nccl()->AllGather(b->d_cands.p, b->d_cands_all.p, bytes, kNcclUint8, b->comm->comm, s));
        da.cands = b->d_cands_all.p;
      }
    }
    if (!fold_decide) {
      LAUNCH_CHECK(b2_launch_decide(&da, (p2p && can_split) ? &b->p2p.pp : nullptr, s));
      st.kernel_launches++;
    }
    mark_phase(b, 4);
    if (!can_split) break;
    const int32_t* ridx_in = d == 0 ? nullptr : b->ridx[cur].p;   // the root's rows are the identity list
    if (last_split_level && leaf_fused) {
      // ---- the children of this level are leaves: no ordered index lists any more.  Leaves that stopped earlier get
      // their rows' leaf index from their segments, rows of the nodes that split here are assigned in one pass
      // (partition_kernel.cu).  With leaf_stream the sums are left to leaf_accumulate_kernel after the last decide.
      long long* sums = leaf_stream ? nullptr : b->d_leaf_sums.p;
      LAUNCH_CHECK(b2_launch_leaf_plan(b->d_leaves.p, &ctl[cur].leaf_base_next, b->d_seg_work.p, ctl + 2, s));
      LAUNCH_CHECK(b2_launch_leaf_sums(gh, b->ridx[0].p, b->ridx[1].p, b->d_seg_work.p, ctl + 2, max_leaf_chunks, b->d_qexp.p, 40,
                                       sums, b->pos.p, ctx->num_sms, s));
      LAUNCH_CHECK(b2_launch_final_assign(m->bins_col.p, m->col_stride, ridx_in, b->d_split_work.p, ctl + cur,
                                          max_part_chunks_total + max_nodes_level, gh, b->d_qexp.p, 40, sums, b->pos.p,
                                          m->any_cat() ? 1 : 0, ctx->num_sms, s));
      st.kernel_launches += 3;
      mark_phase(b, 5);
      continue;
    }
    // ---- partition rows of the expanding nodes into the other index list (decide zeroed the counters); the last CTA
    // of the partition finalises the level: child segments, build-child choice, next histogram work list
    const bool need_hist = d + 1 < D;
    B2FinalizeArgs fin;
    fin.ctl_nxt = ctl + nxt; fin.seg_nxt = b->d_seg[nxt].p; fin.ev_nxt = b->d_ev[nxt].p; fin.pair_parent_hist = b->d_pair_parent.p;
    fin.hist_work = b->d_hist_work.p; fin.triples = b->d_triples.p; fin.stat_rows = d_level_rows + d + 1; fin.done = b->d_part_done.p;
    fin.max_pairs = max_nodes_level; fin.need_hist = need_hist ? 1 : 0; fin.n_streams = n_streams; fin.window_rows = window;
    fin.chunk_rows_override = p.hist_chunk_rows;
    LAUNCH_CHECK(b2_launch_partition(m->bins_col.p, m->col_stride, ridx_in, b->ridx[nxt].p, b->d_split_work.p, ctl + cur,
                                     max_part_chunks_total + max_nodes_level, b->d_counters.p, m->any_cat() ? 1 : 0, fin,
                                     ctx->num_sms, s));
    st.kernel_launches++;
    mark_phase(b, 5);
    if (need_hist) {
      // ---- histograms of level d+1: built children in slots [0, 2^d), siblings in [2^d, 2^(d+1))
      const int nh = hb ^ 1;
      long long* tgt = build_target(b, b->hist[nh].p);
      // (peer-memory exchange: every peer finished reading this rank's build buffer before it published the candidates
      // that the decide kernel above waited for, so the buffer can be zeroed here without another handshake)
      CUDA_CHECK(cudaMemsetAsync(tgt, 0, (size_t)max_nodes_level * b->node_elems * sizeof(long long), s));
      cudaEvent_t e0 = nullptr, e1 = nullptr;
      record_hist_launch(b, st, e0, e1, true);
      if (use_tma_hist() && m->has_tmap)
        LAUNCH_CHECK(b2_launch_hist_tma(m->bins.p, m->row_stride, m->tmap_tile, b->q.p, b->ridx[nxt].p, b->d_hist_work.p, 0, 0, 0, window, G, tgt, ctl + nxt, sh,
                                        max_nodes_level, n, ctx->num_sms, s));
      else
        LAUNCH_CHECK(b2_launch_hist(m->bins.p, m->row_stride, b->q.p, b->ridx[nxt].p, b->d_hist_work.p, 0, 0, 0, window, G, tgt,
                                    ctl + nxt, sh, max_nodes_level, m->narrow_w, ctx->num_sms, s));
      record_hist_launch(b, st, e0, e1, false);
      st.hist_launches++; st.kernel_launches++;
      mark_phase(b, 1);
      exchange_and_subtract(b, st, b->hist[hb].p, b->hist[nh].p, sub_in_scan ? nullptr : b->d_triples.p, ctl + nxt,
                            max_nodes_level, max_nodes_level);
      hb = nh;
    }
  }
  // ---- leaves: 40-bit fixed-point leaf sums -> sum over the ranks -> weights -> margin update
  if (!leaf_fused) {
    LAUNCH_CHECK(b2_launch_leaf_plan(b->d_leaves.p, d_n_leaves, b->d_seg_work.p, ctl + 2, s));
    LAUNCH_CHECK(b2_launch_leaf_sums(gh, b->ridx[0].p, b->ridx[1].p, b->d_seg_work.p, ctl + 2, max_leaf_chunks, b->d_qexp.p, 40,
                                     b->d_leaf_sums.p, nullptr, ctx->num_sms, s));
    st.kernel_launches += 2;
  } else if (leaf_stream) {   // every row's leaf index is in pos: sum the leaves in row order
    LAUNCH_CHECK(b2_launch_leaf_accumulate(gh, b->pos.p, n, D, b->d_qexp.p, 40, b->d_leaf_sums.p, ctx->num_sms, s));
    st.kernel_launches++;
  }
  if (p2p) { LAUNCH_CHECK(b2_launch_p2p_leaf_sums(&b->p2p.pp, d_n_leaves, b->d_leaf_sums.p, s)); st.kernel_launches++; }
  else allreduce(b->comm, b->d_leaf_sums.p, 2 * lcap, kNcclInt64, kNcclSum, s);
  LAUNCH_CHECK(b2_launch_leaf_values(b->d_leaves.p, d_n_leaves, b->d_leaf_sums.p, b->d_qexp.p, 40, cp, b->d_leaf_values.p, tree, b->t_qexp.p, s));
  if (leaf_fused)
    LAUNCH_CHECK(b2_launch_margin_update(b->margin.p, K, k, b->pos.p, b->d_leaf_values.p, n, ctx->num_sms, s));
  else
    LAUNCH_CHECK(b2_launch_pred_update(b->margin.p, K, k, b->ridx[0].p, b->ridx[1].p, b->d_seg_work.p, ctl + 2, max_leaf_chunks,
                                       b->d_leaf_values.p, ctx->num_sms, s));
  st.kernel_launches += 2;
  mark_phase(b, 6);
  // ---- read the finished tree back (pinned, asynchronous; resolved at the end of the round)
  char* stg = (char*)b->staging[slot];
  // one copy: the category sets (the block's tail) only when the matrix has categorical features
  CUDA_CHECK(cudaMemcpyAsync(stg, b->t_block.p, m->any_cat() ? L.bytes : L.off_cat, cudaMemcpyDeviceToHost, s));
}

void apply_tree_stats(Booster* b, long long hist_launches, long long kernel_launches, double allreduce_bytes,
                      const std::vector<std::pair<cudaEvent_t, cudaEvent_t>>& ev) {
  b->t.hist_launches += hist_launches; b->t.kernel_launches += kernel_launches; b->t.allreduce_bytes += allreduce_bytes;
  for (auto& pr : ev) b->hist_events.push_back(pr);
}

// buffers a tree needs, allocated outside of any capture
void prepare_tree_buffers(Booster* b, int slot) {
  Matrix* m = b->train; const int64_t n = m->n;
  ensure_ctl_tables(b);
  const TreeLayout L = tree_layout(b->p.max_depth);
  const size_t rows = (size_t)std::max<int64_t>(n, 1);
  b->d_absmax.ensure(2 * (size_t)b->p.num_class); b->d_qexp.ensure(2);
  b->q.ensure(rows); b->ridx[0].ensure(rows); b->ridx[1].ensure(rows); b->pos.ensure(rows);
  if (b->staging_bytes != L.bytes) {
    for (void* h : b->staging) cudaFreeHost(h);
    b->staging.clear(); b->staging_bytes = L.bytes;
  }
  while ((int)b->staging.size() <= slot) { void* h = nullptr; CUDA_CHECK(cudaMallocHost(&h, L.bytes)); b->staging.push_back(h); }
}

// One class tree: replay its CUDA graph when the launch sequence is the same for every tree (no row / column sampling,
// fused |g|,|h| maxima, no per-phase profiling), otherwise enqueue the kernels one by one.  The first tree of a class
// slot always runs with direct launches (it allocates), the second is captured, the following ones replay.
void run_tree(Booster* b, int k, int slot) {
  cudaStream_t s = b->ctx->stream; const Params& p = b->p;
  prepare_tree_buffers(b, slot);
  static const bool want_graph = env_flag("B2_GRAPH", true);
  const bool eligible = want_graph && !b->graph_failed && b->absmax_fused && p.subsample >= 1.0f && !p.use_cols() &&
                        p.profile < 2 && !use_tma_hist() && p.num_parallel_tree == 1;
  auto direct = [&]() {
    TreeStats st;
    grow_tree(b, k, slot, st);
    apply_tree_stats(b, st.hist_launches, st.kernel_launches, st.allreduce_bytes, st.hist_ev);
    b->direct_trees[k]++;
  };
  if (!eligible) { direct(); return; }
  auto it = b->graphs.find(k);
  if (it == b->graphs.end()) {
    if (b->direct_trees[k] == 0) { direct(); return; }
    TreeStats st; st.capturing = true;
    cudaGraph_t graph = nullptr; cudaGraphExec_t exec = nullptr;
    bool ok = cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
    if (ok) {
      try { grow_tree(b, k, slot, st); }
      catch (const B2Error& e) { cudaStreamEndCapture(s, &graph); if (graph) cudaGraphDestroy(graph); cudaGetLastError(); throw; }
      ok = cudaStreamEndCapture(s, &graph) == cudaSuccess && graph != nullptr;
    }
    if (ok) ok = cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess;
    if (graph) cudaGraphDestroy(graph);
    if (!ok) {
      cudaGetLastError();
      for (auto& pr : st.hist_ev) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
      b->graph_failed = true;
      fprintf(stderr, "[b2hist] CUDA graph capture of the tree failed; continuing with direct launches\n");
      direct();
      return;
    }
    Booster::TreeGraph g;
    g.exec = exec; g.hist_ev = st.hist_ev; g.hist_launches = st.hist_launches; g.kernel_launches = st.kernel_launches;
    g.allreduce_bytes = st.allreduce_bytes;
    it = b->graphs.emplace(k, std::move(g)).first;
  }
  CUDA_CHECK(cudaGraphLaunch(it->second.exec, s));
  apply_tree_stats(b, it->second.hist_launches, it->second.kernel_launches, it->second.allreduce_bytes, it->second.hist_ev);
}

// after the stream is synchronised: turn read-back block `slot` into a host tree (A.7 bookkeeping)
void materialize_tree(Booster* b, int slot) {
  Matrix* m = b->train; const Params& p = b->p;
  const TreeLayout L = tree_layout(p.max_depth);
  const char* st = (const char*)b->staging[slot];
  const int32_t* i32 = (const int32_t*)st; const size_t mx = L.max_nodes;
  const float* f32 = (const float*)(st + L.off_f32);
  const long long* i64 = (const long long*)(st + L.off_i64);
  const int32_t* qexp = (const int32_t*)(st + L.off_qexp);
  const int nn = i32[7 * mx];
  const uint32_t* cat = (const uint32_t*)(st + L.off_cat);
  if (nn < 1 || (size_t)nn > mx) fail("corrupt tree read-back (n_nodes=%d)", nn);
  const double inv_sg = ldexp(1.0, qexp[0] - p.qbits), inv_sh = ldexp(1.0, qexp[1] - p.qbits);
  TreeHost t;
  for (int i = 0; i < nn; ++i) {
    t.add(i32[2 * mx + i]);
    t.left[i] = i32[i]; t.right[i] = i32[mx + i]; t.feature[i] = i32[3 * mx + i];
    const double G = (double)i64[i] * inv_sg, H = (double)i64[mx + i] * inv_sh;
    t.sum_hess[i] = H;
    if (t.feature[i] >= 0) {
      const int f = t.feature[i], bin = i32[4 * mx + i];
      t.split_bin[i] = bin; t.default_left[i] = (uint8_t)i32[5 * mx + i]; t.loss_chg[i] = f32[i];
      if (m->any_cat() && i32[6 * mx + i]) {
        // categorical split: one-hot keeps the category as split condition, a partition split stores NaN (RegTree::ExpandCategorical)
        t.split_type[i] = 1; t.any_cat = true;
        for (int w8 = 0; w8 < 8; ++w8) t.cat_bits[(size_t)i * 8 + w8] = cat[(size_t)i * 8 + w8];
        t.cond[i] = bin >= 0 ? (float)bin : NAN;
      } else
      t.cond[i] = bin < 0 ? m->min_vals[f] : m->cut_vals[m->cut_ptrs[f] + bin];
      t.base_weight[i] = h_calc_weight(p, G, H);
      t.value[i] = t.base_weight[i];
    } else {
      t.base_weight[i] = f32[mx + i];
      t.value[i] = f32[2 * mx + i];
    }
  }
  // histogram rows of this tree for the roofline accounting: root + built children per level
  const long long* level_rows = i64 + 2 * mx;
  long long rows = m->n; int launches_nonempty = m->n > 0 ? 1 : 0;
  for (int d = 1; d < p.max_depth; ++d) { rows += level_rows[d]; if (level_rows[d] > 0) launches_nonempty++; }
  long long gathered = rows - m->n;
  int built_nodes = 0;
  for (int i = 0; i < nn; ++i) if (t.feature[i] >= 0) built_nodes++;   // one built child per split (+ root)
  b->t.hist_rows += rows;
  b->t.hist_bytes += (double)rows * (m->F + 8) + (double)gathered * 4 + (double)(built_nodes + 1) * m->F * 256.0 * 16.0;
  b->trees.push_back(std::move(t));
}

void sync_device_trees(Booster* b) {
  if (b->d_trees_synced == (int)b->trees.size()) return;
  b->h_nodes.clear(); b->h_tree_offset.clear(); b->h_cat_table.clear();
  for (auto& t : b->trees) {
    b->h_tree_offset.push_back((int32_t)b->h_nodes.size());
    for (int i = 0; i < t.size(); ++i) {
      int32_t cat_slot = -1;
      if (t.feature[i] >= 0 && t.split_type[i]) {
        cat_slot = (int32_t)(b->h_cat_table.size() / 8);
        b->h_cat_table.insert(b->h_cat_table.end(), t.cat_bits.begin() + (size_t)i * 8, t.cat_bits.begin() + (size_t)i * 8 + 8);
      }
      b->h_nodes.push_back(B2TreeNodeDev{t.left[i], t.right[i], t.feature[i], t.cond[i], t.value[i], (int32_t)t.default_left[i],
                                         cat_slot, 0});
    }
  }
  cudaStream_t s = b->ctx->stream;
  upload(b->d_nodes, b->h_nodes, s); upload(b->d_tree_offset, b->h_tree_offset, s); upload(b->d_cat_table, b->h_cat_table, s);
  CUDA_CHECK(cudaStreamSynchronize(s));
  b->d_trees_synced = (int)b->trees.size();
}

// ---- TreeSHAP path table (common.cuh B2PathElem / B2PathInfo; shap_kernel.cu).  Walks every tree root -> leaf; on the
// way each split is merged into the element of its feature (appended the first time the feature is seen): the interval
// of a numeric feature narrows, the category set of a categorical feature is intersected with the side taken (keeping
// predict_kernel's rule that a category outside [0, 256) goes left), the missing flag is AND-ed with "the default
// direction is the side taken", and zero_fraction is multiplied by cover(child) / cover(parent) (0 for a zero-cover
// parent, never NaN).  The tree's expected value, sum over leaves of value * prod zero_fraction, is its SHAP bias.
struct PathBuildElem {
  int32_t feature; bool is_cat; float lo, hi; uint32_t flags; uint32_t bits[8]; double z;
};
void walk_paths(const TreeHost& t, int nid, std::vector<PathBuildElem>& path, int tree, int cls, Booster* b,
                std::vector<B2PathElem>& elems, std::vector<B2PathInfo>& infos, std::vector<uint32_t>& cats, double* expected) {
  if (t.feature[nid] < 0) {
    if (path.size() + 1 > B2_SHAP_MAX_PATH)
      fail("tree %d has a leaf below %d distinct features; TreeSHAP supports at most %d (max_depth <= 14)", tree,
           (int)path.size(), B2_SHAP_MAX_PATH - 1);
    B2PathInfo pi{(int32_t)elems.size(), (int32_t)path.size() + 1, cls, 0, (double)t.value[nid]};
    elems.push_back(B2PathElem{-1, -1, 0.f, 0.f, 0u, 0u, 1.0});
    double zprod = 1.0;
    for (const PathBuildElem& e : path) {
      int32_t slot = -1;
      if (e.is_cat) { slot = (int32_t)(cats.size() / 8); cats.insert(cats.end(), e.bits, e.bits + 8); }
      elems.push_back(B2PathElem{e.feature, slot, e.lo, e.hi, e.flags, 0u, e.z});
      zprod *= e.z;
    }
    *expected += (double)t.value[nid] * zprod;
    infos.push_back(pi);
    return;
  }
  const int f = t.feature[nid];
  const bool is_cat = t.split_type[nid] != 0;
  const double cover = t.sum_hess[nid];
  for (int side = 0; side < 2; ++side) {
    const int child = side == 0 ? t.left[nid] : t.right[nid];
    const bool left = side == 0;
    std::vector<PathBuildElem> next = path;
    PathBuildElem* e = nullptr;
    for (auto& x : next) if (x.feature == f) e = &x;
    if (!e) {
      PathBuildElem ne;
      ne.feature = f; ne.is_cat = is_cat; ne.lo = -INFINITY; ne.hi = INFINITY;
      ne.flags = B2_PATH_MISSING_OK | B2_PATH_OUTSIDE_OK; ne.z = 1.0;
      for (int w = 0; w < 8; ++w) ne.bits[w] = 0xffffffffu;
      next.push_back(ne); e = &next.back();
    }
    e->z *= cover > 0.0 ? t.sum_hess[child] / cover : 0.0;
    if ((t.default_left[nid] != 0) != left) e->flags &= ~B2_PATH_MISSING_OK;
    if (is_cat) {
      e->is_cat = true;
      for (int w = 0; w < 8; ++w) e->bits[w] &= left ? ~t.cat_bits[(size_t)nid * 8 + w] : t.cat_bits[(size_t)nid * 8 + w];
      if (!left) e->flags &= ~B2_PATH_OUTSIDE_OK;
    } else if (left) {
      if (!(e->flags & B2_PATH_HAS_HI) || t.cond[nid] < e->hi) e->hi = t.cond[nid];
      e->flags |= B2_PATH_HAS_HI;
    } else if (t.cond[nid] > e->lo) {
      e->lo = t.cond[nid];
    }
    walk_paths(t, child, next, tree, cls, b, elems, infos, cats, expected);
  }
}

void build_paths(Booster* b) {
  if (b->paths_synced == (int)b->trees.size()) return;
  std::vector<B2PathElem> elems; std::vector<B2PathInfo> infos; std::vector<uint32_t> cats;
  b->tree_path_offset.assign(1, 0); b->tree_expected.clear();
  const int K = b->p.num_class, npt = std::max(1, b->p.num_parallel_tree);
  for (int t = 0; t < (int)b->trees.size(); ++t) {
    std::vector<PathBuildElem> path;
    double expected = 0.0;
    walk_paths(b->trees[t], 0, path, t, (t / npt) % K, b, elems, infos, cats, &expected);
    b->tree_path_offset.push_back((int32_t)infos.size());
    b->tree_expected.push_back(expected);
  }
  cudaStream_t s = b->ctx->stream;
  upload(b->d_path_elems, elems, s); upload(b->d_paths, infos, s); upload(b->d_path_cats, cats, s);
  CUDA_CHECK(cudaStreamSynchronize(s));
  b->paths_synced = (int)b->trees.size();
}

void init_margin(Booster* b, float* margin, Matrix* m) {
  const int K = b->p.num_class; cudaStream_t s = b->ctx->stream;
  if (m->n_base_margin > 0) {
    if (m->n_base_margin != m->n * K) fail("base_margin has %lld values, expected %lld", (long long)m->n_base_margin, (long long)(m->n * K));
    CUDA_CHECK(cudaMemcpyAsync(margin, m->base_margin.p, (size_t)m->n * K * sizeof(float), cudaMemcpyDeviceToDevice, s));
  } else {
    LAUNCH_CHECK(b2_launch_fill(margin, m->n * K, base_margin_value(b->p), b->ctx->num_sms, s));
  }
}

// base_score when the user gave none (xgboost >= 2.0: ObjFunction::InitEstimation -> FitIntercept, tree::FitStump;
// SURVEY.md A.3): one Newton step of a stump at margin 0, -sum(g)/sum(h) over ALL workers, then the inverse link.
// Sums are 40-bit fixed-point integers, so every rank (and the oracle) computes the same value.
void estimate_base_score(Booster* b) {
  Matrix* m = b->train; cudaStream_t s = b->ctx->stream; Params& p = b->p;
  if (p.base_score_set || p.objective == kObjSoftprob) { p.base_score_set = true; return; }
  // existing trees were fitted around the intercept of the model they came from: never assume the default for them
  if (!b->trees.empty()) fail("continuing from existing trees needs an explicit base_score (the source model's intercept)");
  if (m->n_label != m->n) fail("train matrix has %lld labels for %lld rows", (long long)m->n_label, (long long)m->n);
  const int64_t n = m->n;
  DevBuf<float> zeros; DevBuf<float2> gh; DevBuf<long long> sums;
  zeros.ensure((size_t)std::max<int64_t>(n, 1)); gh.ensure((size_t)std::max<int64_t>(n, 1)); sums.ensure(2);
  CUDA_CHECK(cudaMemsetAsync(zeros.p, 0, (size_t)std::max<int64_t>(n, 1) * sizeof(float), s));
  LAUNCH_CHECK(b2_launch_gradient(p.objective, 1, zeros.p, m->label.p, m->n_weight ? m->weight.p : nullptr, n, p.scale_pos_weight,
                                  objective_param(p), gh.p, nullptr, nullptr, b->ctx->num_sms, s));
  b->d_absmax.ensure(2); b->d_qexp.ensure(2);
  CUDA_CHECK(cudaMemsetAsync(b->d_absmax.p, 0, 2 * sizeof(uint32_t), s));
  LAUNCH_CHECK(b2_launch_absmax(gh.p, n, b->d_absmax.p, b->ctx->num_sms, s));
  allreduce(b->comm, b->d_absmax.p, 2, kNcclUint32, kNcclMax, s);
  LAUNCH_CHECK(b2_launch_quant_exponent(b->d_absmax.p, b->d_qexp.p, s));
  CUDA_CHECK(cudaMemsetAsync(sums.p, 0, 2 * sizeof(long long), s));
  LAUNCH_CHECK(b2_launch_sum_fixed(gh.p, n, b->d_qexp.p, 40, sums.p, b->ctx->num_sms, s));
  allreduce(b->comm, sums.p, 2, kNcclInt64, kNcclSum, s);
  long long h_s[2]; int32_t h_e[2];
  CUDA_CHECK(cudaMemcpyAsync(h_s, sums.p, sizeof(h_s), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaMemcpyAsync(h_e, b->d_qexp.p, sizeof(h_e), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  const double G = (double)h_s[0] / ldexp(1.0, 40 - h_e[0]), H = (double)h_s[1] / ldexp(1.0, 40 - h_e[1]);
  const float stump = H <= 1e-6 ? 0.0f : (float)(-G / H);
  if (obj_sigmoid(p.objective) || obj_log_link(p.objective)) {
    // margin -> output space with the engine's own sigmoid / exp (same IEEE sequence as the kernels): evaluated on the device
    DevBuf<float> one; one.ensure(1);
    CUDA_CHECK(cudaMemcpyAsync(one.p, &stump, sizeof(float), cudaMemcpyHostToDevice, s));
    LAUNCH_CHECK(b2_launch_transform(p.objective, 1, one.p, 1, b->ctx->num_sms, s));
    float prob = 0.5f;
    CUDA_CHECK(cudaMemcpyAsync(&prob, one.p, sizeof(float), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    p.base_score = prob;
  } else {
    p.base_score = stump;
  }
  p.base_score_set = true;
}

// survival:aft reads the label bounds instead of the label: both present, no NaN, 0 <= lower (finite) <= upper, and an
// uncensored row (lower == upper) needs y > 0.  Once per train matrix, like check_labels.
void check_bounds(Booster* b) {
  Matrix* m = b->train; cudaStream_t s = b->ctx->stream;
  if (b->labels_checked) return;
  if (!m->has_bounds()) fail("survival:aft needs label_lower_bound and label_upper_bound");
  DevBuf<uint32_t> bad; bad.ensure(4);
  CUDA_CHECK(cudaMemsetAsync(bad.p, 0, 4 * sizeof(uint32_t), s));
  LAUNCH_CHECK(b2_launch_aft_bounds_check(m->lower.p, m->upper.p, m->n, bad.p, b->ctx->num_sms, s));
  allreduce(b->comm, bad.p, 4, kNcclUint32, kNcclMax, s);
  uint32_t h[4] = {0, 0, 0, 0};
  CUDA_CHECK(cudaMemcpyAsync(h, bad.p, sizeof(h), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  if (h[0]) fail("survival:aft: label bounds must not be NaN");
  if (h[1]) fail("survival:aft: label_lower_bound must be finite and >= 0");
  if (h[2]) fail("survival:aft: label_upper_bound must be >= label_lower_bound");
  if (h[3]) fail("survival:aft: an uncensored row (lower == upper) needs a label > 0");
  b->labels_checked = true;
}

// the rank objectives need query groups and labels that are finite, >= 0 and, with the exponential gain, <= 31
void check_rank_labels(Booster* b) {
  Matrix* m = b->train; cudaStream_t s = b->ctx->stream;
  if (!m->has_qgroups())
    fail("%s needs query groups on the train matrix: pass qid (or group) to the DMatrix", b->p.objective_name.c_str());
  if (b->labels_checked) return;
  if (m->n_label != m->n) fail("train matrix has %lld labels for %lld rows", (long long)m->n_label, (long long)m->n);
  DevBuf<uint32_t> bad; bad.ensure(2);
  CUDA_CHECK(cudaMemsetAsync(bad.p, 0, 2 * sizeof(uint32_t), s));
  LAUNCH_CHECK(b2_launch_rank_label_check(m->label.p, m->n, b->p.ndcg_exp_gain ? 1 : 0, bad.p, b->ctx->num_sms, s));
  allreduce(b->comm, bad.p, 2, kNcclUint32, kNcclMax, s);
  uint32_t h[2] = {0, 0};
  CUDA_CHECK(cudaMemcpyAsync(h, bad.p, sizeof(h), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  if (h[0]) fail("%s: labels must be finite and >= 0", b->p.objective_name.c_str());
  if (h[1]) fail("%s: with ndcg_exp_gain the labels must be <= 31 (the gain is 2^label - 1); set ndcg_exp_gain=false "
                 "for larger relevance degrees", b->p.objective_name.c_str());
  b->labels_checked = true;
}

// discount table ln2 / log(r + 2) for model positions r < len
void ensure_rank_disc(Booster* b, int64_t len) {
  len = std::max<int64_t>(len, 1);
  if (b->rank_disc_len >= len) return;
  b->rank_disc.ensure((size_t)len);
  LAUNCH_CHECK(b2_launch_rank_disc(b->rank_disc.p, len, b->ctx->num_sms, b->ctx->stream));
  b->rank_disc_len = len;
}

// LambdaMART gradients of the train matrix (rank_kernel.cu): order the margins per group, then one pass over the groups
void rank_gradient(Booster* b, uint32_t* absmax, uint32_t* err) {
  Matrix* m = b->train; cudaStream_t s = b->ctx->stream; const Params& p = b->p; const int sms = b->ctx->num_sms;
  ensure_rank_disc(b, m->max_qgroup);
  const bool ndcg = p.objective == kObjRankNdcg;
  if (ndcg && (b->idcg_uid != m->uid || b->idcg_version != m->rank_version || b->idcg_k != p.rank_k ||
               b->idcg_gain != (int)p.ndcg_exp_gain)) {
    // 1/IDCG depends on the labels, k and the gain only: computed once per (matrix, k, gain)
    RankOrder lo;
    lo.run(m, m->label.p, sms, s);
    b->rank_inv_idcg.ensure((size_t)std::max<int64_t>(m->n_qgroups, 1));
    LAUNCH_CHECK(b2_launch_rank_inv_idcg(m->qgroup_ptr.p, m->n_qgroups, lo.keys_sorted.p, b->rank_disc.p, p.rank_k,
                                         p.ndcg_exp_gain ? 1 : 0, b->rank_inv_idcg.p, sms, s));
    CUDA_CHECK(cudaStreamSynchronize(s));   // lo's buffers go back to the pool
    b->idcg_uid = m->uid; b->idcg_version = m->rank_version; b->idcg_k = p.rank_k; b->idcg_gain = (int)p.ndcg_exp_gain;
  }
  b->rank_order.run(m, b->margin.p, sms, s);
  if (m->max_qgroup > b2_rank_stage_rows()) {
    const size_t rows = (size_t)std::max<int64_t>(m->n, 1);
    b->rank_scratch_m.ensure(rows); b->rank_scratch_y.ensure(rows); b->rank_scratch_p.ensure(rows);
  }
  LAUNCH_CHECK(b2_launch_lambdarank_gradient(ndcg ? 1 : 0, m->qgroup_ptr.p, m->n_qgroups, m->max_qgroup,
                                             b->rank_order.keys_sorted.p, b->rank_order.rows.p, m->label.p,
                                             ndcg ? b->rank_inv_idcg.p : nullptr, b->rank_disc.p, p.rank_k,
                                             p.ndcg_exp_gain ? 1 : 0, b->rank_scratch_m.p, b->rank_scratch_y.p,
                                             b->rank_scratch_p.p, b->gh.p, absmax, err, sms, s));
}

// labels outside the objective's domain fail training (xgboost's CheckLabel); once per train matrix, before the first tree
void check_labels(Booster* b) {
  Matrix* m = b->train; const int o = b->p.objective; cudaStream_t s = b->ctx->stream;
  if (o == kObjAft) { check_bounds(b); return; }
  if (obj_rank(o)) { check_rank_labels(b); return; }
  if (o == kObjSquaredError || o == kObjLogistic || o == kObjPseudoHuber || b->labels_checked) return;
  if (m->n_label != m->n) fail("train matrix has %lld labels for %lld rows", (long long)m->n_label, (long long)m->n);
  DevBuf<uint32_t> bad; bad.ensure(1);
  CUDA_CHECK(cudaMemsetAsync(bad.p, 0, sizeof(uint32_t), s));
  LAUNCH_CHECK(b2_launch_label_check(o, b->p.num_class, m->label.p, m->n, bad.p, b->ctx->num_sms, s));
  allreduce(b->comm, bad.p, 1, kNcclUint32, kNcclMax, s);
  uint32_t h = 0;
  CUDA_CHECK(cudaMemcpyAsync(&h, bad.p, sizeof(h), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  if (h) {
    // a class index; non-integer labels truncate like xgboost's, NaN is rejected (xgboost lets it through)
    if (o == kObjSoftprob)
      fail("label must be in [0, num_class) for %s, num_class = %d", b->p.objective_name.c_str(), b->p.num_class);
    const char* cond = (o == kObjRegLogistic || o == kObjLogitRaw) ? "label must be in [0, 1]"
                       : o == kObjSquaredLog ? "label must be greater than -1"
                       : o == kObjGamma ? "label must be positive" : "label must be nonnegative";
    fail("%s for %s", cond, b->p.objective_name.c_str());
  }
  b->labels_checked = true;
}

void ensure_train_margin(Booster* b) {
  if (b->margin_ready) return;
  Matrix* m = b->train;
  check_labels(b);
  estimate_base_score(b);
  b->margin.ensure((size_t)std::max<int64_t>(m->n * b->p.num_class, 1));
  init_margin(b, b->margin.p, m);
  if (!b->trees.empty()) {
    if (!m->has_raw) fail("continuing training from existing trees needs the raw data of the train matrix (B2_MatrixEnsureRaw)");
    sync_device_trees(b);
    LAUNCH_CHECK(b2_launch_predict(m->raw.p, m->n, m->F, m->missing, b->d_nodes.p, b->d_tree_offset.p, b->d_cat_table.p, 0, (int)b->trees.size(),
                                   b->p.num_class, b->p.num_parallel_tree, b->margin.p, b->ctx->num_sms, b->ctx->stream));
  }
  b->margin_ready = true;
}

void boost_round(Booster* b, const float* custom_g, const float* custom_h, int64_t len) {
  if (!b->train) fail("this booster has no train matrix (prediction-only)");
  Matrix* m = b->train; cudaStream_t s = b->ctx->stream; const int K = b->p.num_class; const int64_t n = m->n;
  CUDA_CHECK(cudaSetDevice(b->ctx->device));
  if (b->cancel.load()) fail("training cancelled");
  if (!b->round_start) { CUDA_CHECK(cudaEventCreate(&b->round_start)); CUDA_CHECK(cudaEventCreate(&b->round_stop)); }
  if (b->p.profile) CUDA_CHECK(cudaEventRecord(b->round_start, s));
  ensure_train_margin(b);
  b->gh.ensure((size_t)std::max<int64_t>(n * K, 1));
  b->d_absmax.ensure(2 * (size_t)K); b->d_qexp.ensure(2);
  b->absmax_fused = false;
  bool check_finite = false;
  if (custom_g) {
    if (len != n * K) fail("custom gradient has %lld values, expected %lld", (long long)len, (long long)(n * K));
    b->d_custom_g.ensure((size_t)std::max<int64_t>(len, 1)); b->d_custom_h.ensure((size_t)std::max<int64_t>(len, 1));
    CUDA_CHECK(cudaMemcpyAsync(b->d_custom_g.p, custom_g, len * sizeof(float), cudaMemcpyHostToDevice, s));
    CUDA_CHECK(cudaMemcpyAsync(b->d_custom_h.p, custom_h, len * sizeof(float), cudaMemcpyHostToDevice, s));
    LAUNCH_CHECK(b2_launch_pack_custom(b->d_custom_g.p, b->d_custom_h.p, K, n, b->gh.p, b->ctx->num_sms, s));
  } else {
    if (b->p.objective != kObjAft && m->n_label != n)
      fail("train matrix has %lld labels for %lld rows", (long long)m->n_label, (long long)n);
    // the |g|,|h| maxima of every class tree come out of the same pass unless rows are dropped afterwards (subsample)
    b->absmax_fused = b->p.subsample >= 1.0f && K <= b2_gradient_fused_max_classes();
    if (b->absmax_fused) CUDA_CHECK(cudaMemsetAsync(b->d_absmax.p, 0, 2 * (size_t)K * sizeof(uint32_t), s));
    check_finite = obj_checks_finite(b->p.objective);
    if (check_finite) {
      if (!b->h_grad_err) { CUDA_CHECK(cudaMallocHost(&b->h_grad_err, sizeof(uint32_t))); b->d_grad_err.ensure(1); }
      CUDA_CHECK(cudaMemsetAsync(b->d_grad_err.p, 0, sizeof(uint32_t), s));
    }
    if (b->p.objective == kObjAft)
      LAUNCH_CHECK(b2_launch_gradient_aft(b->p.aft_dist, (double)b->p.aft_sigma, b->margin.p, m->lower.p, m->upper.p,
                                          m->n_weight ? m->weight.p : nullptr, n, b->gh.p,
                                          b->absmax_fused ? b->d_absmax.p : nullptr, b->d_grad_err.p, b->ctx->num_sms, s));
    else if (obj_rank(b->p.objective))
      rank_gradient(b, b->absmax_fused ? b->d_absmax.p : nullptr, b->d_grad_err.p);
    else
      LAUNCH_CHECK(b2_launch_gradient(b->p.objective, K, b->margin.p, m->label.p, m->n_weight ? m->weight.p : nullptr, n,
                                      b->p.scale_pos_weight, objective_param(b->p), b->gh.p,
                                      b->absmax_fused ? b->d_absmax.p : nullptr, check_finite ? b->d_grad_err.p : nullptr,
                                      b->ctx->num_sms, s));
  }
  b->gh_ready = true;
  b->t.kernel_launches++;
  const int npt = b->p.num_parallel_tree;
  // row sampling zeroes the dropped rows' gradient pairs in place: the parallel trees of a round each sample from the
  // round's ORIGINAL gradients, so those are kept aside and restored in front of every further tree
  const bool restore_gh = npt > 1 && b->p.subsample < 1.0f;
  if (restore_gh) {
    b->gh_round.ensure((size_t)std::max<int64_t>(n * K, 1));
    CUDA_CHECK(cudaMemcpyAsync(b->gh_round.p, b->gh.p, (size_t)n * K * sizeof(float2), cudaMemcpyDeviceToDevice, s));
  }
  for (int k = 0; k < K; ++k)
    for (int j = 0; j < npt; ++j) {
      if (restore_gh && j > 0)
        CUDA_CHECK(cudaMemcpyAsync(b->gh.p + (size_t)k * n, b->gh_round.p + (size_t)k * n, (size_t)n * sizeof(float2), cudaMemcpyDeviceToDevice, s));
      run_tree(b, k, k * npt + j);
    }
  if (check_finite) {
    // every rank fails the round together; the flag is read back with the round's own synchronisation below (pinned
    // memory: the copy is ordered on the stream)
    allreduce(b->comm, b->d_grad_err.p, 1, kNcclUint32, kNcclMax, s);
    CUDA_CHECK(cudaMemcpyAsync(b->h_grad_err, b->d_grad_err.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  }
  if (b->p.profile) {
    CUDA_CHECK(cudaEventRecord(b->round_stop, s));
    CUDA_CHECK(cudaEventSynchronize(b->round_stop));
    float ms = 0.f; CUDA_CHECK(cudaEventElapsedTime(&ms, b->round_start, b->round_stop));
    b->t.round_ms += ms;
    resolve_events(b);
  } else {
    CUDA_CHECK(cudaStreamSynchronize(s));
  }
  if (b->p2p.enabled) {
    uint32_t perr = 0;
    CUDA_CHECK(cudaMemcpy(&perr, b->p2p.pp.err, sizeof(perr), cudaMemcpyDeviceToHost));
    if (perr) fail("peer-memory exchange: %s while waiting for another rank (flag slot %u)",
                   b->comm && b->comm->aborted.load() ? "communicator aborted" : "timed out", perr - 1);
  }
  if (check_finite && *b->h_grad_err) {
    // the trees of this round were grown with those rows zeroed and are dropped; the train margin already holds their
    // leaves, so it is rebuilt from the kept trees before the next round
    b->margin_ready = false;
    fail("%s: a gradient or hessian is not finite (the margin left the range where the objective's exp is finite)",
         b->p.objective_name.c_str());
  }
  for (int slot = 0; slot < K * npt; ++slot) materialize_tree(b, slot);
  b->t.rounds++;
}

// metric id of an eval_metric name; *param receives the metric's parameter (rho of tweedie-nloglik@rho, huber_slope for mphe)
int metric_id(const char* name, const Params& p, float* param, int* minus) {
  std::string s(name ? name : "");
  *param = 0.0f; *minus = 0;
  if (s == "rmsle") return 7;
  if (s == "mape") return 8;
  if (s == "mphe") { *param = p.huber_slope; return 9; }
  if (s == "poisson-nloglik") return 10;
  if (s == "gamma-nloglik") return 11;
  if (s == "gamma-deviance") return 12;
  if (s.rfind("tweedie-nloglik", 0) == 0) {
    *param = 1.5f;   // xgboost's default when the name carries no @rho
    if (s.size() > 15) {
      char* end = nullptr;
      const std::string r = s.substr(16);
      const double v = s[15] == '@' ? strtod(r.c_str(), &end) : NAN;
      if (s[15] != '@' || r.empty() || *end != '\0' || !(v >= 1.0 && v < 2.0))
        fail("eval metric '%s': the Tweedie power must be given as tweedie-nloglik@rho with rho in [1, 2)", s.c_str());
      *param = (float)v;
    }
    return 13;
  }
  if (s == "rmse") return 0;
  if (s == "logloss") return 1;
  if (s == "error") return 2;
  if (s == "mlogloss") return 3;
  if (s == "merror") return 4;
  if (s == "mae") return 5;
  if (s == "auc") return 6;
  if (s == "aft-nloglik") return 14;
  if (s == "interval-regression-accuracy") return 15;
  // ranking metrics: ndcg[@k][-] (16), map[@k][-] (17), pre[@k][-] (18).  *param = k (0: the whole group), *minus = the
  // trailing '-' (a group without relevant rows scores 0 instead of 1)
  for (int id = 16; id <= 18; ++id) {
    const std::string base = id == 16 ? "ndcg" : id == 17 ? "map" : "pre";
    if (s.compare(0, base.size(), base) != 0) continue;
    std::string rest = s.substr(base.size());
    if (!rest.empty() && rest.back() == '-') { *minus = 1; rest.pop_back(); }
    if (rest.empty()) return id;
    char* end = nullptr;
    const long long k = rest[0] == '@' && rest.size() > 1 ? strtoll(rest.c_str() + 1, &end, 10) : -1;
    if (rest[0] != '@' || rest.size() < 2 || *end != '\0' || k < 1 || k > (1 << 24))
      fail("eval metric '%s': the cut-off must be given as %s@k with an integer k >= 1", s.c_str(), base.c_str());
    *param = (float)k;
    return id;
  }
  fail("unsupported eval metric '%s' (supported: rmse, mae, logloss, error, auc, mlogloss, merror, rmsle, mape, mphe, "
       "poisson-nloglik, gamma-nloglik, gamma-deviance, tweedie-nloglik@rho, aft-nloglik, interval-regression-accuracy, "
       "ndcg[@k][-], map[@k][-], pre[@k][-])", s.c_str());
}

// margin of matrix m under the current model (cached per matrix, only new trees are applied)
float* eval_margin(Booster* b, Matrix* m) {
  if (b->train && m == b->train) { ensure_train_margin(b); return b->margin.p; }
  if (!m->has_raw) fail("evaluation / prediction matrix has no raw data on the device");
  if (m->F != b->n_features) fail("feature count mismatch: matrix has %d, model has %d", m->F, b->n_features);
  {   // drop the cached margins of matrices that were freed since the last call
    std::lock_guard<std::mutex> lk(g_matrix_mu);
    for (auto it = b->eval_cache.begin(); it != b->eval_cache.end();) {
      if (!g_live_matrices.count(it->first)) { delete it->second; it = b->eval_cache.erase(it); } else ++it;
    }
  }
  if (!m->uid) fail("evaluation matrix is not a registered matrix handle");
  EvalCache*& c = b->eval_cache[m->uid];
  const int K = b->p.num_class;
  if (!c || c->n != m->n || c->margin_version != m->margin_version) {
    delete c; c = new EvalCache(); c->n = m->n; c->margin_version = m->margin_version;
    c->margin.ensure((size_t)std::max<int64_t>(m->n * K, 1));
    init_margin(b, c->margin.p, m);
    c->n_trees_applied = 0;
  }
  const int nt = (int)b->trees.size();
  if (c->n_trees_applied < nt) {
    sync_device_trees(b);
    LAUNCH_CHECK(b2_launch_predict(m->raw.p, m->n, m->F, m->missing, b->d_nodes.p, b->d_tree_offset.p, b->d_cat_table.p, c->n_trees_applied, nt, K, b->p.num_parallel_tree,
                                   c->margin.p, b->ctx->num_sms, b->ctx->stream));
    c->n_trees_applied = nt;
  }
  return c->margin.p;
}

}  // namespace

// =================================================================== C ABI
extern "C" {

const char* B2_GetLastError(void) { return g_last_error.c_str(); }
int B2_SetOption(const char* key, const char* value) {
  API_BEGIN
  std::string k(key ? key : ""), v(value ? value : "");
  if (k == "hist_narrow") g_hist_narrow = atoi(v.c_str()) != 0 ? 1 : 0;   // layout of matrices quantised from now on
  else fail("unknown option '%s'", k.c_str());
  API_END
}
int B2_GetVersion(void) { return 100; }
int B2_DeviceCount(int* out) {
  API_BEGIN
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) { n = 0; cudaGetLastError(); }
  *out = n;
  API_END
}

int B2_GetUniqueId(uint8_t out[128]) {
  API_BEGIN
  ncclUniqueId id;
  NCCL_CHECK(nccl()->GetUniqueId(&id));
  memcpy(out, id.internal, 128);
  API_END
}
int B2_CommCreate(const uint8_t uid[128], int rank, int world, int device, B2Handle* out) {
  API_BEGIN
  if (world < 1 || rank < 0 || rank >= world) fail("invalid rank %d / world %d", rank, world);
  get_ctx(device);
  CommH* h = new CommH(); h->kind = kComm;
  h->c.rank = rank; h->c.world = world; h->c.device = device;
  if (world > 1) {
    ncclUniqueId id; memcpy(id.internal, uid, 128);
    int r = nccl()->CommInitRank(&h->c.comm, world, id, rank);
    if (r != 0) { delete h; fail("ncclCommInitRank failed: %s", nccl()->GetErrorString(r)); }
    // abort word of the peer-memory waits, written through its own stream while a kernel may be spinning
    if (cudaMalloc((void**)&h->c.d_abort, sizeof(uint32_t)) != cudaSuccess || cudaMemset(h->c.d_abort, 0, sizeof(uint32_t)) != cudaSuccess ||
        cudaStreamCreateWithFlags(&h->c.abort_stream, cudaStreamNonBlocking) != cudaSuccess) {
      cudaGetLastError(); h->c.d_abort = nullptr; h->c.abort_stream = nullptr;
    }
  }
  *out = (B2Handle)h;
  API_END
}
int B2_CommRank(B2Handle comm, int* rank, int* world) {
  API_BEGIN
  CommH* h = from_handle<CommH>(comm, kComm, "communicator");
  *rank = h->c.rank; *world = h->c.world;
  API_END
}
int B2_CommAllReduce(B2Handle comm, double* inout, int32_t n, int32_t op) {
  API_BEGIN
  if (n < 0 || op < 0 || op > 2) fail("invalid allreduce arguments (n=%d, op=%d)", n, op);
  if (!comm || n == 0) return 0;                      // single process: identity
  CommH* h = from_handle<CommH>(comm, kComm, "communicator");
  if (h->c.world <= 1) return 0;
  Ctx* ctx = get_ctx(h->c.device);
  CUDA_CHECK(cudaSetDevice(ctx->device));
  DevBuf<double> d; d.ensure((size_t)n);
  CUDA_CHECK(cudaMemcpyAsync(d.p, inout, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
  allreduce(&h->c, d.p, (size_t)n, kNcclFloat64, op == 0 ? kNcclSum : op == 1 ? kNcclMax : kNcclMin, ctx->stream);
  CUDA_CHECK(cudaMemcpyAsync(inout, d.p, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  API_END
}
int B2_CommAbort(B2Handle comm) {
  API_BEGIN
  CommH* h = from_handle<CommH>(comm, kComm, "communicator");
  if (h->c.comm && !h->c.aborted.exchange(true)) {
    if (h->c.d_abort && h->c.abort_stream) {   // release kernels that spin on a peer flag (p2p.cuh) before NCCL is torn down
      static const uint32_t one = 1;
      cudaSetDevice(h->c.device);
      cudaMemcpyAsync(h->c.d_abort, &one, sizeof(one), cudaMemcpyHostToDevice, h->c.abort_stream);
      cudaStreamSynchronize(h->c.abort_stream);
    }
    nccl()->CommAbort(h->c.comm);
  }
  API_END
}
int B2_CommFree(B2Handle comm) {
  API_BEGIN
  CommH* h = from_handle<CommH>(comm, kComm, "communicator");
  if (h->c.comm && !h->c.aborted.load()) nccl()->CommDestroy(h->c.comm);
  if (h->c.abort_stream) cudaStreamDestroy(h->c.abort_stream);
  if (h->c.d_abort) cudaFree(h->c.d_abort);
  delete h;
  API_END
}

int B2_MatrixCreateFromDense(const float* data, int64_t n_rows, int32_t n_cols, float missing, int device, B2Handle* out) {
  API_BEGIN
  if (n_rows < 0 || n_cols <= 0) fail("invalid matrix shape %lld x %d", (long long)n_rows, n_cols);
  if (n_rows >= (1LL << 31)) fail("at most 2^31-1 rows per GPU shard (row ids are int32), got %lld", (long long)n_rows);
  Ctx* ctx = get_ctx(device);
  Matrix* m = new Matrix(); m->kind = kMatrix; m->ctx = ctx; m->n = n_rows; m->F = n_cols; m->missing = missing;
  try {
    m->raw.ensure((size_t)std::max<int64_t>(n_rows * n_cols, 1));
    upload_pipelined(ctx, m->raw.p, data, (size_t)n_rows * n_cols * sizeof(float));
  } catch (...) { delete m; throw; }
  m->has_raw = true;
  { std::lock_guard<std::mutex> lk(g_matrix_mu); m->uid = g_next_matrix_uid++; g_live_matrices.insert(m->uid); }
  *out = (B2Handle)m;
  API_END
}
int B2_MatrixCreate(int64_t n_rows, int32_t n_cols, float missing, int device, B2Handle* out) {
  API_BEGIN
  if (n_rows < 0 || n_cols <= 0) fail("invalid matrix shape %lld x %d", (long long)n_rows, n_cols);
  if (n_rows >= (1LL << 31)) fail("at most 2^31-1 rows per GPU shard (row ids are int32), got %lld", (long long)n_rows);
  Ctx* ctx = get_ctx(device);
  Matrix* m = new Matrix(); m->kind = kMatrix; m->ctx = ctx; m->n = n_rows; m->F = n_cols; m->missing = missing;
  try { m->raw.ensure((size_t)std::max<int64_t>(n_rows * n_cols, 1)); } catch (...) { delete m; throw; }
  m->has_raw = true;
  { std::lock_guard<std::mutex> lk(g_matrix_mu); m->uid = g_next_matrix_uid++; g_live_matrices.insert(m->uid); }
  *out = (B2Handle)m;
  API_END
}
int B2_MatrixCreateFromProcess(int64_t pid, uint64_t remote_addr, int64_t remote_row_stride_bytes, int64_t n_rows, int32_t n_cols,
                               float missing, int device, B2Handle* out) {
  API_BEGIN
  if (n_rows < 0 || n_cols <= 0) fail("invalid matrix shape %lld x %d", (long long)n_rows, n_cols);
  if (n_rows >= (1LL << 31)) fail("at most 2^31-1 rows per GPU shard (row ids are int32), got %lld", (long long)n_rows);
  if (pid <= 0 || remote_row_stride_bytes < (int64_t)n_cols * 4) fail("invalid remote source (pid %lld, row stride %lld)", (long long)pid, (long long)remote_row_stride_bytes);
  Ctx* ctx = get_ctx(device);
  Matrix* m = new Matrix(); m->kind = kMatrix; m->ctx = ctx; m->n = n_rows; m->F = n_cols; m->missing = missing;
  try {
    m->raw.ensure((size_t)std::max<int64_t>(n_rows * n_cols, 1));
    UploadSource u; u.pid = pid; u.remote_addr = remote_addr; u.row_bytes = (size_t)n_cols * 4; u.row_stride = (size_t)remote_row_stride_bytes;
    upload_pipelined(ctx, m->raw.p, u, (size_t)n_rows * n_cols * sizeof(float));
  } catch (...) { delete m; throw; }
  m->has_raw = true;
  { std::lock_guard<std::mutex> lk(g_matrix_mu); m->uid = g_next_matrix_uid++; g_live_matrices.insert(m->uid); }
  *out = (B2Handle)m;
  API_END
}
// host mirror of b2::B2RowBlocks (p2p_exchange.cu)
struct RowBlocksHost {
  const float* base[B2_P2P_MAX_WORLD];
  long long start[B2_P2P_MAX_WORLD + 1];
  int world, rank, n_cols;
  long long n_mine;
};
// Staging block of the interleaved ingest: persistent per device (grow-only), exported ONCE; the peers keep their mapping
// of it across calls (mapping / unmapping a multi-GB allocation costs more than moving the rows).  A block that had to
// grow is retired and freed only after the call's closing barrier, when every peer has dropped its mapping of it.
struct IngestStage { float* p = nullptr; size_t bytes = 0; cudaIpcMemHandle_t h; bool exported = false; };
IngestStage g_ingest_stage[64];
std::map<std::string, void*> g_peer_stage;      // handle bytes -> mapped pointer (this process)
std::mutex g_ingest_mu;
double wall_seconds() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

int B2_MatrixCreateFromProcessInterleaved(int64_t pid, uint64_t remote_addr, int64_t n_total_rows, int32_t n_cols, int32_t shard_rank,
                                          B2Handle commh, float missing, int device, B2Handle* out) {
  API_BEGIN
  if (n_total_rows < 0 || n_cols <= 0 || pid <= 0) fail("invalid remote matrix (%lld x %d, pid %lld)", (long long)n_total_rows, n_cols, (long long)pid);
  Comm* c = commh ? &from_handle<CommH>(commh, kComm, "communicator")->c : nullptr;
  if (!c || c->world < 2 || c->world > B2_P2P_MAX_WORLD) fail("interleaved remote ingest needs a communicator of 2..%d ranks", B2_P2P_MAX_WORLD);
  const int W = c->world, rank = c->rank;
  Ctx* ctx = get_ctx(device); cudaStream_t s = ctx->stream;
  static const bool timing = getenv("B2_INGEST_TIMING") && atoi(getenv("B2_INGEST_TIMING")) != 0;
  double t0 = wall_seconds(), t_prev = t0;
  auto lap = [&](const char* what) {
    if (!timing) return;
    const double t = wall_seconds();
    fprintf(stderr, "[b2 ingest rank %d] %-28s %.4f s\n", rank, what, t - t_prev);
    t_prev = t;
  };
  std::lock_guard<std::mutex> ingest_lock(g_ingest_mu);
  // contiguous block of this rank (BATCH split of the global rows) and the rows it finally owns (INTERLEAVED)
  RowBlocksHost rb; memset(&rb, 0, sizeof(rb));
  const int64_t per = n_total_rows / W, extra = n_total_rows % W;
  for (int w = 0; w <= W; ++w) rb.start[w] = (long long)(w * per + std::min<int64_t>(w, extra));
  const int64_t b0 = rb.start[rank], bn = rb.start[rank + 1] - b0;
  const int64_t n_mine = rank < n_total_rows ? (n_total_rows - rank + W - 1) / W : 0;
  if (n_mine >= (1LL << 31)) fail("at most 2^31-1 rows per GPU shard (row ids are int32), got %lld", (long long)n_mine);
  rb.world = W; rb.rank = rank; rb.n_cols = n_cols; rb.n_mine = (long long)n_mine;
  DevBuf<int32_t> d_flag; d_flag.ensure(1);
  auto any_rank = [&](int32_t mine) {   // max over the ranks of a flag
    CUDA_CHECK(cudaMemcpyAsync(d_flag.p, &mine, sizeof(mine), cudaMemcpyHostToDevice, s));
    allreduce(c, d_flag.p, 1, kNcclInt32, kNcclMax, s);
    CUDA_CHECK(cudaMemcpyAsync(&mine, d_flag.p, sizeof(mine), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    return mine;
  };
  // collective call: every rank must hold the shard of its own rank, or all of them fail together
  if (any_rank(shard_rank == rank ? 0 : 1))
    fail("interleaved remote ingest: shard %d handed to rank %d (or a mismatch on another rank)", shard_rank, rank);
  lap("agreement");
  Matrix* m = new Matrix(); m->kind = kMatrix; m->ctx = ctx; m->n = n_mine; m->F = n_cols; m->missing = missing;
  void* retired = nullptr;
  try {
    IngestStage& st = g_ingest_stage[(device >= 0 && device < 64) ? device : 0];
    const size_t need = (size_t)std::max<int64_t>(bn * n_cols, 1) * sizeof(float);
    int ok = 1;
    if (st.bytes < need) {
      retired = st.p; st.p = nullptr; st.bytes = 0; st.exported = false;
      const size_t want = (need + need / 16 + ((size_t)1 << 20)) & ~(((size_t)1 << 20) - 1);
      void* q = nullptr;
      if (cudaMalloc(&q, want) != cudaSuccess) {
        cudaGetLastError();
        { std::lock_guard<std::mutex> lk(g_dev_pool[(device >= 0 && device < 64) ? device : 0].mu); pool_trim(g_dev_pool[(device >= 0 && device < 64) ? device : 0], 0); }
        if (cudaMalloc(&q, want) != cudaSuccess) { cudaGetLastError(); fail("cudaMalloc of the %zu-byte ingest staging block failed", want); }
      }
      st.p = (float*)q; st.bytes = want;
    }
    if (!st.exported) {
      if (cudaIpcGetMemHandle(&st.h, st.p) == cudaSuccess) st.exported = true;
      else { ok = 0; cudaGetLastError(); memset(&st.h, 0, sizeof(st.h)); }
    }
    lap("staging block");
    UploadSource u; u.pid = pid; u.remote_addr = remote_addr + (uint64_t)b0 * (uint64_t)n_cols * 4u; u.row_bytes = (size_t)n_cols * 4; u.row_stride = u.row_bytes;
    upload_pipelined(ctx, st.p, u, (size_t)bn * n_cols * sizeof(float));
    lap("read block from the driver");
    m->raw.ensure((size_t)std::max<int64_t>(n_mine * n_cols, 1));
    // exchange the IPC handles of the staging blocks (also: every rank's block is uploaded)
    DevBuf<uint8_t> d_mine, d_all; d_mine.ensure(sizeof(st.h)); d_all.ensure(sizeof(st.h) * (size_t)W);
    CUDA_CHECK(cudaMemcpyAsync(d_mine.p, &st.h, sizeof(st.h), cudaMemcpyHostToDevice, s));
    NCCL_CHECK(nccl()->AllGather(d_mine.p, d_all.p, sizeof(st.h), kNcclUint8, c->comm, s));
    std::vector<cudaIpcMemHandle_t> all((size_t)W);
    CUDA_CHECK(cudaMemcpyAsync(all.data(), d_all.p, sizeof(st.h) * (size_t)W, cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    lap("handle exchange");
    // drop mappings of blocks that no peer exports any more (a peer's block grew), then map what is new
    std::set<std::string> current;
    for (int w = 0; w < W; ++w) if (w != rank) current.insert(std::string((const char*)&all[w], sizeof(all[w])));
    for (auto it = g_peer_stage.begin(); it != g_peer_stage.end();) {
      if (!current.count(it->first)) { cudaIpcCloseMemHandle(it->second); it = g_peer_stage.erase(it); } else ++it;
    }
    for (int w = 0; w < W && ok; ++w) {
      if (w == rank) { rb.base[w] = st.p; continue; }
      const std::string key((const char*)&all[w], sizeof(all[w]));
      auto it = g_peer_stage.find(key);
      if (it == g_peer_stage.end()) {
        void* q = nullptr;
        if (cudaIpcOpenMemHandle(&q, all[w], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { ok = 0; cudaGetLastError(); break; }
        it = g_peer_stage.emplace(key, q).first;
      }
      rb.base[w] = (const float*)it->second;
    }
    lap("peer mappings");
    if (any_rank(ok ? 0 : 1)) {
      // no peer mapping on some rank (no NVLink / IPC): every rank reads its own strided shard from the driver instead
      UploadSource us; us.pid = pid; us.remote_addr = remote_addr + (uint64_t)rank * (uint64_t)n_cols * 4u;
      us.row_bytes = (size_t)n_cols * 4; us.row_stride = us.row_bytes * (size_t)W;
      upload_pipelined(ctx, m->raw.p, us, (size_t)n_mine * n_cols * sizeof(float));
    } else {
      LAUNCH_CHECK(b2_launch_gather_interleaved_rows(&rb, m->raw.p, ctx->num_sms, s));
    }
    // nobody overwrites (next call) or frees (a retired block) its staging block while a peer may still pull rows out of it
    any_rank(0);
    lap("row gather + closing barrier");
    if (retired) { cudaFree(retired); retired = nullptr; }
  } catch (...) { if (retired) cudaFree(retired); delete m; throw; }
  m->has_raw = true;
  { std::lock_guard<std::mutex> lk(g_matrix_mu); m->uid = g_next_matrix_uid++; g_live_matrices.insert(m->uid); }
  *out = (B2Handle)m;
  if (timing) fprintf(stderr, "[b2 ingest rank %d] total %.4f s (%lld of %lld rows x %d)\n", rank, wall_seconds() - t0, (long long)n_mine, (long long)n_total_rows, n_cols);
  API_END
}
int B2_MatrixSetRows(B2Handle mh, int64_t row_begin, const float* data, int64_t n_rows) {
  API_BEGIN
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  CUDA_CHECK(cudaSetDevice(m->ctx->device));
  if (m->quantized || !m->has_raw) fail("rows can only be set before the matrix is quantised");
  if (row_begin < 0 || n_rows < 0 || row_begin + n_rows > m->n) fail("row block [%lld, %lld) outside the matrix (%lld rows)",
                                                                     (long long)row_begin, (long long)(row_begin + n_rows), (long long)m->n);
  upload_pipelined(m->ctx, m->raw.p + (size_t)row_begin * m->F, data, (size_t)n_rows * m->F * sizeof(float));
  API_END
}
int B2_MatrixSetFloatInfo(B2Handle mh, const char* field, const float* values, int64_t len) {
  API_BEGIN
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  CUDA_CHECK(cudaSetDevice(m->ctx->device));
  std::string f(field ? field : "");
  DevBuf<float>* dst = nullptr; int64_t* cnt = nullptr;
  if (f == "label") { dst = &m->label; cnt = &m->n_label; m->rank_version++; if (len != m->n) fail("label length %lld != rows %lld", (long long)len, (long long)m->n); }
  else if (f == "weight") { dst = &m->weight; cnt = &m->n_weight; if (len != m->n && len != 0) fail("weight length %lld != rows %lld", (long long)len, (long long)m->n); }
  else if (f == "label_lower_bound" || f == "label_upper_bound") {
    const bool lo = f == "label_lower_bound";
    dst = lo ? &m->lower : &m->upper; cnt = lo ? &m->n_lower : &m->n_upper;
    if (len != m->n && len != 0) fail("%s length %lld != rows %lld", f.c_str(), (long long)len, (long long)m->n);
  }
  else if (f == "base_margin") { dst = &m->base_margin; cnt = &m->n_base_margin; m->margin_version++; if (len != 0 && (m->n == 0 || len % m->n != 0)) fail("base_margin length %lld is not a multiple of rows %lld", (long long)len, (long long)m->n); }
  else if (f == "feature_weights") {
    // DMatrix.set_info(feature_weights=...) (main.py:439-442): weights of the column sampler, Q16 fixed point
    if (len != 0 && len != m->F) fail("feature_weights length %lld != features %d", (long long)len, m->F);
    m->fwq.clear();
    for (int64_t i = 0; i < len; ++i) {
      if (!(values[i] >= 0.0f) || std::isinf(values[i])) fail("feature_weights must be finite and non-negative");
      const double q = (double)values[i] * 65536.0;
      m->fwq.push_back(q >= 4294967295.0 ? 0xffffffffu : (uint32_t)llrint(q));
    }
    m->d_fwq.ensure((size_t)std::max<int64_t>(len, 1));
    if (len > 0) CUDA_CHECK(cudaMemcpyAsync(m->d_fwq.p, m->fwq.data(), len * sizeof(uint32_t), cudaMemcpyHostToDevice, m->ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(m->ctx->stream));
    return 0;
  }
  else fail("unknown float info field '%s'", f.c_str());
  dst->ensure((size_t)std::max<int64_t>(len, 1));
  if (len > 0) CUDA_CHECK(cudaMemcpyAsync(dst->p, values, len * sizeof(float), cudaMemcpyHostToDevice, m->ctx->stream));
  CUDA_CHECK(cudaStreamSynchronize(m->ctx->stream));
  *cnt = len;
  API_END
}
int B2_MatrixSetGroups(B2Handle mh, const int32_t* group_sizes, int64_t n_groups) {
  API_BEGIN
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  CUDA_CHECK(cudaSetDevice(m->ctx->device));
  if (n_groups < 0) fail("query groups: negative group count %lld", (long long)n_groups);
  std::vector<int64_t> ptr((size_t)n_groups + 1, 0);
  int64_t mx = 0;
  for (int64_t g = 0; g < n_groups; ++g) {
    if (group_sizes[g] < 1) fail("query group %lld has %d rows: every group needs at least one", (long long)g, group_sizes[g]);
    ptr[g + 1] = ptr[g] + group_sizes[g];
    mx = std::max<int64_t>(mx, group_sizes[g]);
  }
  if (n_groups > 0 && ptr[n_groups] != m->n)
    fail("query groups cover %lld rows, the matrix has %lld", (long long)ptr[n_groups], (long long)m->n);
  m->qgroup_ptr.ensure(ptr.size());
  CUDA_CHECK(cudaMemcpyAsync(m->qgroup_ptr.p, ptr.data(), ptr.size() * sizeof(int64_t), cudaMemcpyHostToDevice, m->ctx->stream));
  CUDA_CHECK(cudaStreamSynchronize(m->ctx->stream));
  m->h_qgroup_ptr = std::move(ptr);
  m->n_qgroups = n_groups; m->max_qgroup = mx;
  m->rank_version++;
  API_END
}
int B2_MatrixSetFeatureTypes(B2Handle mh, const uint8_t* is_cat, int32_t len) {
  API_BEGIN
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  if (m->quantized) fail("feature types must be set before the matrix is quantised");
  if (len != m->F) fail("feature types: %d entries for %d features", len, m->F);
  m->is_cat.assign(is_cat, is_cat + len);
  m->cat_feats.clear();
  for (int f = 0; f < m->F; ++f) { m->is_cat[f] = m->is_cat[f] ? 1 : 0; if (m->is_cat[f]) m->cat_feats.push_back(f); }
  API_END
}
int B2_MatrixGetFeatureTypes(B2Handle mh, uint8_t* is_cat) {
  API_BEGIN
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  for (int f = 0; f < m->F; ++f) is_cat[f] = m->is_cat.empty() ? 0 : m->is_cat[f];
  API_END
}
int B2_MatrixNumRow(B2Handle mh, int64_t* out) { API_BEGIN *out = from_handle<Matrix>(mh, kMatrix, "matrix")->n; API_END }
int B2_MatrixNumCol(B2Handle mh, int32_t* out) { API_BEGIN *out = from_handle<Matrix>(mh, kMatrix, "matrix")->F; API_END }

int B2_MatrixQuantize(B2Handle mh, B2Handle commh, int32_t max_bin, B2Handle refh, int32_t keep_raw) {
  API_BEGIN
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  CUDA_CHECK(cudaSetDevice(m->ctx->device));
  Comm* comm = commh ? &from_handle<CommH>(commh, kComm, "communicator")->c : nullptr;
  if (!m->has_raw) fail("matrix has no raw data on the device (already quantised without keep_raw?)");
  if (refh) {
    Matrix* r = from_handle<Matrix>(refh, kMatrix, "matrix");
    if (!r->quantized) fail("reference matrix is not quantised");
    if (r->F != m->F) fail("reference matrix has %d features, this one %d", r->F, m->F);
    m->cut_ptrs = r->cut_ptrs; m->cut_vals = r->cut_vals; m->min_vals = r->min_vals; m->has_missing = r->has_missing; m->max_bin = r->max_bin;
    m->is_cat = r->is_cat; m->cat_feats = r->cat_feats;
  } else {
    make_cuts(m, comm, max_bin);
  }
  bin_matrix(m);
  if (!keep_raw) { m->raw.release(); m->has_raw = false; }
  API_END
}
int B2_MatrixQuantizeWithCuts(B2Handle mh, const int32_t* ptrs, const float* vals, const float* mins, const uint8_t* has_missing,
                              int32_t max_bin, int32_t keep_raw) {
  API_BEGIN
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  CUDA_CHECK(cudaSetDevice(m->ctx->device));
  if (!m->has_raw) fail("matrix has no raw data on the device (already quantised without keep_raw?)");
  if (max_bin < 2 || max_bin > 256) fail("max_bin must be in [2, 256] (uint8 bin matrix), got %d", max_bin);
  if (ptrs[0] != 0) fail("cut pointers must start at 0");
  for (int f = 0; f < m->F; ++f) {
    const int nc = ptrs[f + 1] - ptrs[f];
    if (nc < 1 || nc > 256) fail("feature %d has %d cuts; expected 1..256", f, nc);
  }
  m->cut_ptrs.assign(ptrs, ptrs + m->F + 1);
  m->cut_vals.assign(vals, vals + ptrs[m->F]);
  m->min_vals.assign(mins, mins + m->F);
  m->has_missing.assign(has_missing, has_missing + m->F);
  m->max_bin = max_bin;
  bin_matrix(m);
  if (!keep_raw) { m->raw.release(); m->has_raw = false; }
  API_END
}
int B2_MatrixEnsureRaw(B2Handle mh, const float* data) {
  API_BEGIN
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  CUDA_CHECK(cudaSetDevice(m->ctx->device));
  if (m->has_raw) return 0;
  m->raw.ensure((size_t)std::max<int64_t>(m->n * m->F, 1));
  upload_pipelined(m->ctx, m->raw.p, data, (size_t)m->n * m->F * sizeof(float));
  m->has_raw = true;
  API_END
}
int B2_MatrixCutsSize(B2Handle mh, int32_t* total) {
  API_BEGIN
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  if (!m->quantized) fail("matrix is not quantised");
  *total = m->cut_ptrs[m->F];
  API_END
}
int B2_MatrixGetCuts(B2Handle mh, int32_t* ptrs, float* vals, float* mins, uint8_t* has_missing) {
  API_BEGIN
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  if (!m->quantized) fail("matrix is not quantised");
  memcpy(ptrs, m->cut_ptrs.data(), (m->F + 1) * sizeof(int32_t));
  memcpy(vals, m->cut_vals.data(), m->cut_vals.size() * sizeof(float));
  memcpy(mins, m->min_vals.data(), m->F * sizeof(float));
  memcpy(has_missing, m->has_missing.data(), m->F);
  API_END
}
int B2_MatrixGetBins(B2Handle mh, uint8_t* out) {
  API_BEGIN
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  CUDA_CHECK(cudaSetDevice(m->ctx->device));
  if (!m->quantized) fail("matrix is not quantised");
  std::vector<uint8_t> h((size_t)m->n * m->row_stride);
  if (m->n > 0) CUDA_CHECK(cudaMemcpy(h.data(), m->bins.p, h.size(), cudaMemcpyDeviceToHost));
  for (int64_t i = 0; i < m->n; ++i)
    for (int f = 0; f < m->F; ++f) out[i * m->F + f] = h[(size_t)i * m->row_stride + m->feat_byte[f]];
  API_END
}
int B2_MatrixFree(B2Handle mh) {
  API_BEGIN
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  cudaSetDevice(m->ctx->device);
  { std::lock_guard<std::mutex> lk(g_matrix_mu); g_live_matrices.erase(m->uid); }
  delete m;
  API_END
}

int B2_BoosterCreate(const char* params, B2Handle trainh, B2Handle commh, B2Handle* out) {
  API_BEGIN
  Matrix* m = trainh ? from_handle<Matrix>(trainh, kMatrix, "matrix") : nullptr;
  if (m && !m->quantized) fail("train matrix must be quantised (B2_MatrixQuantize) before B2_BoosterCreate");
  Booster* b = new Booster(); b->kind = kBooster; b->train = m;
  b->comm = commh ? &from_handle<CommH>(commh, kComm, "communicator")->c : nullptr;
  try {
    parse_params(params, &b->p, nullptr);
    if (m) { b->ctx = m->ctx; b->n_features = m->F; CUDA_CHECK(cudaSetDevice(m->ctx->device)); }
    else {  // prediction-only booster (model loaded with B2_BoosterAddTree)
      if (b->p.num_feature <= 0) fail("a booster without a train matrix needs num_feature=<n> in params");
      b->ctx = get_ctx(b->p.device); b->n_features = b->p.num_feature;
    }
  } catch (...) { delete b; throw; }
  *out = (B2Handle)b;
  API_END
}
int B2_BoosterUpdateOneIter(B2Handle bh, int32_t iter) {
  API_BEGIN
  (void)iter;
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  boost_round(b, nullptr, nullptr, 0);
  API_END
}
int B2_BoosterBoostOneIter(B2Handle bh, const float* grad, const float* hess, int64_t len) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  if (!grad || !hess) fail("grad/hess must not be NULL");
  boost_round(b, grad, hess, len);
  API_END
}
int B2_BoosterGetGradients(B2Handle bh, float* grad, float* hess, int64_t len) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  if (!b->train) fail("this booster has no train matrix (prediction-only)");
  const int64_t nk = b->train->n * b->p.num_class;
  if (len != nk) fail("gradient buffers have %lld values, expected %lld", (long long)len, (long long)nk);
  if (!b->gh_ready) fail("no gradients yet: run a boosting round first");
  CUDA_CHECK(cudaSetDevice(b->ctx->device));
  std::vector<float2> h((size_t)std::max<int64_t>(nk, 1));
  if (nk > 0) CUDA_CHECK(cudaMemcpyAsync(h.data(), b->gh.p, (size_t)nk * sizeof(float2), cudaMemcpyDeviceToHost, b->ctx->stream));
  CUDA_CHECK(cudaStreamSynchronize(b->ctx->stream));
  for (int64_t i = 0; i < nk; ++i) { grad[i] = h[i].x; hess[i] = h[i].y; }
  API_END
}
int B2_BoosterEvalSet(B2Handle bh, B2Handle mh, const char* metric, double* out) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  CUDA_CHECK(cudaSetDevice(b->ctx->device));
  cudaStream_t s = b->ctx->stream;
  float mparam = 0.0f;
  int minus = 0;
  const int mid = metric_id(metric, b->p, &mparam, &minus);
  const bool aft_metric = mid == 14 || mid == 15;
  if (mid >= 16 && mid <= 18) {
    // ndcg / map / pre: per query group on the prediction order (rank_kernel.cu), averaged over the groups of all workers
    if (b->p.num_class > 1) fail("metric '%s' needs a single-output objective", metric);
    if (!m->has_qgroups()) fail("metric '%s' needs query groups (qid) on the evaluation matrix", metric);
    if (m->n_label != m->n) fail("evaluation matrix has no labels");
    float* margin = eval_margin(b, m);
    DevBuf<float> pred; DevBuf<double> vals; RankOrder po, lo;
    pred.ensure((size_t)std::max<int64_t>(m->n, 1));
    if (m->n > 0) CUDA_CHECK(cudaMemcpyAsync(pred.p, margin, (size_t)m->n * sizeof(float), cudaMemcpyDeviceToDevice, s));
    LAUNCH_CHECK(b2_launch_transform(b->p.objective, 1, pred.p, m->n, b->ctx->num_sms, s));
    po.run(m, pred.p, b->ctx->num_sms, s);
    if (mid == 16) lo.run(m, m->label.p, b->ctx->num_sms, s);
    ensure_rank_disc(b, m->max_qgroup);
    vals.ensure((size_t)std::max<int64_t>(m->n_qgroups, 1));
    b->d_metric.ensure(2);
    LAUNCH_CHECK(b2_launch_rank_metric(mid, (int)mparam, minus, b->p.ndcg_exp_gain ? 1 : 0, m->qgroup_ptr.p, m->n_qgroups,
                                       po.rows.p, m->label.p, mid == 16 ? lo.keys_sorted.p : nullptr, b->rank_disc.p, vals.p,
                                       b->d_metric.p, b->ctx->num_sms, s));
    allreduce(b->comm, b->d_metric.p, 2, kNcclFloat64, kNcclSum, s);
    double h[2];
    CUDA_CHECK(cudaMemcpyAsync(h, b->d_metric.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    *out = h[1] > 0 ? h[0] / h[1] : 0.0;
    return 0;
  }
  // xgboost computes a per-group ranking AUC on a matrix with groups; this engine's auc is the binary one only
  if (mid == 6 && m->has_qgroups())
    fail("metric 'auc' on a matrix with query groups (per-group ranking AUC) is not supported; use ndcg or map");
  if (aft_metric && b->p.objective != kObjAft)
    fail("metric '%s' does not fit objective '%s'", metric, b->p.objective_name.c_str());
  if (aft_metric && !m->has_bounds()) fail("metric '%s' needs label_lower_bound and label_upper_bound on the evaluation matrix", metric);
  if (!aft_metric && m->n_label != m->n) fail("evaluation matrix has no labels");
  float* margin = eval_margin(b, m);
  b->d_metric.ensure(3);
  CUDA_CHECK(cudaMemsetAsync(b->d_metric.p, 0, 3 * sizeof(double), s));
  if ((mid == 3 || mid == 4) != (b->p.objective == kObjSoftprob))
    fail("metric '%s' does not fit objective '%s'", metric, b->p.objective_name.c_str());
  if (aft_metric) {
    LAUNCH_CHECK(b2_launch_aft_metric(b->p.aft_dist, mid, (double)b->p.aft_sigma, margin, m->lower.p, m->upper.p,
                                      m->n_weight ? m->weight.p : nullptr, m->n, b->d_metric.p, b->ctx->num_sms, s));
    allreduce(b->comm, b->d_metric.p, 2, kNcclFloat64, kNcclSum, s);
    double h[2];
    CUDA_CHECK(cudaMemcpyAsync(h, b->d_metric.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    *out = h[1] > 0 ? h[0] / h[1] : 0.0;
    return 0;
  }
  if (mid == 6) {
    // binary ROC AUC on the transformed prediction (auc_kernel.cu): local (area, fp*tp) pairs summed over the workers
    if (b->p.objective == kObjSoftprob) fail("metric 'auc' is implemented for binary labels (binary:logistic / regression scores) only");
    DevBuf<float> pred; DevBuf<uint8_t> tmp;
    const size_t rows = (size_t)std::max<int64_t>(m->n, 1);
    pred.ensure(rows);
    if (m->n > 0) CUDA_CHECK(cudaMemcpyAsync(pred.p, margin, (size_t)m->n * sizeof(float), cudaMemcpyDeviceToDevice, s));
    LAUNCH_CHECK(b2_launch_transform(b->p.objective, 1, pred.p, m->n, b->ctx->num_sms, s));
    const size_t tb = b2_auc_temp_bytes(m->n);
    tmp.ensure(tb);
    LAUNCH_CHECK(b2_auc_binary(pred.p, m->label.p, m->n_weight ? m->weight.p : nullptr, m->n, tmp.p, tb, b->d_metric.p, b->ctx->num_sms, s));
    allreduce(b->comm, b->d_metric.p, 2, kNcclFloat64, kNcclSum, s);
    double h[2];
    CUDA_CHECK(cudaMemcpyAsync(h, b->d_metric.p, sizeof(h), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    *out = h[1] > 0 ? h[0] / h[1] : 0.5;   // only one class present: xgboost reports 0.5
    return 0;
  }
  LAUNCH_CHECK(b2_launch_metric(b->p.objective, mid, b->p.num_class, mparam, margin, m->label.p, m->n_weight ? m->weight.p : nullptr, m->n, b->d_metric.p,
                                b->ctx->num_sms, s));
  // (sum, wsum, rows with a label outside [0, num_class)): the count travels with the sums, so every rank fails together
  allreduce(b->comm, b->d_metric.p, 3, kNcclFloat64, kNcclSum, s);
  double h[3];
  CUDA_CHECK(cudaMemcpyAsync(h, b->d_metric.p, sizeof(h), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  if (h[2] > 0)
    fail("metric '%s': label must be in [0, num_class), num_class = %d (%.0f rows outside)", metric, b->p.num_class, h[2]);
  double v = h[1] > 0 ? h[0] / h[1] : 0.0;
  *out = (mid == 0 || mid == 7) ? sqrt(v) : v;
  API_END
}
int B2_BoosterPredict(B2Handle bh, B2Handle mh, int32_t output_margin, int32_t tree_begin, int32_t tree_end, float* out,
                      int64_t out_len) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  CUDA_CHECK(cudaSetDevice(b->ctx->device));
  cudaStream_t s = b->ctx->stream; const int K = b->p.num_class;
  if (out_len != m->n * K) fail("output buffer has %lld values, expected %lld", (long long)out_len, (long long)(m->n * K));
  if (!m->has_raw) fail("prediction matrix has no raw data on the device (B2_MatrixEnsureRaw)");
  if (m->F != b->n_features) fail("feature count mismatch: matrix has %d, model has %d", m->F, b->n_features);
  const int nt = (int)b->trees.size();
  if (tree_end <= 0 || tree_end > nt) tree_end = nt;
  if (tree_begin < 0 || tree_begin > tree_end) fail("invalid tree range [%d, %d)", tree_begin, tree_end);
  DevBuf<float> tmp; tmp.ensure((size_t)std::max<int64_t>(out_len, 1));
  init_margin(b, tmp.p, m);
  sync_device_trees(b);
  LAUNCH_CHECK(b2_launch_predict(m->raw.p, m->n, m->F, m->missing, b->d_nodes.p, b->d_tree_offset.p, b->d_cat_table.p, tree_begin, tree_end, K, b->p.num_parallel_tree, tmp.p,
                                 b->ctx->num_sms, s));
  if (!output_margin) LAUNCH_CHECK(b2_launch_transform(b->p.objective, K, tmp.p, m->n, b->ctx->num_sms, s));
  if (out_len > 0) CUDA_CHECK(cudaMemcpyAsync(out, tmp.p, out_len * sizeof(float), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  API_END
}
// Common checks of the SHAP / leaf entries (the same as B2_BoosterPredict); resolves tree_end == 0 to all trees
static void check_predict_args(Booster* b, Matrix* m, int32_t tree_begin, int32_t* tree_end) {
  if (!m->has_raw) fail("prediction matrix has no raw data on the device (B2_MatrixEnsureRaw)");
  if (m->F != b->n_features) fail("feature count mismatch: matrix has %d, model has %d", m->F, b->n_features);
  const int nt = (int)b->trees.size();
  if (*tree_end <= 0 || *tree_end > nt) *tree_end = nt;
  if (tree_begin < 0 || tree_begin > *tree_end) fail("invalid tree range [%d, %d)", tree_begin, *tree_end);
  if (m->n_base_margin > 0 && m->n_base_margin != m->n * b->p.num_class)
    fail("base_margin has %lld values, expected %lld", (long long)m->n_base_margin, (long long)(m->n * b->p.num_class));
}

// rows per output block so that the device scratch of one block stays within 1 GiB whatever the row count
static int64_t rows_per_block(int64_t n, size_t bytes_per_row) {
  const size_t budget = (size_t)1 << 30;
  int64_t r = (int64_t)std::max<size_t>(1, budget / std::max<size_t>(bytes_per_row, 1));
  return std::max<int64_t>(1, std::min<int64_t>(r, n));
}

int B2_BoosterPredictContribs(B2Handle bh, B2Handle mh, int32_t tree_begin, int32_t tree_end, int32_t interactions, float* out,
                              int64_t out_len) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  CUDA_CHECK(cudaSetDevice(b->ctx->device));
  cudaStream_t s = b->ctx->stream; const int K = b->p.num_class; const int F = m->F;
  const size_t per_row = (size_t)K * (F + 1) * (interactions ? (size_t)(F + 1) : 1);
  if (out_len != m->n * (int64_t)per_row) fail("output buffer has %lld values, expected %lld", (long long)out_len, (long long)(m->n * (int64_t)per_row));
  check_predict_args(b, m, tree_begin, &tree_end);
  build_paths(b);
  std::vector<double> bias(K, 0.0);   // sum of the expected values of the trees in range, in tree order
  for (int t = tree_begin; t < tree_end; ++t) bias[(t / std::max(1, b->p.num_parallel_tree)) % K] += b->tree_expected[t];
  DevBuf<double> d_bias; upload(d_bias, bias, s);
  const int p_begin = b->tree_path_offset[tree_begin], p_end = b->tree_path_offset[tree_end];
  const float* bm = m->n_base_margin > 0 ? m->base_margin.p : nullptr;
  const float base_value = base_margin_value(b->p);
  // contributions: the row accumulators live in shared memory (up to 8 warps of K (F+1) doubles in <= 200 KiB),
  // otherwise in global scratch; interactions always accumulate in global scratch
  int warps = 8; size_t smem = 0;
  if (!interactions) {
    while (warps > 1 && b2_shap_contribs_smem(K, F, warps) > (size_t)200 * 1024) warps /= 2;
    smem = b2_shap_contribs_smem(K, F, warps);
    if (smem > (size_t)200 * 1024) { smem = 0; warps = 8; }
  }
  const bool gscratch = interactions || smem == 0;
  const int64_t blk = rows_per_block(m->n, per_row * (sizeof(float) + (gscratch ? sizeof(double) : 0)));
  DevBuf<float> d_out; DevBuf<double> d_acc;
  d_out.ensure((size_t)std::max<int64_t>(blk, 1) * per_row);
  if (gscratch) d_acc.ensure((size_t)std::max<int64_t>(blk, 1) * per_row);
  std::vector<cudaEvent_t> ev;
  for (int64_t r0 = 0; r0 < m->n; r0 += blk) {
    const int64_t rows = std::min<int64_t>(blk, m->n - r0);
    cudaEvent_t e0, e1; CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
    ev.push_back(e0); ev.push_back(e1);
    CUDA_CHECK(cudaEventRecord(e0, s));
    if (interactions)
      LAUNCH_CHECK(b2_launch_shap_interactions(m->raw.p, r0, rows, F, m->missing, b->d_path_elems.p, b->d_paths.p, p_begin, p_end,
                                               b->d_path_cats.p, K, d_bias.p, bm, base_value, d_acc.p, d_out.p, b->ctx->num_sms, s));
    else
      LAUNCH_CHECK(b2_launch_shap_contribs(m->raw.p, r0, rows, F, m->missing, b->d_path_elems.p, b->d_paths.p, p_begin, p_end,
                                           b->d_path_cats.p, K, d_bias.p, bm, base_value, gscratch ? d_acc.p : nullptr, warps, smem,
                                           d_out.p, b->ctx->num_sms, s));
    CUDA_CHECK(cudaEventRecord(e1, s));
    CUDA_CHECK(cudaMemcpyAsync(out + (size_t)r0 * per_row, d_out.p, (size_t)rows * per_row * sizeof(float), cudaMemcpyDeviceToHost, s));
  }
  CUDA_CHECK(cudaStreamSynchronize(s));
  for (size_t i = 0; i < ev.size(); i += 2) {
    float ms = 0; cudaEventElapsedTime(&ms, ev[i], ev[i + 1]);
    b->t.shap_ms += ms;
    cudaEventDestroy(ev[i]); cudaEventDestroy(ev[i + 1]);
  }
  b->t.shap_rows += m->n;
  API_END
}

int B2_BoosterPredictLeaf(B2Handle bh, B2Handle mh, int32_t tree_begin, int32_t tree_end, float* out, int64_t out_len) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  CUDA_CHECK(cudaSetDevice(b->ctx->device));
  cudaStream_t s = b->ctx->stream;
  check_predict_args(b, m, tree_begin, &tree_end);
  const int T = tree_end - tree_begin;
  if (out_len != m->n * T) fail("output buffer has %lld values, expected %lld", (long long)out_len, (long long)(m->n * T));
  if (T == 0 || m->n == 0) return 0;
  sync_device_trees(b);
  const int64_t blk = rows_per_block(m->n, (size_t)T * sizeof(float));
  DevBuf<float> d_out; d_out.ensure((size_t)blk * T);
  for (int64_t r0 = 0; r0 < m->n; r0 += blk) {
    const int64_t rows = std::min<int64_t>(blk, m->n - r0);
    LAUNCH_CHECK(b2_launch_leaf_index(m->raw.p, r0, rows, m->F, m->missing, b->d_nodes.p, b->d_tree_offset.p, b->d_cat_table.p,
                                      tree_begin, tree_end, d_out.p, b->ctx->num_sms, s));
    CUDA_CHECK(cudaMemcpyAsync(out + (size_t)r0 * T, d_out.p, (size_t)rows * T * sizeof(float), cudaMemcpyDeviceToHost, s));
  }
  CUDA_CHECK(cudaStreamSynchronize(s));
  API_END
}

int B2_BoosterGetTrainMargin(B2Handle bh, float* out, int64_t out_len) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  CUDA_CHECK(cudaSetDevice(b->ctx->device));
  if (!b->train) fail("this booster has no train matrix (prediction-only)");
  const int64_t want = b->train->n * b->p.num_class;
  if (out_len != want) fail("output buffer has %lld values, expected %lld", (long long)out_len, (long long)want);
  ensure_train_margin(b);
  if (want > 0) CUDA_CHECK(cudaMemcpyAsync(out, b->margin.p, want * sizeof(float), cudaMemcpyDeviceToHost, b->ctx->stream));
  CUDA_CHECK(cudaStreamSynchronize(b->ctx->stream));
  API_END
}
int B2_BoosterResetTrainMargin(B2Handle bh) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  CUDA_CHECK(cudaSetDevice(b->ctx->device));
  if (!b->train) fail("this booster has no train matrix (prediction-only)");
  b->margin_ready = false;
  ensure_train_margin(b);
  CUDA_CHECK(cudaStreamSynchronize(b->ctx->stream));
  API_END
}
int B2_BoosterGetBaseScore(B2Handle bh, float* out, int32_t* is_final) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  *out = b->p.base_score; *is_final = b->p.base_score_set ? 1 : 0;
  API_END
}
int B2_BoosterNumTrees(B2Handle bh, int32_t* out) { API_BEGIN *out = (int32_t)from_handle<Booster>(bh, kBooster, "booster")->trees.size(); API_END }
int B2_BoosterTreeNumNodes(B2Handle bh, int32_t tree, int32_t* out) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  if (tree < 0 || tree >= (int)b->trees.size()) fail("tree index %d out of range", tree);
  *out = b->trees[tree].size();
  API_END
}
int B2_BoosterGetTree(B2Handle bh, int32_t tree, int32_t* left, int32_t* right, int32_t* parent, int32_t* split_feature,
                      int32_t* split_bin, float* split_cond, uint8_t* default_left, float* value, float* base_weight,
                      float* loss_chg, double* sum_hess) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  if (tree < 0 || tree >= (int)b->trees.size()) fail("tree index %d out of range", tree);
  const TreeHost& t = b->trees[tree]; const size_t n = t.size();
  memcpy(left, t.left.data(), n * 4); memcpy(right, t.right.data(), n * 4); memcpy(parent, t.parent.data(), n * 4);
  memcpy(split_feature, t.feature.data(), n * 4); memcpy(split_bin, t.split_bin.data(), n * 4);
  memcpy(split_cond, t.cond.data(), n * 4); memcpy(default_left, t.default_left.data(), n);
  memcpy(value, t.value.data(), n * 4); memcpy(base_weight, t.base_weight.data(), n * 4);
  memcpy(loss_chg, t.loss_chg.data(), n * 4); memcpy(sum_hess, t.sum_hess.data(), n * 8);
  API_END
}
int B2_BoosterAddTree(B2Handle bh, int32_t n_nodes, const int32_t* left, const int32_t* right, const int32_t* parent,
                      const int32_t* split_feature, const int32_t* split_bin, const float* split_cond,
                      const uint8_t* default_left, const float* value, const float* base_weight, const float* loss_chg,
                      const double* sum_hess) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  if (n_nodes < 1) fail("a tree needs at least one node");
  TreeHost t;
  for (int i = 0; i < n_nodes; ++i) {
    t.add(parent[i]);
    if (left[i] >= n_nodes || right[i] >= n_nodes) fail("child index out of range in tree");
    if (split_feature[i] >= b->n_features) fail("split feature %d out of range", split_feature[i]);
    t.left[i] = left[i]; t.right[i] = right[i]; t.feature[i] = split_feature[i]; t.split_bin[i] = split_bin ? split_bin[i] : -1;
    t.cond[i] = split_cond[i]; t.default_left[i] = default_left[i]; t.value[i] = value[i];
    t.base_weight[i] = base_weight ? base_weight[i] : 0.f; t.loss_chg[i] = loss_chg ? loss_chg[i] : 0.f;
    t.sum_hess[i] = sum_hess ? sum_hess[i] : 0.0;
  }
  b->trees.push_back(std::move(t));
  b->margin_ready = false;
  API_END
}
int B2_BoosterGetTreeCategories(B2Handle bh, int32_t tree, uint8_t* split_type, uint32_t* cat_bits) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  if (tree < 0 || tree >= (int)b->trees.size()) fail("tree index %d out of range", tree);
  const TreeHost& t = b->trees[tree]; const size_t n = t.size();
  memcpy(split_type, t.split_type.data(), n); memcpy(cat_bits, t.cat_bits.data(), n * 8 * sizeof(uint32_t));
  API_END
}
int B2_BoosterSetTreeCategories(B2Handle bh, int32_t tree, const uint8_t* split_type, const uint32_t* cat_bits) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  if (tree < 0 || tree >= (int)b->trees.size()) fail("tree index %d out of range", tree);
  TreeHost& t = b->trees[tree]; const size_t n = t.size();
  for (size_t i = 0; i < n; ++i) {
    t.split_type[i] = split_type[i] ? 1 : 0;
    if (t.split_type[i]) t.any_cat = true;
    for (int w8 = 0; w8 < 8; ++w8) t.cat_bits[i * 8 + w8] = split_type[i] ? cat_bits[i * 8 + w8] : 0u;
  }
  b->d_trees_synced = 0; b->paths_synced = -1; b->margin_ready = false;
  for (auto& kv : b->eval_cache) if (kv.second) kv.second->n_trees_applied = 0, kv.second->n = -1;
  API_END
}
int B2_BoosterGetTimers(B2Handle bh, int32_t reset, char* out, int64_t out_cap) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  const Timers& t = b->t;
  snprintf(out, (size_t)out_cap,
           "{\"hist_ms\": %.6f, \"hist_launches\": %lld, \"hist_rows\": %lld, \"hist_bytes\": %.1f, \"kernel_launches\": %lld, "
           "\"round_ms\": %.6f, \"rounds\": %lld, \"allreduce_bytes\": %.1f, \"num_sms\": %d, \"n_groups\": %d, \"row_stride\": %d, "
           "\"phase_ms\": {\"quant\": %.4f, \"hist\": %.4f, \"allreduce\": %.4f, \"subtract\": %.4f, \"eval_decide\": %.4f, "
           "\"partition_finalize\": %.4f, \"leaf\": %.4f}, \"shap_ms\": %.6f, \"shap_rows\": %lld}",
           t.hist_ms, t.hist_launches, t.hist_rows, t.hist_bytes, t.kernel_launches, t.round_ms, t.rounds, t.allreduce_bytes,
           b->ctx->num_sms, b->train ? b->train->n_groups : 0, b->train ? b->train->row_stride : 0, t.phase_ms[0], t.phase_ms[1],
           t.phase_ms[2], t.phase_ms[3], t.phase_ms[4], t.phase_ms[5], t.phase_ms[6], t.shap_ms, t.shap_rows);
  if (reset) b->t.reset();
  API_END
}
int B2_BoosterCancel(B2Handle bh) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  b->cancel.store(true);
  API_END
}
int B2_BoosterFree(B2Handle bh) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  cudaSetDevice(b->ctx->device);
  delete b;
  API_END
}

int B2_HistBuildRaw(const uint8_t* bins, int64_t n_rows, int32_t n_cols, const int32_t* qg, const int32_t* qh,
                    const int32_t* ridx, int64_t n_sel, int32_t window_rows, int32_t chunk_rows, int device, int64_t* out,
                    float* kernel_ms) {
  API_BEGIN
  Ctx* ctx = get_ctx(device); cudaStream_t s = ctx->stream;
  Matrix m; m.kind = kMatrix; m.ctx = ctx; m.n = n_rows; m.F = n_cols;
  setup_groups(&m);
  std::vector<uint8_t> padded((size_t)std::max<int64_t>(n_rows, 1) * m.row_stride, 0);
  for (int64_t i = 0; i < n_rows; ++i)
    for (int f = 0; f < n_cols; ++f) padded[(size_t)i * m.row_stride + m.feat_byte[f]] = bins[i * n_cols + f];
  std::vector<int2> gp((size_t)std::max<int64_t>(n_rows, 1));
  for (int64_t i = 0; i < n_rows; ++i) gp[i] = make_int2(qg[i], qh[i]);
  DevBuf<uint8_t> d_bins; DevBuf<int2> d_gp; DevBuf<int32_t> d_ridx; DevBuf<long long> d_hist; DevBuf<B2HistWork> d_work;
  d_bins.ensure(padded.size()); d_gp.ensure(gp.size());
  CUDA_CHECK(cudaMemcpyAsync(d_bins.p, padded.data(), padded.size(), cudaMemcpyHostToDevice, s));
  CUDA_CHECK(cudaMemcpyAsync(d_gp.p, gp.data(), gp.size() * sizeof(int2), cudaMemcpyHostToDevice, s));
  if (ridx) {
    d_ridx.ensure((size_t)std::max<int64_t>(n_sel, 1));
    if (n_sel > 0) CUDA_CHECK(cudaMemcpyAsync(d_ridx.p, ridx, n_sel * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  }
  const size_t node_elems = (size_t)m.n_groups * B2_GROUP_ELEMS;
  d_hist.ensure(node_elems);
  CUDA_CHECK(cudaMemsetAsync(d_hist.p, 0, node_elems * sizeof(long long), s));
  if (window_rows <= 0) window_rows = 4096;
  if (chunk_rows <= 0) chunk_rows = 2048;
  if (chunk_rows > window_rows) chunk_rows = window_rows;
  B2HistWork w{0, (int32_t)n_sel, 0, 0};
  d_work.ensure(1);
  CUDA_CHECK(cudaMemcpyAsync(d_work.p, &w, sizeof(w), cudaMemcpyHostToDevice, s));
  const int chunks = (int)((n_sel + chunk_rows - 1) / chunk_rows);
  cudaEvent_t e0, e1; CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
  CUDA_CHECK(cudaEventRecord(e0, s));
  if (n_sel > 0)
  {
    alignas(64) unsigned char tt[128];
    if (use_tma_hist() && b2_make_bins_tensor_map(tt, d_bins.p, n_rows, m.row_stride, 64) == 0)
      LAUNCH_CHECK(b2_launch_hist_tma(d_bins.p, m.row_stride, tt, d_gp.p, ridx ? d_ridx.p : nullptr, d_work.p, 1, chunks, chunk_rows, window_rows, m.n_groups,
                                      d_hist.p, nullptr, 0, 1, n_rows, ctx->num_sms, s));
    else
      LAUNCH_CHECK(b2_launch_hist(d_bins.p, m.row_stride, d_gp.p, ridx ? d_ridx.p : nullptr, d_work.p, 1, chunks, chunk_rows,
                                  window_rows, m.n_groups, d_hist.p, nullptr, 0, 1, m.narrow_w, ctx->num_sms, s));
  }
  CUDA_CHECK(cudaEventRecord(e1, s));
  std::vector<long long> h(node_elems);
  CUDA_CHECK(cudaMemcpyAsync(h.data(), d_hist.p, node_elems * sizeof(long long), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  if (kernel_ms) { float ms = 0; cudaEventElapsedTime(&ms, e0, e1); *kernel_ms = ms; }
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  for (int f = 0; f < n_cols; ++f) {
    const int g = m.feat_byte[f] / B2_GROUP_SLOTS, sl = m.feat_byte[f] % B2_GROUP_SLOTS;
    for (int bb = 0; bb < 256; ++bb) {
      out[((size_t)f * 256 + bb) * 2] = h[(size_t)g * B2_GROUP_ELEMS + bb * 32 + sl];
      out[((size_t)f * 256 + bb) * 2 + 1] = h[(size_t)g * B2_GROUP_ELEMS + B2_PLANE_ELEMS + bb * 32 + sl];
    }
  }
  API_END
}

}  // extern "C"
