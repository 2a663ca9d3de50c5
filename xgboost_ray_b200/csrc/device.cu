// device.cu -- the device context of every GPU, the caching device-memory pool, the pinned host -> device upload
// pipeline, and the NCCL communicator (libnccl is loaded with dlopen on first use).
#include <dlfcn.h>
#include <errno.h>
#include <sys/types.h>
#include <sys/uio.h>
#include <stdlib.h>
#include <string.h>

#include <thread>

#include "host.h"

namespace b2host __attribute__((visibility("hidden"))) {

// ---------------------------------------------------------------- device context
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

// the caching device-memory pool (DevPool in host.h says why)
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
void allreduce(Comm* c, void* buf, size_t count, int dtype, int op, cudaStream_t s) {
  if (!c || c->world <= 1 || count == 0) return;
  if (c->aborted.load()) fail("communicator aborted");
  NCCL_CHECK(nccl()->AllReduce(buf, buf, count, dtype, op, c->comm, s));
}

}  // namespace b2host
