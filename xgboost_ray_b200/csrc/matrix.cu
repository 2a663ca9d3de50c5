// matrix.cu -- the matrix lifecycle (construction, the registry, the interleaved NVLink ingest), the feature -> group
// layout of the bin matrix, the GPU sketch that makes the cuts, the checks of categorical codes, and the binning of the
// raw values.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <chrono>
#include <climits>

#include "host.h"
#include "launch.h"

namespace b2host __attribute__((visibility("hidden"))) {

// A quantised matrix normally keeps two byte copies of its bins: bins [n][row_stride] (row-major, read by the histogram
// build and the DART walk) and bins_col [F][col_stride] (feature-major, read by the partition and the final assign).
// The CSR layout keeps ebins [nnz] instead, one bin per stored entry aligned with the CSR's indices; csr_indptr /
// csr_indices then stay on the device after the raw values are released (DESIGN.md 2 item 26).
struct MatrixBins {
  bool csr_bins = false;
  DevBuf<uint8_t> bins, bins_col, ebins;
  int64_t col_stride = 0;
};
Matrix::Matrix() : qbins(new MatrixBins()) {}
Matrix::~Matrix() = default;

// ids of the matrices that are alive: a Booster's evaluation cache is keyed by the id, never by the address (a freed
// matrix and a new one of the same shape can share an address)
static std::mutex g_matrix_mu;
static std::set<uint64_t> g_live_matrices;
static uint64_t g_next_matrix_uid = 1;
std::unique_ptr<Matrix> new_matrix(int64_t n, int F, float missing) {
  if (n < 0 || F <= 0) fail("invalid matrix shape %lld x %d", (long long)n, F);
  if (n >= (1LL << 31)) fail("at most 2^31-1 rows per GPU shard (row ids are int32), got %lld", (long long)n);
  std::unique_ptr<Matrix> m(new Matrix());
  m->kind = kMatrix; m->n = n; m->F = F; m->missing = missing;
  return m;
}
B2Handle register_matrix(std::unique_ptr<Matrix> m) {
  { std::lock_guard<std::mutex> lk(g_matrix_mu); m->uid = g_next_matrix_uid++; g_live_matrices.insert(m->uid); }
  return (B2Handle)m.release();
}
void free_matrix(Matrix* m) {
  { std::lock_guard<std::mutex> lk(g_matrix_mu); g_live_matrices.erase(m->uid); }
  delete m;
}
bool matrix_alive(uint64_t uid) { std::lock_guard<std::mutex> lk(g_matrix_mu); return g_live_matrices.count(uid) != 0; }

void upload_raw(Matrix* m, const UploadSource& u) {
  m->raw.ensure((size_t)std::max<int64_t>(m->n * m->F, 1));
  upload_pipelined(m->ctx, m->raw.p, u, (size_t)m->n * m->F * sizeof(float));
  m->has_raw = true;
}

// Staging block of the interleaved ingest: persistent per device (grow-only), exported ONCE; the peers keep their mapping
// of it across calls (mapping / unmapping a multi-GB allocation costs more than moving the rows).  A block that had to
// grow is retired and freed only after the call's closing barrier, when every peer has dropped its mapping of it.
struct IngestStage { float* p = nullptr; size_t bytes = 0; cudaIpcMemHandle_t h; bool exported = false; };
static IngestStage g_ingest_stage[64];
static std::map<std::string, void*> g_peer_stage;      // handle bytes -> mapped pointer (this process)
static std::mutex g_ingest_mu;
static double wall_seconds() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

B2Handle ingest_interleaved(Comm* c, int64_t pid, uint64_t remote_addr, int64_t n_total_rows, int n_cols, int shard_rank,
                            float missing, int device) {
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
  B2RowBlocks rb; memset(&rb, 0, sizeof(rb));
  const int64_t per = n_total_rows / W, extra = n_total_rows % W;
  for (int w = 0; w <= W; ++w) rb.start[w] = (long long)(w * per + std::min<int64_t>(w, extra));
  const int64_t b0 = rb.start[rank], bn = rb.start[rank + 1] - b0;
  const int64_t n_mine = rank < n_total_rows ? (n_total_rows - rank + W - 1) / W : 0;
  std::unique_ptr<Matrix> m = new_matrix(n_mine, n_cols, missing);
  m->ctx = ctx;
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
  } catch (...) { if (retired) cudaFree(retired); throw; }
  m->has_raw = true;
  const B2Handle h = register_matrix(std::move(m));
  if (timing) fprintf(stderr, "[b2 ingest rank %d] total %.4f s (%lld of %lld rows x %d)\n", rank, wall_seconds() - t0, (long long)n_mine, (long long)n_total_rows, n_cols);
  return h;
}

// Feature -> (group, slot) layout of the bin matrix: the features are spread EVENLY over ceil(F / 32) groups, so that
// every CTA type of the histogram kernel (one pair of groups) costs the same and the types walk the chunk list in lock
// step -- the CTAs that read the two 64-byte halves of a row do it at the same time and the row is fetched from DRAM
// once.  (Packing the F mod 32 leftover features into a narrow last group saves padding-slot atomics, but the types then
// differ in cost, drift apart and read the halves of a row at different times; DESIGN.md 4.1.)
void setup_groups(Matrix* m) {
  const int F = m->F;
  m->n_groups = (F + B2_GROUP_SLOTS - 1) / B2_GROUP_SLOTS;
  if (m->n_groups < 1) m->n_groups = 1;
  m->row_stride = m->n_groups * B2_GROUP_SLOTS;
  m->group_first.assign(m->n_groups, 0);
  m->group_size.assign(m->n_groups, 0);
  m->feat_byte.assign(F, 0);
  const int base = F / m->n_groups, rem = F % m->n_groups;
  int f = 0;
  for (int g = 0; g < m->n_groups; ++g) {
    const int sz = base + (g < rem ? 1 : 0);
    m->group_first[g] = f; m->group_size[g] = sz;
    for (int s = 0; s < sz; ++s) m->feat_byte[f + s] = g * B2_GROUP_SLOTS + s;
    f += sz;
  }
}

int64_t raw_tile_rows(const Matrix* m) {
  if (!m->csr) return std::max<int64_t>(m->n, 1);
  const int64_t rows = (int64_t)(kRawTileBytes / (4 * (size_t)m->F)) & ~(int64_t)127;
  return std::max<int64_t>(rows, 128);
}

const float* raw_rows(Matrix* m, int64_t r0, int64_t rows, DevBuf<float>& tile) {
  if (!m->has_raw) fail("matrix has no raw data on the device");
  if (!m->csr) return m->raw.p + (size_t)r0 * m->F;
  tile.ensure((size_t)std::max<int64_t>(rows, 1) * m->F);
  LAUNCH_CHECK(b2_launch_csr_densify(m->csr_indptr.p, m->csr_indices.p, m->csr_values.p, r0, rows, m->F, tile.p, m->ctx->num_sms,
                                     m->ctx->stream));
  return tile.p;
}

B2RawRows raw_source(const Matrix* m) {
  if (!m->has_raw) fail("matrix has no raw data on the device");
  if (m->csr) return B2RawRows{nullptr, m->csr_indptr.p, m->csr_indices.p, m->csr_values.p};
  return B2RawRows{m->raw.p, nullptr, nullptr, nullptr};
}

// Uploads the CSR arrays of m (n rows, F columns and nnz set) and checks them on the device in one pass; the first row
// that breaks a rule is named, with the rule read back from the caller's arrays.  The check guards the C ABI: an
// out-of-range column would be written outside a densified tile.  A matrix in the CSR bin layout kept indptr and
// indices on the device with its bins (release_raw): only the values come back.
void upload_csr(Matrix* m, const int64_t* indptr, const int32_t* indices, const float* values) {
  Ctx* ctx = m->ctx; cudaStream_t s = ctx->stream;
  const int64_t n = m->n, nnz = m->nnz;
  if (m->qbins->csr_bins) {
    m->csr_values.ensure((size_t)nnz);
    upload_pipelined(ctx, m->csr_values.p, values, (size_t)nnz * sizeof(float));
    m->has_raw = true;
    return;
  }
  m->csr_indptr.ensure((size_t)n + 1); m->csr_indices.ensure((size_t)nnz); m->csr_values.ensure((size_t)nnz);
  upload_pipelined(ctx, m->csr_indptr.p, indptr, ((size_t)n + 1) * sizeof(int64_t));
  upload_pipelined(ctx, m->csr_indices.p, indices, (size_t)nnz * sizeof(int32_t));
  upload_pipelined(ctx, m->csr_values.p, values, (size_t)nnz * sizeof(float));
  if (n == 0) {
    if (indptr[0] != 0 || nnz != 0) fail("CSR matrix without rows: indptr[0] = %lld and nnz = %lld must be 0", (long long)indptr[0], (long long)nnz);
    m->has_raw = true;
    return;
  }
  DevBuf<unsigned long long> d_bad; d_bad.ensure(1);
  LAUNCH_CHECK(b2_launch_csr_validate(m->csr_indptr.p, m->csr_indices.p, n, m->F, nnz, d_bad.p, ctx->num_sms, s));
  unsigned long long bad = 0;
  CUDA_CHECK(cudaMemcpyAsync(&bad, d_bad.p, sizeof(bad), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  if (bad != ~0ull) {
    const int64_t i = (int64_t)bad, b = indptr[i], e = indptr[i + 1];
    if (i == 0 && b != 0) fail("CSR row 0: indptr[0] = %lld, must be 0", (long long)b);
    if (b > e) fail("CSR row %lld: indptr decreases (indptr[%lld] = %lld > indptr[%lld] = %lld)", (long long)i, (long long)i,
                    (long long)b, (long long)(i + 1), (long long)e);
    if (b < 0 || e > nnz) fail("CSR row %lld: entries [%lld, %lld) outside the %lld stored entries", (long long)i, (long long)b,
                               (long long)e, (long long)nnz);
    for (int64_t k = b; k < e; ++k) {
      const int c = indices[k];
      if (c < 0 || c >= m->F) fail("CSR row %lld: column %d is outside [0, %d)", (long long)i, c, m->F);
      if (k > b && c == indices[k - 1]) fail("CSR row %lld: column %d is stored twice", (long long)i, c);
      if (k > b && c < indices[k - 1])
        fail("CSR row %lld: column %d follows column %d (the columns of a row must increase)", (long long)i, c, indices[k - 1]);
    }
    fail("CSR row %lld: indptr[%lld] = %lld, must equal nnz = %lld", (long long)i, (long long)(i + 1), (long long)e, (long long)nnz);
  }
  m->has_raw = true;
}

// The slice holds raw values (dense or CSR, as the parent) and the gathered side arrays, and is quantised with its own
// cuts when it is first trained or evaluated.  The parent is only read.
B2Handle slice_matrix(Matrix* p, const int64_t* rows, int64_t n) {
  if (n < 1) fail("slice: no row index given (a slice needs at least one row)");
  for (int64_t i = 0; i < n; ++i)
    if (rows[i] < 0 || rows[i] >= p->n)
      fail("slice: row index %lld (position %lld) is outside [0, %lld)", (long long)rows[i], (long long)i, (long long)p->n);
  if (!p->has_raw) fail("slice: the matrix has no raw data on the device (re-upload it with B2_MatrixEnsureRaw / B2_MatrixEnsureRawCSR)");
  std::unique_ptr<Matrix> m = new_matrix(n, p->F, p->missing);
  Ctx* ctx = p->ctx; cudaStream_t s = ctx->stream;
  m->ctx = ctx;
  DevBuf<int64_t> d_rows;
  upload(d_rows, rows, (size_t)n, s);
  if (p->csr) {
    m->csr = true;
    m->bin_layout = p->qbins->csr_bins ? B2_BIN_LAYOUT_CSR : p->bin_layout;
    m->csr_indptr.ensure((size_t)n + 1);
    DevBuf<int64_t> lengths; lengths.ensure((size_t)n);
    DevBuf<uint8_t> temp; const size_t tb = b2_csr_slice_temp_bytes(n); temp.ensure(std::max<size_t>(tb, 1));
    LAUNCH_CHECK(b2_launch_csr_slice_indptr(p->csr_indptr.p, d_rows.p, n, lengths.p, m->csr_indptr.p, temp.p, tb, ctx->num_sms, s));
    int64_t nnz = 0;
    CUDA_CHECK(cudaMemcpyAsync(&nnz, m->csr_indptr.p + n, sizeof(nnz), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    m->nnz = nnz;
    m->csr_indices.ensure((size_t)nnz); m->csr_values.ensure((size_t)nnz);   // the capacities B2_MatrixCreateFromCSR gives
    LAUNCH_CHECK(b2_launch_csr_slice_entries(p->csr_indptr.p, p->csr_indices.p, p->csr_values.p, d_rows.p, n, m->csr_indptr.p,
                                             m->csr_indices.p, m->csr_values.p, ctx->num_sms, s));
  } else {
    m->raw.ensure((size_t)n * p->F);
    LAUNCH_CHECK(b2_launch_gather_rows(p->raw.p, p->F, d_rows.p, n, m->raw.p, ctx->num_sms, s));
  }
  m->has_raw = true;
  // a per-row array of `len` values ([p->n][len / p->n]; len 0 = not set)
  auto gather = [&](const DevBuf<float>& src, int64_t len, DevBuf<float>& dst, int64_t* dst_len) {
    if (len == 0) return;
    const int64_t width = len / p->n;
    dst.ensure((size_t)n * width);
    LAUNCH_CHECK(b2_launch_gather_rows(src.p, width, d_rows.p, n, dst.p, ctx->num_sms, s));
    *dst_len = n * width;
  };
  gather(p->label, p->n_label, m->label, &m->n_label);
  m->n_targets = p->n_targets;
  gather(p->weight, p->n_weight, m->weight, &m->n_weight);
  gather(p->base_margin, p->n_base_margin, m->base_margin, &m->n_base_margin);
  gather(p->lower, p->n_lower, m->lower, &m->n_lower);
  gather(p->upper, p->n_upper, m->upper, &m->n_upper);
  m->is_cat = p->is_cat; m->cat_feats = p->cat_feats;
  m->fwq = p->fwq;
  if (!m->fwq.empty()) upload(m->d_fwq, m->fwq, s);
  CUDA_CHECK(cudaStreamSynchronize(s));
  return register_matrix(std::move(m));
}

// the CSR bin layout keeps indptr and indices: they locate its bins
static void release_raw(Matrix* m) {
  m->raw.release();
  if (!m->qbins->csr_bins) { m->csr_indptr.release(); m->csr_indices.release(); }
  m->csr_values.release();
  m->has_raw = false;
}

template <typename T>
static size_t buf_bytes(const DevBuf<T>& d) { return d.cap * sizeof(T); }
size_t matrix_device_bytes(const Matrix* m) {
  const MatrixBins& q = *m->qbins;
  return buf_bytes(m->raw) + buf_bytes(m->csr_indptr) + buf_bytes(m->csr_indices) + buf_bytes(m->csr_values) +
         buf_bytes(q.bins) + buf_bytes(q.bins_col) + buf_bytes(q.ebins) + buf_bytes(m->d_group_first) + buf_bytes(m->d_group_size) +
         buf_bytes(m->d_feat_byte) + buf_bytes(m->d_cut_ptrs) + buf_bytes(m->d_nbins) + buf_bytes(m->d_cat_feats) +
         buf_bytes(m->d_cut_vals) + buf_bytes(m->d_has_missing) + buf_bytes(m->d_is_cat) + buf_bytes(m->label) +
         buf_bytes(m->weight) + buf_bytes(m->base_margin) + buf_bytes(m->lower) + buf_bytes(m->upper) +
         buf_bytes(m->qgroup_ptr) + buf_bytes(m->d_fwq);
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

// Categorical features: global {max code, has missing, largest invalid value's key} per entry of m->cat_feats
// (cat_stats_kernel, allreduce max over the ranks).  Synchronises the stream.
std::vector<int32_t> category_stats(Matrix* m, Comm* comm) {
  cudaStream_t s = m->ctx->stream;
  const int n_cat = (int)m->cat_feats.size();
  std::vector<int32_t> h_cat((size_t)n_cat * 3);
  if (n_cat == 0) { CUDA_CHECK(cudaStreamSynchronize(s)); return h_cat; }   // callers read earlier copies after this
  for (int i = 0; i < n_cat; ++i) { h_cat[i * 3] = -1; h_cat[i * 3 + 1] = 0; h_cat[i * 3 + 2] = INT_MIN; }
  DevBuf<int32_t> d_cat, d_catf;
  d_cat.ensure((size_t)n_cat * 3); d_catf.ensure((size_t)n_cat);
  CUDA_CHECK(cudaMemcpyAsync(d_cat.p, h_cat.data(), (size_t)n_cat * 3 * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  CUDA_CHECK(cudaMemcpyAsync(d_catf.p, m->cat_feats.data(), (size_t)n_cat * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  if (m->csr) {   // one pass over the stored entries; a feature some row does not store has a missing value
    if (!m->has_raw) fail("matrix has no raw data on the device");
    std::vector<int32_t> cat_of(m->F, -1);
    for (int i = 0; i < n_cat; ++i) cat_of[m->cat_feats[i]] = i;
    DevBuf<int32_t> d_cat_of; DevBuf<unsigned long long> d_stored;
    upload(d_cat_of, cat_of, s); d_stored.ensure((size_t)n_cat);
    LAUNCH_CHECK(b2_launch_csr_cat_stats(m->csr_indices.p, m->csr_values.p, m->nnz, m->n, m->missing, d_cat_of.p, n_cat, d_stored.p,
                                         d_cat.p, m->ctx->num_sms, s));
    allreduce(comm, d_cat.p, (size_t)n_cat * 3, kNcclInt32, kNcclMax, s);
    CUDA_CHECK(cudaMemcpyAsync(h_cat.data(), d_cat.p, (size_t)n_cat * 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    return h_cat;
  }
  for_raw_tiles(m, [&](const float* X, int64_t, int64_t rows) {   // the stats are maxima: they accumulate over the tiles
    LAUNCH_CHECK(b2_launch_cat_stats(X, rows, m->F, m->missing, d_catf.p, n_cat, d_cat.p, m->ctx->num_sms, s));
  });
  allreduce(comm, d_cat.p, (size_t)n_cat * 3, kNcclInt32, kNcclMax, s);
  CUDA_CHECK(cudaMemcpyAsync(h_cat.data(), d_cat.p, (size_t)n_cat * 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  return h_cat;
}
// the value behind cat_stats_kernel's signed order-preserving key
double category_key_value(int32_t key) {
  const uint32_t k = (uint32_t)key ^ 0x80000000u;
  const uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  float f; memcpy(&f, &u, sizeof(f));
  return (double)f;
}

// Borrowed cuts (a ref matrix, or the frozen cuts of a restart) were made from other data.  bin_kernel clamps a code
// they do not know to their largest code (a negative one to 0), and a code of 255 shares bin 255 with the missing
// values, while prediction sends every unknown code left: training would see another category than predict().
// Such codes are refused, as make_cuts refuses codes that are not valid, instead of silently changing the model.
static void check_borrowed_categories(Matrix* m, Comm* comm) {
  const std::vector<int32_t> h_cat = category_stats(m, comm);
  for (size_t i = 0; i < m->cat_feats.size(); ++i) {
    const int f = m->cat_feats[i], mx = h_cat[i * 3], miss = h_cat[i * 3 + 1];
    const int known = m->cut_ptrs[f + 1] - m->cut_ptrs[f] - 1;   // the cuts of a categorical feature are the codes 0..known
    if (h_cat[i * 3 + 2] != INT_MIN)
      fail("categorical feature %d: category codes must be integers in [0, %d], got %.9g", f, known,
           category_key_value(h_cat[i * 3 + 2]));
    if (mx > known)
      fail("categorical feature %d: category code %d is above the largest code %d of the cuts this matrix is binned with",
           f, mx, known);
    if (miss && known > 254)
      fail("categorical feature %d: the feature has missing values, but its cuts use bin 255 (the missing sentinel) for "
           "category code 255", f);
    // cuts borrowed from a matrix without missing values: the split scan and partition must still treat bin 255 as
    // missing (default direction), as prediction does, instead of as an unknown category.  The oracle applies the same
    // rule when it trains with borrowed cuts (oracle.train(cuts=...), Cuts.borrowed_by).
    if (miss) m->has_missing[f] = 1;
  }
}

// Sketch of a CSR matrix's numeric features from its stored entries only (DESIGN.md 7 "Sketch over the stored entries").
// A feature's valid keys are the keys the dense twin's sort puts ahead of its missing sentinels, in the same order, so
// the summaries and cuts are the twin's.  Features are taken in batches of at most kSketchBatchEntries valid entries
// (summed over the ranks; a feature with more is a batch of its own).  Per batch each rank keys its entries into their
// feature's segment; with several ranks the blocks are allgathered, padded to the largest rank's block with sentinels
// that sort last.  Every rank sorts the batch, the owner rank of a feature (f % world) prunes it into the table.
constexpr int64_t kSketchBatchEntries = (int64_t)1 << 24;   // tests/test_gpu_sparse_native.py BATCH_ENTRIES
static void sketch_csr(Matrix* m, Comm* comm, int max_bin, long long n_global, const int32_t* wq, float* d_cuts, int32_t* d_ncuts,
                       float* d_mins, int32_t* d_hasmiss) {
  Ctx* ctx = m->ctx; cudaStream_t s = ctx->stream;
  const int world = comm ? comm->world : 1, rank = comm ? comm->rank : 0, F = m->F;
  DevBuf<uint8_t> d_iscat; upload(d_iscat, m->is_cat, s);
  // valid entries per feature of every rank: [world][F]
  DevBuf<unsigned long long> d_counts;
  d_counts.ensure((size_t)world * F);
  unsigned long long* mine = d_counts.p + (size_t)rank * F;
  CUDA_CHECK(cudaMemsetAsync(mine, 0, (size_t)F * sizeof(unsigned long long), s));
  LAUNCH_CHECK(b2_launch_csr_column_counts(m->csr_indices.p, m->csr_values.p, m->nnz, m->missing, d_iscat.p, mine, ctx->num_sms, s));
  if (world > 1) NCCL_CHECK(nccl()->AllGather(mine, d_counts.p, (size_t)F, kNcclUint64, comm->comm, s));
  std::vector<unsigned long long> cnt((size_t)world * F);
  CUDA_CHECK(cudaMemcpyAsync(cnt.data(), d_counts.p, cnt.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  std::vector<int64_t> total(F, 0);
  for (int r = 0; r < world; ++r)
    for (int f = 0; f < F; ++f) total[f] += (int64_t)cnt[(size_t)r * F + f];
  // batches [f0, f1): the same on every rank (planned from the global counts)
  std::vector<std::pair<int, int>> batches;
  int64_t max_local = 1, max_sort = 1;
  for (int f0 = 0; f0 < F;) {
    int f1 = f0; int64_t e = 0;
    while (f1 < F && (f1 == f0 || e + total[f1] <= kSketchBatchEntries)) e += total[f1++];
    int64_t emax = 0;
    for (int r = 0; r < world; ++r) {
      int64_t er = 0;
      for (int f = f0; f < f1; ++f) er += (int64_t)cnt[(size_t)r * F + f];
      emax = std::max(emax, er);
    }
    if (e >= ((int64_t)1 << 31)) fail("sketch: %lld valid entries in features [%d, %d) exceed the int32 summary index", (long long)e, f0, f1);
    max_local = std::max(max_local, emax);
    max_sort = std::max(max_sort, world > 1 ? emax * world : e);
    batches.push_back({f0, f1});
    f0 = f1;
  }
  // scratch: peak bytes = max_sort * (8 + 8 + 4 + 4 + 4 + 8 [+ 4 + 4 + 8 weighted]) + CUB + world > 1: the local block
  DevBuf<uint64_t> keys_local, keys_all, keys_sorted; DevBuf<int32_t> wq_local, wq_all, wq_sorted, flags, idx;
  DevBuf<float> uval; DevBuf<long long> rmin, wpre; DevBuf<int64_t> d_seg; DevBuf<unsigned int> d_cursor; DevBuf<uint8_t> temp;
  keys_local.ensure((size_t)max_local);
  if (world > 1) keys_all.ensure((size_t)max_sort);
  keys_sorted.ensure((size_t)max_sort); flags.ensure((size_t)max_sort); idx.ensure((size_t)max_sort); uval.ensure((size_t)max_sort);
  rmin.ensure((size_t)max_sort);
  if (wq) {
    wq_local.ensure((size_t)max_local); wq_sorted.ensure((size_t)max_sort); wpre.ensure((size_t)max_sort);
    if (world > 1) wq_all.ensure((size_t)max_sort);
  }
  const size_t temp_bytes = b2_sketch_batch_temp_bytes(max_sort);
  temp.ensure(temp_bytes ? temp_bytes : 1);
  d_seg.ensure((size_t)F + 1); d_cursor.ensure((size_t)F);
  for (const auto& bt : batches) {
    const int f0 = bt.first, nf = bt.second - f0;
    std::vector<int64_t> seg(nf + 1, 0);
    std::vector<unsigned int> cursor(nf, 0);
    int64_t local = 0, emax = 0;
    for (int j = 0; j < nf; ++j) {
      seg[j + 1] = seg[j] + total[f0 + j];
      cursor[j] = (unsigned int)local;
      local += (int64_t)cnt[(size_t)rank * F + f0 + j];
    }
    for (int r = 0; r < world; ++r) {
      int64_t er = 0;
      for (int j = 0; j < nf; ++j) er += (int64_t)cnt[(size_t)r * F + f0 + j];
      emax = std::max(emax, er);
    }
    // the local block is in feature-segment order; with several ranks the sort regroups the gathered blocks, whose
    // per-feature order the global segments in seg describe
    upload(d_seg, seg, s); upload(d_cursor, cursor, s);
    LAUNCH_CHECK(b2_launch_csr_sketch_keys(m->csr_indptr.p, m->csr_indices.p, m->csr_values.p, m->n, f0, nf, m->missing, d_iscat.p,
                                           wq, d_cursor.p, keys_local.p, wq ? wq_local.p : nullptr, ctx->num_sms, s));
    const uint64_t* kin = keys_local.p; const int32_t* win = wq ? wq_local.p : nullptr;
    int64_t n_sort = local;
    if (world > 1) {
      if (emax > local) {
        CUDA_CHECK(cudaMemsetAsync(keys_local.p + local, 0xff, (size_t)(emax - local) * sizeof(uint64_t), s));
        if (wq) CUDA_CHECK(cudaMemsetAsync(wq_local.p + local, 0, (size_t)(emax - local) * sizeof(int32_t), s));
      }
      if (emax > 0) {
        NCCL_CHECK(nccl()->AllGather(keys_local.p, keys_all.p, (size_t)emax, kNcclUint64, comm->comm, s));
        if (wq) NCCL_CHECK(nccl()->AllGather(wq_local.p, wq_all.p, (size_t)emax, kNcclInt32, comm->comm, s));
      }
      kin = keys_all.p; win = wq ? wq_all.p : nullptr; n_sort = emax * world;
    }
    LAUNCH_CHECK(b2_sketch_batch(kin, win, keys_sorted.p, wq_sorted.p, wpre.p, n_sort, d_seg.p, seg.data(), f0, nf, d_iscat.p, world,
                                 rank, n_global, temp.p, temp_bytes, flags.p, idx.p, uval.p, rmin.p, max_bin, d_cuts, d_ncuts, d_mins,
                                 d_hasmiss, ctx->num_sms, s));
    CUDA_CHECK(cudaStreamSynchronize(s));   // seg and cursor are host vectors of this iteration
  }
}

// Sketch of a dense matrix's numeric features: the keys of kExtractBatch columns per pass, every column of n_pad keys
// per rank (padding rows and missing values are the 0xffffffff sentinel).  Multi-GPU: the column keys and the integer
// weights of every rank are allgathered (padded to the largest shard); feature f is sorted and pruned only by its owner
// rank f % world.
static void sketch_dense(Matrix* m, Comm* comm, int max_bin, int64_t n_pad, long long n_global, const int32_t* wq_local,
                         float* d_cuts, int32_t* d_ncuts, float* d_mins, int32_t* d_hasmiss) {
  Ctx* ctx = m->ctx; cudaStream_t s = ctx->stream;
  const int world = comm ? comm->world : 1, rank = comm ? comm->rank : 0;
  const int64_t n_total = n_pad * world;
  const int B = b2_extract_batch(); const int F = m->F;
  DevBuf<uint32_t> keys_local, keys_all, keys_sorted;
  DevBuf<int32_t> flags, idx, m_scratch, wq_all, wq_sorted; DevBuf<float> uval; DevBuf<long long> rmin, nvalid, wpre;
  DevBuf<uint8_t> temp;
  const size_t nt = (size_t)std::max<int64_t>(n_total, 1);
  keys_local.ensure((size_t)std::max<int64_t>(n_pad, 1) * B);
  if (world > 1) keys_all.ensure(nt);
  keys_sorted.ensure(nt); flags.ensure(nt); idx.ensure(nt); uval.ensure(nt); rmin.ensure(nt); m_scratch.ensure(1); nvalid.ensure(2);
  const int32_t* wq = wq_local;
  if (wq_local) {
    if (world > 1) {
      wq_all.ensure(nt);
      NCCL_CHECK(nccl()->AllGather(wq_local, wq_all.p, (size_t)n_pad, kNcclInt32, comm->comm, s));
      wq = wq_all.p;
    }
    wq_sorted.ensure(nt); wpre.ensure(nt);
  }
  const size_t temp_bytes = b2_sort_temp_bytes(n_total > 0 ? n_total : 1);
  temp.ensure(temp_bytes ? temp_bytes : 1);
  for (int f0 = 0; f0 < F; f0 += B) {
    const int nf = std::min(B, F - f0);
    bool any_numeric = false;
    for (int j = 0; j < nf; ++j) any_numeric = any_numeric || !m->is_cat[f0 + j];
    if (!any_numeric) continue;
    LAUNCH_CHECK(b2_launch_extract_keys(m->raw.p, m->n, m->F, f0, nf, m->missing, keys_local.p, n_pad, ctx->num_sms, s));
    for (int j = 0; j < nf; ++j) {
      const int f = f0 + j;
      if (m->is_cat[f]) continue;   // categorical: cuts are the codes 0..max (make_cuts)
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
  CUDA_CHECK(cudaStreamSynchronize(s));   // the scratch buffers are freed on return
}

// GPU sketch: exact global summary per feature -> cuts (sketch.cu).  No host round trip per feature.  Each feature is
// sketched by one owner rank (sketch_dense, sketch_csr), and the cut tables are merged with one integer allreduce
// (non-owners contribute zeros), so every rank ends up with identical global cuts.
static void make_cuts(Matrix* m, Comm* comm, int max_bin) {
  Ctx* ctx = m->ctx; cudaStream_t s = ctx->stream;
  if (max_bin < 2 || max_bin > 256) fail("max_bin must be in [2, 256] (uint8 bin matrix), got %d", max_bin);
  if (!m->has_raw) fail("matrix has no raw data to sketch");
  const int world = comm ? comm->world : 1;
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
  const int64_t n_pad = h_cnt[0]; const long long n_global = h_cnt[1];
  const int F = m->F;
  DevBuf<int32_t> d_tab;   // [F*256 cut bits][F n_cuts][F min bits][F has_missing]
  // sample weights make the sketch a weighted one (xgboost SketchContainer pushes info.weights_): quantise them to
  // integers with a global power-of-two scale so that the weighted ranks are exact and identical on every rank
  DevBuf<int32_t> wq_local; DevBuf<uint32_t> d_wmax;
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
    }
  }
  const size_t tab_n = (size_t)F * 256 + 3 * (size_t)F;
  d_tab.ensure(tab_n);
  CUDA_CHECK(cudaMemsetAsync(d_tab.p, 0, tab_n * sizeof(int32_t), s));
  float* d_cuts = (float*)d_tab.p; int32_t* d_ncuts = d_tab.p + (size_t)F * 256;
  float* d_mins = (float*)(d_ncuts + F); int32_t* d_hasmiss = d_ncuts + 2 * (size_t)F;
  if (m->is_cat.empty()) m->is_cat.assign(F, 0);
  if (m->csr) sketch_csr(m, comm, max_bin, n_global, wq, d_cuts, d_ncuts, d_mins, d_hasmiss);
  else sketch_dense(m, comm, max_bin, n_pad, n_global, wq, d_cuts, d_ncuts, d_mins, d_hasmiss);
  // merge the per-owner tables: exact because every entry is written by exactly one rank (others hold 0 bits)
  allreduce(comm, d_tab.p, tab_n, kNcclInt32, kNcclSum, s);
  std::vector<int32_t> h_tab(tab_n);
  CUDA_CHECK(cudaMemcpyAsync(h_tab.data(), d_tab.p, tab_n * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  const int n_cat = (int)m->cat_feats.size();
  const std::vector<int32_t> h_cat = category_stats(m, comm);   // synchronises the stream
  for (int i = 0; i < n_cat; ++i) {
    const int f = m->cat_feats[i], mx = h_cat[i * 3], miss = h_cat[i * 3 + 1];
    if (h_cat[i * 3 + 2] != INT_MIN || (miss && mx > 254))
      fail("categorical feature %d: category codes must be integers in [0, %d]%s, got %.9g", f, miss ? 254 : 255,
           miss ? " (the feature has missing values; bin 255 is the missing sentinel)" : "",
           h_cat[i * 3 + 2] != INT_MIN ? category_key_value(h_cat[i * 3 + 2]) : (double)mx);
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

size_t dense_bin_bytes(int64_t n, int F) {
  Matrix t; t.F = F;
  setup_groups(&t);
  const int64_t rows = std::max<int64_t>(n, 1), col_stride = (rows + 127) & ~(int64_t)127;
  return (size_t)rows * t.row_stride + (size_t)col_stride * F;
}

// "auto" takes the CSR layout only where the two dense copies would not fit: above half of the device's memory
static bool use_csr_bins(const Matrix* m) {
  if (!m->csr || m->bin_layout == B2_BIN_LAYOUT_DENSE) return false;
  if (m->bin_layout == B2_BIN_LAYOUT_CSR) return true;
  cudaDeviceProp prop;
  CUDA_CHECK(cudaGetDeviceProperties(&prop, m->ctx->device));
  return dense_bin_bytes(m->n, m->F) > prop.totalGlobalMem / 2;
}

static void bin_matrix(Matrix* m) {
  Ctx* ctx = m->ctx; cudaStream_t s = ctx->stream; MatrixBins& q = *m->qbins;
  setup_groups(m);
  upload_cuts(m);
  if (use_csr_bins(m)) {
    q.csr_bins = true;
    q.ebins.ensure((size_t)std::max<int64_t>(m->nnz, 1));
    LAUNCH_CHECK(b2_launch_bin_csr(m->csr_indices.p, m->csr_values.p, m->nnz, m->missing, m->d_cut_ptrs.p, m->d_cut_vals.p,
                                   m->any_cat() ? m->d_is_cat.p : nullptr, q.ebins.p, ctx->num_sms, s));
    CUDA_CHECK(cudaStreamSynchronize(s));
    m->quantized = true;
    return;
  }
  q.bins.ensure((size_t)std::max<int64_t>(m->n, 1) * m->row_stride);
  CUDA_CHECK(cudaMemsetAsync(q.bins.p, 0, (size_t)std::max<int64_t>(m->n, 1) * m->row_stride, s));
  q.col_stride = (std::max<int64_t>(m->n, 1) + 127) & ~(int64_t)127;
  q.bins_col.ensure((size_t)q.col_stride * m->F);
  // both bin kernels write rows [0, rows) of the bins / bins_col they are given and nothing else, so a tile writes its
  // own rows only
  for_raw_tiles(m, [&](const float* X, int64_t r0, int64_t rows) {
    LAUNCH_CHECK(b2_launch_bin(X, rows, m->F, m->missing, m->d_cut_ptrs.p, m->d_cut_vals.p, m->d_feat_byte.p,
                               m->any_cat() ? m->d_is_cat.p : nullptr, m->row_stride, q.bins.p + (size_t)r0 * m->row_stride,
                               q.bins_col.p + r0, q.col_stride, ctx->num_sms, s));
  });
  CUDA_CHECK(cudaStreamSynchronize(s));
  m->quantized = true;
}

void quantize_matrix(Matrix* m, Comm* comm, int max_bin, bool borrowed_cuts, bool keep_raw) {
  if (borrowed_cuts) check_borrowed_categories(m, comm);
  else make_cuts(m, comm, max_bin);
  bin_matrix(m);
  if (!keep_raw) release_raw(m);
}

B2BinRows bin_source(const Matrix* m) {
  if (!m->quantized) fail("matrix is not quantised");
  const MatrixBins& q = *m->qbins;
  if (q.csr_bins) return B2BinRows{nullptr, 0, m->d_feat_byte.p, nullptr, 0, m->csr_indptr.p, m->csr_indices.p, q.ebins.p};
  return B2BinRows{q.bins.p, m->row_stride, m->d_feat_byte.p, q.bins_col.p, q.col_stride, nullptr, nullptr, nullptr};
}

void bins_to_host(const Matrix* m, uint8_t* out) {
  if (!m->quantized) fail("matrix is not quantised");
  const MatrixBins& q = *m->qbins;
  if (q.csr_bins) {
    DevBuf<uint8_t> d; d.ensure((size_t)std::max<int64_t>(m->n * m->F, 1));
    LAUNCH_CHECK(b2_launch_csr_bins_densify(m->csr_indptr.p, m->csr_indices.p, q.ebins.p, m->n, m->F, d.p, m->ctx->num_sms,
                                            m->ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(out, d.p, (size_t)m->n * m->F, cudaMemcpyDeviceToHost, m->ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(m->ctx->stream));
    return;
  }
  std::vector<uint8_t> h((size_t)m->n * m->row_stride);
  if (m->n > 0) CUDA_CHECK(cudaMemcpy(h.data(), q.bins.p, h.size(), cudaMemcpyDeviceToHost));
  for (int64_t i = 0; i < m->n; ++i)
    for (int f = 0; f < m->F; ++f) out[i * m->F + f] = h[(size_t)i * m->row_stride + m->feat_byte[f]];
}

void upload_bins(Matrix* m, const uint8_t* bins) {
  cudaStream_t s = m->ctx->stream; MatrixBins& q = *m->qbins;
  setup_groups(m);
  upload(m->d_feat_byte, m->feat_byte, s); upload(m->d_group_size, m->group_size, s);
  if (m->csr) {
    q.csr_bins = true;
    upload(q.ebins, bins, (size_t)m->nnz, s);
  } else {
    std::vector<uint8_t> padded((size_t)std::max<int64_t>(m->n, 1) * m->row_stride, 0);
    for (int64_t i = 0; i < m->n; ++i)
      for (int f = 0; f < m->F; ++f) padded[(size_t)i * m->row_stride + m->feat_byte[f]] = bins[i * m->F + f];
    upload(q.bins, padded, s);   // pageable source: staged before return
  }
  m->quantized = true;
}

}  // namespace b2host
