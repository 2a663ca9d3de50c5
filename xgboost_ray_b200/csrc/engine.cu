// engine.cu -- the C ABI of libb2hist.so (include/b2hist.h).  Every entry point runs inside API_BEGIN / API_END: a
// B2Error (fail) or any other exception becomes the return value -1 and the message of B2_GetLastError.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <climits>
#include <string>
#include <vector>

#include "../../include/b2hist.h"
#include "host.h"
#include "launch.h"

namespace b2host __attribute__((visibility("hidden"))) {

// ---------------------------------------------------------------- errors
thread_local std::string g_last_error;
[[noreturn]] void fail(const char* fmt, ...) {
  char buf[1024];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
  throw B2Error{buf};
}
#define API_BEGIN try {
#define API_END                                            \
  }                                                        \
  catch (const B2Error& e) { g_last_error = e.msg; return -1; } \
  catch (const std::exception& e) { g_last_error = e.what(); return -1; } \
  return 0;

struct CommH : HandleBase { Comm c; };
Comm* comm_of(B2Handle h) { return h ? &from_handle<CommH>(h, kComm, "communicator")->c : nullptr; }   // 0: single process

// the matrix of handle mh, its device made current
Matrix* matrix_of(B2Handle mh) {
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  CUDA_CHECK(cudaSetDevice(m->ctx->device));
  return m;
}
// the booster of handle bh with its pending round finished: every entry that reads or changes the model opens with this
Booster* drained(B2Handle bh) {
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  drain_round(b);
  return b;
}
TreeHost& tree_at(Booster* b, int tree) {
  if (tree < 0 || tree >= (int)b->trees.size()) fail("tree index %d out of range", tree);
  return b->trees[tree];
}

// n host values into a device field of m, copied before return (the caller may reuse its array); n < 0 copies none
template <typename T>
void set_field(Matrix* m, DevBuf<T>& d, const T* values, int64_t n) {
  upload(d, values, (size_t)std::max<int64_t>(n, 0), m->ctx->stream);
  CUDA_CHECK(cudaStreamSynchronize(m->ctx->stream));
}
// an entry that reads matrix mh under the model of booster bh: its pending round drained, the booster's device current
template <typename Fn>
int with_matrix(B2Handle bh, B2Handle mh, Fn fn) {
  API_BEGIN
  Booster* b = drained(bh);
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  CUDA_CHECK(cudaSetDevice(b->ctx->device));
  fn(b, m);
  API_END
}

}  // namespace b2host

using namespace b2host;

// =================================================================== C ABI
extern "C" {

const char* B2_GetLastError(void) { return g_last_error.c_str(); }
int B2_GetVersion(void) { return 100; }
int B2_CheckParams(const char* params) {
  API_BEGIN
  Params p;
  parse_params(params, &p, nullptr);
  API_END
}
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
  std::unique_ptr<Matrix> m = new_matrix(n_rows, n_cols, missing);
  m->ctx = get_ctx(device);
  upload_raw(m.get(), UploadSource{data});
  *out = register_matrix(std::move(m));
  API_END
}
int B2_MatrixCreateFromCSR(int64_t* indptr, const int32_t* indices, const float* values, int64_t n_rows, int32_t n_cols,
                           int64_t nnz, float missing, int device, B2Handle* out) {
  API_BEGIN
  if (n_rows < 0 || n_cols <= 0 || nnz < 0) fail("invalid CSR matrix %lld x %d with %lld entries", (long long)n_rows, n_cols, (long long)nnz);
  std::unique_ptr<Matrix> m = new_matrix(n_rows, n_cols, missing);
  m->ctx = get_ctx(device); m->csr = true; m->nnz = nnz;
  upload_csr(m.get(), indptr, indices, values);
  *out = register_matrix(std::move(m));
  API_END
}
int B2_MatrixCreate(int64_t n_rows, int32_t n_cols, float missing, int device, B2Handle* out) {
  API_BEGIN
  std::unique_ptr<Matrix> m = new_matrix(n_rows, n_cols, missing);
  m->ctx = get_ctx(device);
  m->raw.ensure((size_t)std::max<int64_t>(n_rows * n_cols, 1));   // filled by B2_MatrixSetRows
  m->has_raw = true;
  *out = register_matrix(std::move(m));
  API_END
}
int B2_MatrixCreateFromProcess(int64_t pid, uint64_t remote_addr, int64_t remote_row_stride_bytes, int64_t n_rows, int32_t n_cols,
                               float missing, int device, B2Handle* out) {
  API_BEGIN
  std::unique_ptr<Matrix> m = new_matrix(n_rows, n_cols, missing);
  if (pid <= 0 || remote_row_stride_bytes < (int64_t)n_cols * 4) fail("invalid remote source (pid %lld, row stride %lld)", (long long)pid, (long long)remote_row_stride_bytes);
  m->ctx = get_ctx(device);
  UploadSource u; u.pid = pid; u.remote_addr = remote_addr; u.row_bytes = (size_t)n_cols * 4; u.row_stride = (size_t)remote_row_stride_bytes;
  upload_raw(m.get(), u);
  *out = register_matrix(std::move(m));
  API_END
}
int B2_MatrixCreateFromProcessInterleaved(int64_t pid, uint64_t remote_addr, int64_t n_total_rows, int32_t n_cols, int32_t shard_rank,
                                          B2Handle commh, float missing, int device, B2Handle* out) {
  API_BEGIN
  if (n_total_rows < 0 || n_cols <= 0 || pid <= 0) fail("invalid remote matrix (%lld x %d, pid %lld)", (long long)n_total_rows, n_cols, (long long)pid);
  *out = ingest_interleaved(comm_of(commh), pid, remote_addr, n_total_rows, n_cols, shard_rank, missing, device);
  API_END
}
int B2_MatrixSetRows(B2Handle mh, int64_t row_begin, const float* data, int64_t n_rows) {
  API_BEGIN
  Matrix* m = matrix_of(mh);
  if (m->quantized || !m->has_raw) fail("rows can only be set before the matrix is quantised");
  if (m->csr) fail("rows of a matrix created from CSR arrays cannot be set");
  if (row_begin < 0 || n_rows < 0 || row_begin + n_rows > m->n) fail("row block [%lld, %lld) outside the matrix (%lld rows)",
                                                                     (long long)row_begin, (long long)(row_begin + n_rows), (long long)m->n);
  upload_pipelined(m->ctx, m->raw.p + (size_t)row_begin * m->F, data, (size_t)n_rows * m->F * sizeof(float));
  API_END
}
int B2_MatrixSetFloatInfo(B2Handle mh, const char* field, const float* values, int64_t len) {
  API_BEGIN
  Matrix* m = matrix_of(mh);
  std::string f(field ? field : "");
  DevBuf<float>* dst = nullptr; int64_t* cnt = nullptr;
  if (f == "label") {
    dst = &m->label; cnt = &m->n_label; m->rank_version++; m->n_targets = 1;
    if (len != m->n) fail("label length %lld != rows %lld", (long long)len, (long long)m->n);
  }
  else if (f == "weight") { dst = &m->weight; cnt = &m->n_weight; if (len != m->n && len != 0) fail("weight length %lld != rows %lld", (long long)len, (long long)m->n); }
  else if (f == "label_lower_bound" || f == "label_upper_bound") {
    const bool lo = f == "label_lower_bound";
    dst = lo ? &m->lower : &m->upper; cnt = lo ? &m->n_lower : &m->n_upper;
    if (len != m->n && len != 0) fail("%s length %lld != rows %lld", f.c_str(), (long long)len, (long long)m->n);
    if (len != 0 && m->n_targets > 1) fail("%s: the matrix has a label of %d columns (survival bounds need one)", f.c_str(), m->n_targets);
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
    set_field(m, m->d_fwq, m->fwq.data(), len);
    return 0;
  }
  else fail("unknown float info field '%s'", f.c_str());
  set_field(m, *dst, values, len);
  *cnt = len;
  API_END
}
int B2_MatrixSetLabel(B2Handle mh, const float* values, int64_t rows, int32_t n_targets) {
  API_BEGIN
  Matrix* m = matrix_of(mh);
  if (rows != m->n) fail("label has %lld rows, the matrix %lld", (long long)rows, (long long)m->n);
  if (n_targets < 1 || n_targets > kMaxTargets) fail("label columns must be in [1, %d], got %d", kMaxTargets, n_targets);
  if (n_targets > 1 && m->has_qgroups())
    fail("a label of %d columns on a matrix with query groups (qid) is not supported", n_targets);
  if (n_targets > 1 && (m->n_lower > 0 || m->n_upper > 0))
    fail("a label of %d columns on a matrix with label_lower_bound / label_upper_bound is not supported", n_targets);
  const int64_t len = rows * n_targets;
  set_field(m, m->label, values, len);
  m->n_label = len; m->n_targets = n_targets;
  m->rank_version++;
  API_END
}
int B2_MatrixSetGroups(B2Handle mh, const int32_t* group_sizes, int64_t n_groups) {
  API_BEGIN
  Matrix* m = matrix_of(mh);
  if (n_groups < 0) fail("query groups: negative group count %lld", (long long)n_groups);
  if (n_groups > 0 && m->n_targets > 1)
    fail("query groups (qid) on a matrix with a label of %d columns are not supported", m->n_targets);
  std::vector<int64_t> ptr((size_t)n_groups + 1, 0);
  int64_t mx = 0;
  for (int64_t g = 0; g < n_groups; ++g) {
    if (group_sizes[g] < 1) fail("query group %lld has %d rows: every group needs at least one", (long long)g, group_sizes[g]);
    ptr[g + 1] = ptr[g] + group_sizes[g];
    mx = std::max<int64_t>(mx, group_sizes[g]);
  }
  if (n_groups > 0 && ptr[n_groups] != m->n)
    fail("query groups cover %lld rows, the matrix has %lld", (long long)ptr[n_groups], (long long)m->n);
  set_field(m, m->qgroup_ptr, ptr.data(), (int64_t)ptr.size());
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
  Matrix* m = matrix_of(mh);
  Comm* comm = comm_of(commh);
  if (!m->has_raw) fail("matrix has no raw data on the device (already quantised without keep_raw?)");
  if (refh) {
    Matrix* r = from_handle<Matrix>(refh, kMatrix, "matrix");
    if (!r->quantized) fail("reference matrix is not quantised");
    if (r->F != m->F) fail("reference matrix has %d features, this one %d", r->F, m->F);
    m->cut_ptrs = r->cut_ptrs; m->cut_vals = r->cut_vals; m->min_vals = r->min_vals; m->has_missing = r->has_missing; m->max_bin = r->max_bin;
    m->is_cat = r->is_cat; m->cat_feats = r->cat_feats;
  }
  quantize_matrix(m, comm, max_bin, refh != 0, keep_raw != 0);
  API_END
}
int B2_MatrixQuantizeWithCuts(B2Handle mh, B2Handle commh, const int32_t* ptrs, const float* vals, const float* mins,
                              const uint8_t* has_missing, int32_t max_bin, int32_t keep_raw) {
  API_BEGIN
  Matrix* m = matrix_of(mh);
  Comm* comm = comm_of(commh);
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
  quantize_matrix(m, comm, max_bin, true, keep_raw != 0);
  API_END
}
int B2_MatrixEnsureRaw(B2Handle mh, const float* data) {
  API_BEGIN
  Matrix* m = matrix_of(mh);
  if (m->has_raw) return 0;
  if (m->csr) fail("the matrix was created from CSR arrays: re-upload them with B2_MatrixEnsureRawCSR");
  upload_raw(m, UploadSource{data});
  API_END
}
int B2_MatrixEnsureRawCSR(B2Handle mh, int64_t* indptr, const int32_t* indices, const float* values) {
  API_BEGIN
  Matrix* m = matrix_of(mh);
  if (m->has_raw) return 0;
  if (!m->csr) fail("the matrix was created from dense rows: re-upload them with B2_MatrixEnsureRaw");
  upload_csr(m, indptr, indices, values);
  API_END
}
int B2_MatrixSlice(B2Handle mh, int64_t* rows, int64_t n_rows, B2Handle* out) {
  API_BEGIN
  *out = slice_matrix(matrix_of(mh), rows, n_rows);
  API_END
}
int B2_MatrixDeviceBytes(B2Handle mh, int64_t* out) {
  API_BEGIN
  *out = (int64_t)matrix_device_bytes(from_handle<Matrix>(mh, kMatrix, "matrix"));
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
int B2_MatrixSetBinLayout(B2Handle mh, int32_t layout) {
  API_BEGIN
  Matrix* m = matrix_of(mh);
  if (layout != B2_BIN_LAYOUT_AUTO && layout != B2_BIN_LAYOUT_DENSE && layout != B2_BIN_LAYOUT_CSR)
    fail("unknown bin layout %d (0 auto, 1 dense, 2 csr)", layout);
  if (m->quantized) fail("the bin layout must be set before the matrix is quantised");
  if (layout == B2_BIN_LAYOUT_CSR && !m->csr)
    fail("the CSR bin layout needs a matrix created from CSR arrays (a scipy.sparse matrix); this one holds dense rows");
  m->bin_layout = layout;
  API_END
}
int B2_MatrixGetBins(B2Handle mh, uint8_t* out) {
  API_BEGIN
  bins_to_host(matrix_of(mh), out);
  API_END
}
int B2_MatrixFree(B2Handle mh) {
  API_BEGIN
  Matrix* m = from_handle<Matrix>(mh, kMatrix, "matrix");
  cudaSetDevice(m->ctx->device);
  free_matrix(m);
  API_END
}

int B2_BoosterCreate(const char* params, B2Handle trainh, B2Handle commh, B2Handle* out) {
  API_BEGIN
  Matrix* m = trainh ? from_handle<Matrix>(trainh, kMatrix, "matrix") : nullptr;
  if (m && !m->quantized) fail("train matrix must be quantised (B2_MatrixQuantize) before B2_BoosterCreate");
  *out = (B2Handle)new_booster(params, m, comm_of(commh));
  API_END
}
int B2_BoosterSetParam(B2Handle bh, const char* params) {
  API_BEGIN
  set_booster_params(from_handle<Booster>(bh, kBooster, "booster"), params);
  API_END
}
int B2_BoosterUpdateOneIter(B2Handle bh, int32_t iter) {
  API_BEGIN
  (void)iter;
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  if (b->p.update_mode) fail("this booster has process_type=update: its rounds run through B2_BoosterRefreshOneIter");
  boost_round(b, nullptr, nullptr, 0);
  API_END
}
int B2_BoosterBoostOneIter(B2Handle bh, const float* grad, const float* hess, int64_t len) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  if (b->p.update_mode) fail("this booster has process_type=update: its rounds run through B2_BoosterRefreshOneIter");
  drain_round(b);
  if (!grad || !hess) fail("grad/hess must not be NULL");
  boost_round(b, grad, hess, len);
  API_END
}
int B2_BoosterRefreshOneIter(B2Handle bh, const float* grad, const float* hess, int64_t len) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  if (!b->p.update_mode) fail("B2_BoosterRefreshOneIter needs a booster created with process_type=update");
  if ((grad == nullptr) != (hess == nullptr)) fail("grad and hess must both be given or both be NULL");
  if (grad) drain_round(b);   // the caller computed them from the margin of every round so far
  boost_round(b, grad, hess, len);
  API_END
}
int B2_BoosterGetGradients(B2Handle bh, float* grad, float* hess, int64_t len) {
  API_BEGIN
  Booster* b = drained(bh);
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
  return with_matrix(bh, mh, [&](Booster* b, Matrix* m) { *out = eval_metric(b, m, metric); });
}
int B2_BoosterPredict(B2Handle bh, B2Handle mh, int32_t output_margin, int32_t tree_begin, int32_t tree_end, float* out,
                      int64_t out_len) {
  return with_matrix(bh, mh, [&](Booster* b, Matrix* m) { predict(b, m, output_margin != 0, tree_begin, tree_end, out, out_len); });
}
int B2_BoosterPredictContribs(B2Handle bh, B2Handle mh, int32_t tree_begin, int32_t tree_end, int32_t interactions, float* out,
                              int64_t out_len) {
  return with_matrix(bh, mh, [&](Booster* b, Matrix* m) {
    predict_contribs(b, m, tree_begin, tree_end, interactions != 0, out, out_len);
  });
}
int B2_BoosterPredictLeaf(B2Handle bh, B2Handle mh, int32_t tree_begin, int32_t tree_end, float* out, int64_t out_len) {
  return with_matrix(bh, mh, [&](Booster* b, Matrix* m) { predict_leaf(b, m, tree_begin, tree_end, out, out_len); });
}
int B2_BoosterGetTrainMargin(B2Handle bh, int32_t full, float* out, int64_t out_len) {
  API_BEGIN
  Booster* b = drained(bh);
  CUDA_CHECK(cudaSetDevice(b->ctx->device));
  if (!b->train) fail("this booster has no train matrix (prediction-only)");
  const int64_t want = b->train->n * b->p.num_class;
  if (out_len != want) fail("output buffer has %lld values, expected %lld", (long long)out_len, (long long)want);
  ensure_train_margin(b);
  // DART: the margin the next round's gradients are taken at (its drop margin); B2_BoosterBoostOneIter keeps its drops.
  // full != 0 returns the margin of the whole model instead (what predict and the metrics see)
  const float* src = b->margin.p;
  if (b->p.dart && !full) { dart_prepare(b); if (b->dart_next.n_dropped > 0) src = b->dart_drop.p; }
  if (want > 0) CUDA_CHECK(cudaMemcpyAsync(out, src, want * sizeof(float), cudaMemcpyDeviceToHost, b->ctx->stream));
  CUDA_CHECK(cudaStreamSynchronize(b->ctx->stream));
  API_END
}
int B2_BoosterResetTrainMargin(B2Handle bh) {
  API_BEGIN
  Booster* b = drained(bh);
  CUDA_CHECK(cudaSetDevice(b->ctx->device));
  if (!b->train) fail("this booster has no train matrix (prediction-only)");
  b->margin_ready = false;
  ensure_train_margin(b);
  CUDA_CHECK(cudaStreamSynchronize(b->ctx->stream));
  API_END
}
// No drain: the intercept is settled on the host before the first round is enqueued (estimate_base_score), and the
// Python booster reads it after every update() until it is final -- a drain here would stall the round pipeline.
int B2_BoosterGetBaseScore(B2Handle bh, float* out, int32_t* is_final) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  *out = b->p.base_score; *is_final = b->p.base_score_set ? 1 : 0;
  API_END
}
int B2_BoosterNumTargets(B2Handle bh, int32_t* out) {
  API_BEGIN
  *out = from_handle<Booster>(bh, kBooster, "booster")->p.num_target;
  API_END
}
int B2_BoosterNumTrees(B2Handle bh, int32_t* out) {
  API_BEGIN
  Booster* b = drained(bh);
  *out = (int32_t)b->trees.size();
  API_END
}
int B2_BoosterTreeNumNodes(B2Handle bh, int32_t tree, int32_t* out) {
  API_BEGIN
  *out = tree_at(drained(bh), tree).size();
  API_END
}
int B2_BoosterGetTree(B2Handle bh, int32_t tree, B2Tree* out) {
  API_BEGIN
  Booster* b = drained(bh);
  const TreeHost& t = tree_at(b, tree); const size_t n = t.size();
  if (out->n_nodes != t.size()) fail("tree buffers have %d nodes, tree %d has %d", out->n_nodes, tree, t.size());
  const int64_t len = out->leaf_vector ? out->leaf_vector_len : 0;
  if (len != (int64_t)t.leaf_vec.size()) fail("leaf vector buffer has %lld values, tree %d has %zu", (long long)len, tree, t.leaf_vec.size());
  memcpy(out->left, t.left.data(), n * 4); memcpy(out->right, t.right.data(), n * 4); memcpy(out->parent, t.parent.data(), n * 4);
  memcpy(out->split_feature, t.feature.data(), n * 4); memcpy(out->split_bin, t.split_bin.data(), n * 4);
  memcpy(out->split_cond, t.cond.data(), n * 4); memcpy(out->default_left, t.default_left.data(), n);
  memcpy(out->value, t.value.data(), n * 4); memcpy(out->base_weight, t.base_weight.data(), n * 4);
  memcpy(out->loss_chg, t.loss_chg.data(), n * 4); memcpy(out->sum_hess, t.sum_hess.data(), n * 8);
  memcpy(out->split_type, t.split_type.data(), n); memcpy(out->cat_bits, t.cat_bits.data(), n * 8 * sizeof(uint32_t));
  if (len > 0) memcpy(out->leaf_vector, t.leaf_vec.data(), len * sizeof(float));
  API_END
}
int B2_BoosterAddTree(B2Handle bh, const B2Tree* in) {
  API_BEGIN
  Booster* b = drained(bh);
  if (b->update_started) fail("process_type=update: trees are added before the first refresh round, not after");
  TreeHost t;
  for (int i = 0; i < in->n_nodes; ++i) {
    t.add(in->parent[i]);
    t.left[i] = in->left[i]; t.right[i] = in->right[i]; t.feature[i] = in->split_feature[i];
    t.split_bin[i] = in->split_bin ? in->split_bin[i] : -1;
    t.cond[i] = in->split_cond[i]; t.default_left[i] = in->default_left[i]; t.value[i] = in->value[i];
    t.base_weight[i] = in->base_weight ? in->base_weight[i] : 0.f; t.loss_chg[i] = in->loss_chg ? in->loss_chg[i] : 0.f;
    t.sum_hess[i] = in->sum_hess ? in->sum_hess[i] : 0.0;
    if (in->split_type && in->split_type[i]) {   // numeric nodes keep all-zero category bits
      if (!in->cat_bits) fail("tree %zu node %d has a categorical split_type and no cat_bits", b->trees.size(), i);
      t.split_type[i] = 1; t.any_cat = true;
      for (int w8 = 0; w8 < 8; ++w8) t.cat_bits[(size_t)i * 8 + w8] = in->cat_bits[(size_t)i * 8 + w8];
    }
  }
  if (in->leaf_vector && in->leaf_vector_len > 0) t.leaf_vec.assign(in->leaf_vector, in->leaf_vector + in->leaf_vector_len);
  check_tree(b, t);
  b->trees.push_back(std::move(t));
  if (b->p.dart) b->tree_w.push_back(1.0f);   // B2_BoosterSetTreeWeights sets the model's weights
  b->margin_ready = false;
  API_END
}
int B2_BoosterGetTreeWeights(B2Handle bh, float* out, int64_t len) {
  API_BEGIN
  Booster* b = drained(bh);
  if (len != (int64_t)b->trees.size()) fail("weight buffer has %lld values for %zu trees", (long long)len, b->trees.size());
  for (int64_t t = 0; t < len; ++t) out[t] = b->p.dart ? b->tree_w[t] : 1.0f;
  API_END
}
int B2_BoosterSetTreeWeights(B2Handle bh, const float* w, int64_t len) {
  API_BEGIN
  Booster* b = drained(bh);
  if (!b->p.dart) fail("tree weights belong to booster=dart; this booster is gbtree");
  if (len != (int64_t)b->trees.size()) fail("%lld tree weights for %zu trees", (long long)len, b->trees.size());
  float S = 0.0f;   // the binary32 sum sample_type=weighted divides by (dart_drop_set)
  for (int64_t t = 0; t < len; ++t) {
    if (!std::isfinite(w[t]) || w[t] < 0.0f) fail("tree weight %lld is %g: weights must be finite and >= 0", (long long)t, (double)w[t]);
    S += w[t];
  }
  if (len > 0 && !(S > 0.0f && std::isfinite(S)))
    fail("tree weights sum to %g: a DART model needs a finite, positive total weight", (double)S);
  b->tree_w.assign(w, w + len);
  b->weights_version++;
  b->margin_ready = false;
  API_END
}
int B2_BoosterGetTimers(B2Handle bh, int32_t reset, char* out, int64_t out_cap) {
  API_BEGIN
  Booster* b = drained(bh);
  const Timers& t = b->t;
  snprintf(out, (size_t)out_cap,
           "{\"hist_ms\": %.6f, \"hist_launches\": %lld, \"hist_rows\": %lld, \"hist_bytes\": %.1f, \"kernel_launches\": %lld, "
           "\"round_ms\": %.6f, \"rounds\": %lld, \"allreduce_bytes\": %.1f, \"num_sms\": %d, \"n_groups\": %d, \"row_stride\": %d, "
           "\"phase_ms\": {\"quant\": %.4f, \"hist\": %.4f, \"allreduce\": %.4f, \"subtract\": %.4f, \"eval_decide\": %.4f, "
           "\"partition_finalize\": %.4f, \"leaf\": %.4f}, \"shap_ms\": %.6f, \"shap_rows\": %lld, \"refresh_ms\": %.6f, "
           "\"refresh_launches\": %lld, \"graph_update_ms\": %.6f, \"graph_updates\": %lld, \"graph_reinstantiations\": %lld}",
           t.hist_ms, t.hist_launches, t.hist_rows, t.hist_bytes, t.kernel_launches, t.round_ms, t.rounds, t.allreduce_bytes,
           b->ctx->num_sms, b->train ? b->train->n_groups : 0, b->train ? b->train->row_stride : 0, t.phase_ms[0], t.phase_ms[1],
           t.phase_ms[2], t.phase_ms[3], t.phase_ms[4], t.phase_ms[5], t.phase_ms[6], t.shap_ms, t.shap_rows, t.refresh_ms,
           t.refresh_launches, t.graph_update_ms, t.graph_updates, t.graph_reinstantiations);
  if (reset) b->t.reset();
  API_END
}
// No drain: this only raises a flag and may be called from another thread while update() runs; the next update()
// drains the pending round and then fails.
int B2_BoosterCancel(B2Handle bh) {
  API_BEGIN
  Booster* b = from_handle<Booster>(bh, kBooster, "booster");
  b->cancel.store(true);
  API_END
}
// A pending round is not drained (its trees are dropped with the booster); the destructor waits for it on the stream
// before it frees the read-back blocks.
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
  Matrix m; m.kind = kMatrix; m.ctx = get_ctx(device); m.n = n_rows; m.F = n_cols;
  upload_bins(&m, bins);
  hist_build_raw(&m, qg, qh, ridx, n_sel, window_rows, chunk_rows, out, kernel_ms);
  API_END
}

int B2_HistBuildRawCSR(int64_t* indptr, const int32_t* indices, const uint8_t* bins, int64_t n_rows, int32_t n_cols,
                       const int32_t* qg, const int32_t* qh, const int32_t* ridx, int64_t n_sel, int32_t chunk_rows,
                       int device, int64_t* out, float* kernel_ms) {
  API_BEGIN
  Matrix m; m.kind = kMatrix; m.ctx = get_ctx(device); m.n = n_rows; m.F = n_cols;
  m.csr = true; m.nnz = n_rows > 0 ? indptr[n_rows] : 0;
  const std::vector<float> values((size_t)std::max<int64_t>(m.nnz, 1), 0.0f);   // upload_csr checks indptr and indices
  upload_csr(&m, indptr, indices, values.data());
  upload_bins(&m, bins);
  hist_build_raw(&m, qg, qh, ridx, n_sel, INT_MAX, chunk_rows, out, kernel_ms);   // the CSR build has no int32 window
  API_END
}

int B2_QuantizeRaw(const float* g, const float* h, int64_t n, int32_t qbits, int device, int32_t* out_q,
                   int32_t* out_exp) {
  API_BEGIN
  if (n < 1) fail("B2_QuantizeRaw needs at least one row");
  if (qbits < 8 || qbits > 24) fail("hist_qbits must be in [8, 24], got %d", qbits);
  Ctx* ctx = get_ctx(device); cudaStream_t s = ctx->stream;
  std::vector<float2> gh((size_t)n);
  for (int64_t i = 0; i < n; ++i) gh[i] = make_float2(g[i], h[i]);
  DevBuf<float2> d_gh; DevBuf<uint32_t> d_absmax; DevBuf<int32_t> d_qexp; DevBuf<int2> d_q;
  d_gh.ensure((size_t)n); d_absmax.ensure(2); d_qexp.ensure(2); d_q.ensure((size_t)n);
  CUDA_CHECK(cudaMemcpyAsync(d_gh.p, gh.data(), gh.size() * sizeof(float2), cudaMemcpyHostToDevice, s));
  CUDA_CHECK(cudaMemsetAsync(d_absmax.p, 0, 2 * sizeof(uint32_t), s));
  LAUNCH_CHECK(b2_launch_absmax(d_gh.p, n, d_absmax.p, ctx->num_sms, s));
  LAUNCH_CHECK(b2_launch_quant_exponent(d_absmax.p, d_qexp.p, s));
  LAUNCH_CHECK(b2_launch_quantize(d_gh.p, n, d_qexp.p, qbits, d_q.p, ctx->num_sms, s));
  CUDA_CHECK(cudaMemcpyAsync(out_q, d_q.p, (size_t)n * sizeof(int2), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaMemcpyAsync(out_exp, d_qexp.p, 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  API_END
}

}  // extern "C"
