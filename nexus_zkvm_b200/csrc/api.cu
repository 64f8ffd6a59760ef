// C ABI of libnexus_b200.so (see include/nb200.h).  No CPU fallback anywhere: without a CUDA device
// nb200_ctx_create fails with NB200_ERR_NO_DEVICE.
#include "common.cuh"
#include "circle_host.h"
#include "blake2s.cuh"
#include <cstdlib>
#include <cstring>

#include <chrono>
namespace nb {
void trace_mark(nb200_ctx* ctx, const char* stage) {
  if (!ctx || !ctx->trace) return;
  cudaStreamSynchronize(ctx->stream);
  double now = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
  if (stage) fprintf(stderr, "[nb200] %-28s %9.3f ms\n", stage, now - ctx->trace_t0);
  ctx->trace_t0 = now;
}
void fft_drop_tables(nb200_ctx* ctx);
std::string& global_err() { static std::string e; return e; }
nb200_status merkle_decommit(nb200_ctx* ctx, const nb200_tree* tree, const std::vector<ColRef>& cols_in,
                             const std::vector<std::pair<u32, std::vector<u64>>>& queries,
                             std::vector<u32>& queried_values, std::vector<uint8_t>& hash_witness, std::vector<u32>& column_witness);
nb200_status eval_at_points(nb200_ctx* ctx, const u32* coeffs, size_t n_cols, u32 log_size, const u32* points_xy, size_t n_points, u32* out_qm31);
}  // namespace nb
using namespace nb;

extern "C" {

nb200_status nb200_ctx_create(int device, nb200_ctx** out) {
  if (!out) return NB200_ERR_ARG;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    global_err() = std::string("no CUDA device (") + (e != cudaSuccess ? cudaGetErrorString(e) : "count=0") +
                   "); libnexus_b200 has no CPU fallback";
    return NB200_ERR_NO_DEVICE;
  }
  if (device < 0 || device >= count) { global_err() = "device index out of range"; return NB200_ERR_ARG; }
  e = cudaSetDevice(device);
  if (e != cudaSuccess) { global_err() = cudaGetErrorString(e); return NB200_ERR_CUDA; }
  nb200_ctx* ctx = new nb200_ctx();
  ctx->device = device;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) { ctx->sm_count = prop.multiProcessorCount; ctx->total_mem = prop.totalGlobalMem; }
  e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { global_err() = cudaGetErrorString(e); delete ctx; return NB200_ERR_CUDA; }
  ctx->own_stream = true;
  { const char* t = getenv("NB200_TRACE"); ctx->trace = (t && t[0] && t[0] != '0') ? 1 : 0; }
  {
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
      uint64_t thr = UINT64_MAX;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
  }
  *out = ctx;
  return NB200_OK;
}

void nb200_ctx_destroy(nb200_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  comm_release(ctx);
  fft_drop_tables(ctx);
  if (ctx->tw.d_tw) cudaFree(ctx->tw.d_tw);
  if (ctx->tw.d_itw) cudaFree(ctx->tw.d_itw);
  if (ctx->tw.d_tw2) cudaFree(ctx->tw.d_tw2);
  if (ctx->tw.d_itw2) cudaFree(ctx->tw.d_itw2);
  if (ctx->tw.d_ptw2) cudaFree(ctx->tw.d_ptw2);
  if (ctx->tw.d_iptw2) cudaFree(ctx->tw.d_iptw2);
  if (ctx->h_pinned) cudaFreeHost(ctx->h_pinned);
  if (ctx->copy_stream) {
    cudaStreamDestroy(ctx->copy_stream);
    for (int i = 0; i < 2; ++i) { cudaEventDestroy(ctx->copy_ev[i]); cudaEventDestroy(ctx->done_ev[i]); }
  }
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

const char* nb200_last_error(nb200_ctx* ctx) { return ctx ? ctx->err.c_str() : global_err().c_str(); }

nb200_status nb200_ctx_set_stream(nb200_ctx* ctx, void* s) {
  if (!ctx) return NB200_ERR_ARG;
  if (ctx->own_stream && ctx->stream) { cudaStreamSynchronize(ctx->stream); cudaStreamDestroy(ctx->stream); }
  ctx->stream = (cudaStream_t)s;
  ctx->own_stream = false;
  return NB200_OK;
}

nb200_status nb200_sync(nb200_ctx* ctx) {
  if (!ctx) return NB200_ERR_ARG;
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return NB200_OK;
}

nb200_status nb200_set_flavor(nb200_ctx* ctx, int merkle_hash, int draw_domain_sep, int pow_variant) {
  if (!ctx) return NB200_ERR_ARG;
  NB_ARG(ctx, (merkle_hash == 0 || merkle_hash == 1) && (draw_domain_sep == 0 || draw_domain_sep == 1), "bad flavor");
  NB_ARG(ctx, pow_variant == 0, "pow_variant: only 0 (trailing zero bits of Blake2s(digest || nonce)) is implemented");
  ctx->merkle_hash = merkle_hash; ctx->draw_domain_sep = draw_domain_sep; ctx->pow_variant = pow_variant;
  return NB200_OK;
}

uint64_t nb200_launch_count(nb200_ctx* ctx) { return ctx ? ctx->launches : 0; }

// ---- columns ----
nb200_status nb200_cols_alloc(nb200_ctx* ctx, size_t n_cols, uint32_t log_size, nb200_cols** out) {
  if (!ctx || !out) return NB200_ERR_ARG;
  NB_ARG(ctx, log_size <= 30, "cols_alloc: log_size too large");
  nb200_cols* c = new nb200_cols();
  c->ctx = ctx; c->n_cols = n_cols; c->log_size = log_size;
  size_t bytes = (n_cols << log_size) * 4;
  if (bytes) {
    cudaError_t e = dmalloc(ctx, (void**)&c->d, bytes);
    if (e != cudaSuccess) { cudaGetLastError(); delete c; return set_err(ctx, NB200_ERR_OOM, std::string("cols_alloc: ") + cudaGetErrorString(e)); }
    ctx->live_bytes += bytes;
  }
  *out = c;
  return NB200_OK;
}
nb200_status nb200_cols_from_device(nb200_ctx* ctx, void* device_ptr, size_t n_cols, uint32_t log_size, nb200_cols** out) {
  if (!ctx || !out) return NB200_ERR_ARG;
  NB_ARG(ctx, device_ptr != nullptr && log_size <= 30, "cols_from_device: bad arguments");
  nb200_cols* c = new nb200_cols();
  c->ctx = ctx; c->n_cols = n_cols; c->log_size = log_size; c->d = (uint32_t*)device_ptr; c->owns = false;
  *out = c;
  return NB200_OK;
}
void nb200_cols_free(nb200_ctx*, nb200_cols* c) {
  if (!c) return;
  if (c->owns && c->d) {
    dfree(c->ctx, c->d);
    const size_t bytes = (c->n_cols << c->log_size) * 4;
    c->ctx->live_bytes = c->ctx->live_bytes >= bytes ? c->ctx->live_bytes - bytes : 0;
  }
  delete c;
}
size_t nb200_cols_count(const nb200_cols* c) { return c ? c->n_cols : 0; }
uint32_t nb200_cols_log_size(const nb200_cols* c) { return c ? c->log_size : 0; }
void* nb200_cols_device_ptr(const nb200_cols* c) { return c ? c->d : nullptr; }

nb200_status nb200_cols_upload(nb200_ctx* ctx, nb200_cols* c, size_t first, size_t n, const uint32_t* host, int coset_order) {
  if (!ctx || !c) return NB200_ERR_ARG;
  NB_ARG(ctx, first + n <= c->n_cols, "cols_upload: range");
  if (n == 0) return NB200_OK;
  size_t bytes = (n << c->log_size) * 4;
  if (!coset_order) {
    NB_CUDA(ctx, cudaMemcpyAsync(c->col(first), host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return NB200_OK;
  }
  u32* tmp = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&tmp, bytes));
  cudaError_t e = cudaMemcpyAsync(tmp, host, bytes, cudaMemcpyHostToDevice, ctx->stream);
  nb200_status st = NB200_OK;
  if (e != cudaSuccess) st = set_err(ctx, NB200_ERR_CUDA, cudaGetErrorString(e));
  if (st == NB200_OK) st = reorder_coset_to_bitrev(ctx, tmp, c->col(first), n, c->log_size);
  cudaStreamSynchronize(ctx->stream);
  dfree(ctx, tmp);
  return st;
}
nb200_status nb200_cols_download(nb200_ctx* ctx, const nb200_cols* c, size_t first, size_t n, uint32_t* host) {
  if (!ctx || !c) return NB200_ERR_ARG;
  NB_ARG(ctx, first + n <= c->n_cols, "cols_download: range");
  if (n == 0) return NB200_OK;
  NB_CUDA(ctx, cudaMemcpyAsync(host, c->col(first), (n << c->log_size) * 4, cudaMemcpyDeviceToHost, ctx->stream));
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return NB200_OK;
}
nb200_status nb200_cols_finalize_order(nb200_ctx* ctx, nb200_cols* c) {
  if (!ctx || !c) return NB200_ERR_ARG;
  size_t bytes = (c->n_cols << c->log_size) * 4;
  if (!bytes) return NB200_OK;
  u32* tmp = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&tmp, bytes));
  cudaError_t e = cudaMemcpyAsync(tmp, c->d, bytes, cudaMemcpyDeviceToDevice, ctx->stream);
  nb200_status st = e == cudaSuccess ? reorder_coset_to_bitrev(ctx, tmp, c->d, c->n_cols, c->log_size) : set_err(ctx, NB200_ERR_CUDA, cudaGetErrorString(e));
  cudaStreamSynchronize(ctx->stream);
  dfree(ctx, tmp);
  return st;
}

// ---- PolyOps ----
nb200_status nb200_twiddles_prepare(nb200_ctx* ctx, uint32_t max_domain_log) {
  if (!ctx) return NB200_ERR_ARG;
  return twiddles_prepare(ctx, max_domain_log);
}
uint32_t nb200_twiddles_domain_log(nb200_ctx* ctx) { return (ctx && ctx->tw.d_tw) ? ctx->tw.half_log + 1 : 0; }
nb200_status nb200_twiddles_download(nb200_ctx* ctx, uint32_t* tw, uint32_t* itw) {
  if (!ctx) return NB200_ERR_ARG;
  NB_ARG(ctx, ctx->tw.d_tw, "twiddles not prepared");
  size_t bytes = ((size_t)4) << ctx->tw.half_log;
  NB_CUDA(ctx, cudaMemcpyAsync(tw, ctx->tw.d_tw, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  NB_CUDA(ctx, cudaMemcpyAsync(itw, ctx->tw.d_itw, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return NB200_OK;
}
nb200_status nb200_interpolate(nb200_ctx* ctx, nb200_cols* c) {
  if (!ctx || !c) return NB200_ERR_ARG;
  if (c->log_size >= 1) NB_TRY(twiddles_prepare(ctx, c->log_size));
  return fft_interpolate(ctx, c->d, c->d, c->n_cols, c->log_size);
}
nb200_status nb200_evaluate(nb200_ctx* ctx, const nb200_cols* coeffs, uint32_t log_blowup, nb200_cols* out) {
  if (!ctx || !coeffs || !out) return NB200_ERR_ARG;
  NB_ARG(ctx, out->n_cols == coeffs->n_cols && out->log_size == coeffs->log_size + log_blowup, "evaluate: output batch shape");
  if (out->log_size >= 1) NB_TRY(twiddles_prepare(ctx, out->log_size));
  return fft_evaluate(ctx, coeffs->d, coeffs->log_size, out->d, out->log_size, coeffs->n_cols);
}
nb200_status nb200_eval_at_points(nb200_ctx* ctx, const nb200_cols* coeffs, const uint32_t* points_xy, size_t n_points, uint32_t* out_qm31) {
  if (!ctx || !coeffs) return NB200_ERR_ARG;
  return eval_at_points(ctx, coeffs->d, coeffs->n_cols, coeffs->log_size, points_xy, n_points, out_qm31);
}

// ---- MerkleOps ----
static void collect_cols(const nb200_cols* const* batches, size_t n_batches, std::vector<ColRef>& cols) {
  for (size_t b = 0; b < n_batches; ++b)
    for (size_t c = 0; c < batches[b]->n_cols; ++c) cols.push_back(ColRef{batches[b]->col(c), batches[b]->log_size});
}
nb200_status nb200_merkle_commit(nb200_ctx* ctx, const nb200_cols* const* batches, size_t n_batches, nb200_tree** out, uint8_t root[32]) {
  if (!ctx || !out) return NB200_ERR_ARG;
  std::vector<ColRef> cols;
  collect_cols(batches, n_batches, cols);
  NB_TRY(merkle_commit(ctx, cols, out));
  if (root) memcpy(root, (*out)->root, 32);
  return NB200_OK;
}
void nb200_tree_free(nb200_ctx*, nb200_tree* t) {
  if (!t) return;
  if (t->d_pool) dfree(t->ctx, t->d_pool);
  delete t;
}
uint32_t nb200_tree_log_size(const nb200_tree* t) { return t ? t->max_log : 0; }
nb200_status nb200_tree_layer_download(nb200_ctx* ctx, const nb200_tree* t, uint32_t layer_log, uint8_t* out) {
  if (!ctx || !t) return NB200_ERR_ARG;
  NB_ARG(ctx, layer_log <= t->max_log, "tree layer out of range");
  NB_CUDA(ctx, cudaMemcpyAsync(out, t->layer[layer_log], (size_t)32 << layer_log, cudaMemcpyDeviceToHost, ctx->stream));
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return NB200_OK;
}
static void* dup_bytes(const void* p, size_t n) { void* r = malloc(n ? n : 1); if (n) memcpy(r, p, n); return r; }
nb200_status nb200_merkle_decommit(nb200_ctx* ctx, const nb200_tree* tree, const nb200_cols* const* batches, size_t n_batches,
                                   const uint32_t* q_log_sizes, const uint64_t* q_counts, const uint64_t* q_positions, size_t n_sizes,
                                   uint32_t** queried_values, size_t* n_queried, uint8_t** hash_witness, size_t* n_hashes,
                                   uint32_t** column_witness, size_t* n_column_witness) {
  if (!ctx || !tree) return NB200_ERR_ARG;
  std::vector<ColRef> cols;
  collect_cols(batches, n_batches, cols);
  std::vector<std::pair<u32, std::vector<u64>>> queries;
  size_t off = 0;
  for (size_t k = 0; k < n_sizes; ++k) {
    queries.push_back({q_log_sizes[k], std::vector<u64>(q_positions + off, q_positions + off + q_counts[k])});
    off += q_counts[k];
  }
  std::vector<u32> qv, cw; std::vector<uint8_t> hw;
  NB_TRY(merkle_decommit(ctx, tree, cols, queries, qv, hw, cw));
  *queried_values = (uint32_t*)dup_bytes(qv.data(), qv.size() * 4); *n_queried = qv.size();
  *hash_witness = (uint8_t*)dup_bytes(hw.data(), hw.size()); *n_hashes = hw.size() / 32;
  *column_witness = (uint32_t*)dup_bytes(cw.data(), cw.size() * 4); *n_column_witness = cw.size();
  return NB200_OK;
}
void nb200_free(void* p) { free(p); }

// Blake2sMerkleHasher::hash_node on the host (cap combination of row-sharded trees, verifier-side use in a shim)
nb200_status nb200_hash_node(int merkle_hash, const uint8_t* left, const uint8_t* right, const uint32_t* values, size_t n_values, uint8_t out[32]) {
  if ((left == nullptr) != (right == nullptr) || !out || (n_values && !values)) return NB200_ERR_ARG;
  if (merkle_hash == 0) {
    u32 h[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    u32 m[16];
    if (left) {
      for (int i = 0; i < 8; ++i) {
        m[i] = (u32)left[4 * i] | ((u32)left[4 * i + 1] << 8) | ((u32)left[4 * i + 2] << 16) | ((u32)left[4 * i + 3] << 24);
        m[8 + i] = (u32)right[4 * i] | ((u32)right[4 * i + 1] << 8) | ((u32)right[4 * i + 2] << 16) | ((u32)right[4 * i + 3] << 24);
      }
      b2s_compress(h, m, 0, 0, 0, 0);
    }
    for (size_t i = 0; i < n_values; i += 16) {
      for (size_t j = 0; j < 16; ++j) m[j] = i + j < n_values ? values[i + j] : 0u;
      b2s_compress(h, m, 0, 0, 0, 0);
    }
    for (int i = 0; i < 8; ++i) { out[4 * i] = h[i] & 0xff; out[4 * i + 1] = (h[i] >> 8) & 0xff; out[4 * i + 2] = (h[i] >> 16) & 0xff; out[4 * i + 3] = (h[i] >> 24) & 0xff; }
    return NB200_OK;
  }
  if (merkle_hash != 1) return NB200_ERR_ARG;
  Blake2sHost b;
  if (left) { b.update(left, 32); b.update(right, 32); }
  for (size_t i = 0; i < n_values; ++i) { uint8_t le[4] = {(uint8_t)values[i], (uint8_t)(values[i] >> 8), (uint8_t)(values[i] >> 16), (uint8_t)(values[i] >> 24)}; b.update(le, 4); }
  b.finalize(out);
  return NB200_OK;
}

}  // extern "C" (reopened below)

namespace nb {
// index of the batch whose columns alone form the leaf layer of the tree (the only batch of the maximal size), or -1
long leaf_sink_batch(const size_t* n_cols, const u32* log_sizes, size_t n_batches) {
  u32 mx = 0; long idx = -1; size_t count = 0;
  for (size_t b = 0; b < n_batches; ++b) if (n_cols[b] && log_sizes[b] > mx) mx = log_sizes[b];
  for (size_t b = 0; b < n_batches; ++b) if (n_cols[b] && log_sizes[b] == mx) { idx = (long)b; ++count; }
  return count == 1 ? idx : -1;
}

nb200_status upload_transform_pipelined(nb200_ctx* ctx, const void* host_v, size_t n_cols, u32 log_size, int coset_order, u32 log_blowup,
                                        u32* d_evals, u32* d_coeffs, u32* d_lde, u32* d_half_ext, LeafSink* leaf, u32 elem_bytes) {
  if (n_cols == 0) return NB200_OK;
  const uint8_t* host = (const uint8_t*)host_v;
  const bool staged = coset_order || elem_bytes != 4;   // the chunk lands in a staging buffer and a kernel writes d_evals
  if (!ctx->copy_stream) {
    NB_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
      NB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->copy_ev[i], cudaEventDisableTiming));
      NB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->done_ev[i], cudaEventDisableTiming));
    }
  }
  const size_t len = (size_t)1 << log_size, lde_len = len << log_blowup;
  // ~256 MiB chunks, multiples of 4 columns (the FFT kernels batch 4 columns per CTA)
  size_t chunk = std::max<size_t>(4, ((size_t)64 << 20) / len);
  chunk = (chunk + 3) & ~(size_t)3;
  if (leaf && leaf->tree) chunk = (chunk + 15) & ~(size_t)15;   // whole 16-column Blake2s message blocks per chunk
  if (chunk > n_cols) chunk = n_cols;
  u32* tmp[2] = {nullptr, nullptr};
  if (staged) for (int i = 0; i < 2; ++i) {
    cudaError_t e = dmalloc(ctx, (void**)&tmp[i], chunk * len * elem_bytes);
    if (e != cudaSuccess) { cudaGetLastError(); dfree(ctx, tmp[0]); return set_err(ctx, NB200_ERR_OOM, "pipelined upload: staging buffers"); }
  }
  auto done = [&](nb200_status st) { if (staged) { dfree(ctx, tmp[0]); dfree(ctx, tmp[1]); } return st; };
#define NB_CUDAP(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) return done(set_err(ctx, NB200_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e))); } while (0)
  // the copy stream must not overtake work already queued on the compute stream that still reads the targets
  NB_CUDAP(cudaEventRecord(ctx->done_ev[0], ctx->stream));
  NB_CUDAP(cudaStreamWaitEvent(ctx->copy_stream, ctx->done_ev[0], 0));
  nb200_status st = NB200_OK;
  size_t k = 0;
  for (size_t c0 = 0; c0 < n_cols && st == NB200_OK; c0 += chunk, ++k) {
    const size_t nc = std::min(chunk, n_cols - c0);
    const int slot = (int)(k & 1);
    void* dst = staged ? (void*)tmp[slot] : (void*)(d_evals + c0 * len);
    if (staged && k >= 2) NB_CUDAP(cudaStreamWaitEvent(ctx->copy_stream, ctx->done_ev[slot], 0));  // tmp[slot] consumed?
    NB_CUDAP(cudaMemcpyAsync(dst, host + c0 * len * elem_bytes, nc * len * elem_bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
    NB_CUDAP(cudaEventRecord(ctx->copy_ev[slot], ctx->copy_stream));
    NB_CUDAP(cudaStreamWaitEvent(ctx->stream, ctx->copy_ev[slot], 0));
    if (staged) {
      st = expand_reorder(ctx, tmp[slot], elem_bytes, d_evals + c0 * len, nc, log_size, coset_order);
      if (st == NB200_OK) NB_CUDAP(cudaEventRecord(ctx->done_ev[slot], ctx->stream));
    }
    // iFFT + LDE (+ optionally the same polynomials on the first half of the next larger canonic domain) of this chunk
    if (st == NB200_OK) st = commit_transforms(ctx, d_evals + c0 * len, d_coeffs + c0 * len, d_lde + c0 * lde_len, d_half_ext ? d_half_ext + c0 * lde_len : nullptr, nc, log_size, log_blowup);
    // optional: continue the Merkle leaf hashes over this chunk's LDE columns
    if (st == NB200_OK && leaf && leaf->tree) st = merkle_leaf_absorb(ctx, leaf->tree, d_lde + c0 * lde_len, lde_len, nc, c0, n_cols, c0 + nc == n_cols);
  }
#undef NB_CUDAP
  return done(st);
}
}  // namespace nb

extern "C" {

nb200_status nb200_host_alloc(size_t bytes, void** out) {
  if (!out) return NB200_ERR_ARG;
  cudaError_t e = cudaHostAlloc(out, bytes ? bytes : 16, cudaHostAllocDefault);
  return e == cudaSuccess ? NB200_OK : NB200_ERR_OOM;
}
void nb200_host_free(void* p) { if (p) cudaFreeHost(p); }

nb200_status nb200_commit_host(nb200_ctx* ctx, const uint32_t* const* host_batches, const size_t* n_cols, const uint32_t* log_sizes, size_t n_batches,
                               int coset_order, uint32_t log_blowup, nb200_cols** evals_io, nb200_cols** coeffs_io, nb200_cols** lde_io,
                               nb200_tree** tree_out, uint8_t root[32]) {
  return nb200_commit_host_packed(ctx, (const void* const*)host_batches, nullptr, n_cols, log_sizes, n_batches, coset_order, log_blowup, evals_io, coeffs_io, lde_io, tree_out, root);
}

nb200_status nb200_commit_host_packed(nb200_ctx* ctx, const void* const* host_batches, const uint32_t* elem_bytes, const size_t* n_cols, const uint32_t* log_sizes,
                                      size_t n_batches, int coset_order, uint32_t log_blowup, nb200_cols** evals_io, nb200_cols** coeffs_io, nb200_cols** lde_io,
                                      nb200_tree** tree_out, uint8_t root[32]) {
  if (!ctx || !host_batches || !evals_io || !coeffs_io || !lde_io || !tree_out) return NB200_ERR_ARG;
  for (size_t b = 0; elem_bytes && b < n_batches; ++b) NB_ARG(ctx, elem_bytes[b] == 1 || elem_bytes[b] == 2 || elem_bytes[b] == 4, "commit_host: 1, 2 or 4 bytes per host word");
  u32 max_log = 0;
  for (size_t b = 0; b < n_batches; ++b) max_log = std::max(max_log, log_sizes[b] + log_blowup);
  if (max_log >= 1) NB_TRY(twiddles_prepare(ctx, max_log));
  std::vector<ColRef> cols;
  LeafSink sink;
  const long leaf_batch = leaf_sink_batch(n_cols, log_sizes, n_batches);
  // batches allocated here stay in the caller's arrays (the caller owns them either way); the partial tree does not leak
  auto fail = [&](nb200_status st) { if (sink.tree) { nb200_tree_free(ctx, sink.tree); sink.tree = nullptr; } return st; };
#define NB_TRYC(expr) do { nb200_status _s = (expr); if (_s != NB200_OK) return fail(_s); } while (0)
  if (leaf_batch >= 0) NB_TRYC(merkle_tree_alloc(ctx, max_log, &sink.tree));
  for (size_t b = 0; b < n_batches; ++b) {
    if (!evals_io[b]) NB_TRYC(nb200_cols_alloc(ctx, n_cols[b], log_sizes[b], &evals_io[b]));
    if (!coeffs_io[b]) NB_TRYC(nb200_cols_alloc(ctx, n_cols[b], log_sizes[b], &coeffs_io[b]));
    if (!lde_io[b]) NB_TRYC(nb200_cols_alloc(ctx, n_cols[b], log_sizes[b] + log_blowup, &lde_io[b]));
    if (!(evals_io[b]->n_cols == n_cols[b] && evals_io[b]->log_size == log_sizes[b] && coeffs_io[b]->n_cols == n_cols[b] &&
          coeffs_io[b]->log_size == log_sizes[b] && lde_io[b]->n_cols == n_cols[b] && lde_io[b]->log_size == log_sizes[b] + log_blowup))
      return fail(set_err(ctx, NB200_ERR_ARG, "commit_host: batch shapes"));
    NB_TRYC(upload_transform_pipelined(ctx, host_batches[b], n_cols[b], log_sizes[b], coset_order, log_blowup, evals_io[b]->d, coeffs_io[b]->d, lde_io[b]->d,
                                       nullptr, (long)b == leaf_batch ? &sink : nullptr, elem_bytes ? elem_bytes[b] : 4u));
    for (size_t c = 0; c < n_cols[b]; ++c) cols.push_back(ColRef{lde_io[b]->col(c), lde_io[b]->log_size});
  }
#undef NB_TRYC
  NB_TRY(merkle_commit(ctx, cols, tree_out, sink.tree));
  if (root) memcpy(root, (*tree_out)->root, 32);
  return NB200_OK;
}

// PolyOps::interpolate_columns + evaluate_polynomials as one call (the transform half of nb200_commit_evals; evaluations are only read)
nb200_status nb200_interpolate_evaluate(nb200_ctx* ctx, const nb200_cols* evals, uint32_t log_blowup, nb200_cols* coeffs, nb200_cols* lde) {
  if (!ctx || !evals || !coeffs || !lde) return NB200_ERR_ARG;
  NB_ARG(ctx, coeffs->n_cols == evals->n_cols && coeffs->log_size == evals->log_size, "interpolate_evaluate: coefficient batch shape");
  NB_ARG(ctx, lde->n_cols == evals->n_cols && lde->log_size == evals->log_size + log_blowup, "interpolate_evaluate: LDE batch shape");
  if (lde->log_size >= 1) NB_TRY(twiddles_prepare(ctx, lde->log_size));
  return commit_transforms(ctx, evals->d, coeffs->d, lde->d, nullptr, evals->n_cols, evals->log_size, log_blowup);
}

// ---- fused commitment ----
nb200_status nb200_commit_evals(nb200_ctx* ctx, const nb200_cols* const* eval_batches, size_t n_batches, uint32_t log_blowup,
                                nb200_cols** coeffs_io, nb200_cols** lde_io, nb200_tree** tree_out, uint8_t root[32]) {
  if (!ctx || !coeffs_io || !lde_io || !tree_out) return NB200_ERR_ARG;
  u32 max_log = 0;
  for (size_t b = 0; b < n_batches; ++b) max_log = std::max(max_log, eval_batches[b]->log_size + log_blowup);
  if (max_log >= 1) NB_TRY(twiddles_prepare(ctx, max_log));
  std::vector<ColRef> cols;
  for (size_t b = 0; b < n_batches; ++b) {
    const nb200_cols* ev = eval_batches[b];
    if (!coeffs_io[b]) NB_TRY(nb200_cols_alloc(ctx, ev->n_cols, ev->log_size, &coeffs_io[b]));
    if (!lde_io[b]) NB_TRY(nb200_cols_alloc(ctx, ev->n_cols, ev->log_size + log_blowup, &lde_io[b]));
    nb200_cols *co = coeffs_io[b], *lde = lde_io[b];
    NB_ARG(ctx, co->n_cols == ev->n_cols && co->log_size == ev->log_size, "commit_evals: coefficient batch shape");
    NB_ARG(ctx, lde->n_cols == ev->n_cols && lde->log_size == ev->log_size + log_blowup, "commit_evals: LDE batch shape");
    NB_TRY(commit_transforms(ctx, ev->d, co->d, lde->d, nullptr, ev->n_cols, ev->log_size, log_blowup));
    for (size_t c = 0; c < lde->n_cols; ++c) cols.push_back(ColRef{lde->col(c), lde->log_size});
  }
  NB_TRY(merkle_commit(ctx, cols, tree_out));
  if (root) memcpy(root, (*tree_out)->root, 32);
  return NB200_OK;
}

}  // extern "C"
