// Shared definitions of the product library (context, device column batches, trees, error plumbing).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <memory>
#include <string>
#include <vector>
#include "../../include/nb200.h"
#include "m31.cuh"

namespace nb {

struct TwiddleBank {
  u32 half_log = 0;       // log size k of the root half coset; buffers hold 2^k words
  u32* d_tw = nullptr;    // x-coordinates, layer l at offset 2^k - 2^(k-l), bit-reversed within the layer
  u32* d_itw = nullptr;   // element-wise inverses
  u32* d_tw2 = nullptr;   // 2 * twiddle (< 2^32): the FFT's Mersenne multiply wants the doubled constant (m31_mul_dbl)
  u32* d_itw2 = nullptr;  // 2 * inverse twiddle
  // product banks for the radix-4 steps (fft_common.cuh radix16p): entry j of layer l = 2 * (t_l[j] * t_{l+1}[j >> 1]), negated for odd j
  u32* d_ptw2 = nullptr;
  u32* d_iptw2 = nullptr;
};

}  // namespace nb

struct nb200_ctx {
  int device = 0;
  int sm_count = 132;   // H100 SXM; overwritten from the device properties at ctx creation
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  std::string err;
  nb::TwiddleBank tw;
  int merkle_hash = 0, draw_domain_sep = 0, pow_variant = 0;
  uint64_t launches = 0;
  int trace = 0;          // NB200_TRACE=1: per-stage wall clock (after a stream sync) on stderr
  double trace_t0 = 0;
  cudaStream_t copy_stream = nullptr;  // H2D side stream of the pipelined host-column path
  cudaEvent_t copy_ev[2] = {nullptr, nullptr}, done_ev[2] = {nullptr, nullptr};
  // scratch for small device->host transfers
  void* h_pinned = nullptr;
  size_t h_pinned_bytes = 0;
  void* fft_tables = nullptr;          // per-ctx circle-twiddle tables (fft.cu)
  void* comm = nullptr;                // NCCL communicator state (comm.cu), nullptr = single GPU
  size_t total_mem = 0;                // device memory (bytes), read once at ctx creation
  size_t live_bytes = 0;               // bytes held by nb200_cols batches of this ctx (the dominant allocations): the library's own accounting —
                                       // cudaMemGetInfo stalls for milliseconds while stream-ordered frees are pending and does not see the pool
};
#define NB_MAX_DEVICES 64

struct nb200_cols {
  nb200_ctx* ctx = nullptr;
  size_t n_cols = 0;
  uint32_t log_size = 0;
  uint32_t* d = nullptr;  // n_cols * 2^log_size words, column-major
  bool owns = true;
  size_t col_len() const { return (size_t)1 << log_size; }
  uint32_t* col(size_t c) const { return d + c * col_len(); }
};

struct nb200_tree {
  nb200_ctx* ctx = nullptr;
  uint32_t max_log = 0;
  uint8_t* d_pool = nullptr;              // all layers, root first
  std::vector<uint8_t*> layer;            // layer[l] -> 32 * 2^l bytes
  uint8_t root[32];
};

namespace nb {

inline nb200_status set_err(nb200_ctx* ctx, nb200_status st, const std::string& msg) {
  if (ctx) ctx->err = msg;
  return st;
}
std::string& global_err();

#define NB_CUDA(ctx, call)                                                                                   \
  do {                                                                                                       \
    cudaError_t _e = (call);                                                                                 \
    if (_e != cudaSuccess) {                                                                                 \
      return nb::set_err(ctx, _e == cudaErrorMemoryAllocation ? NB200_ERR_OOM : NB200_ERR_CUDA,              \
                         std::string(#call) + ": " + cudaGetErrorString(_e) + " @" + __FILE__ + ":" + std::to_string(__LINE__)); \
    }                                                                                                        \
  } while (0)

#define NB_LAUNCH_CHECK(ctx)                                                                                 \
  do {                                                                                                       \
    (ctx)->launches += 1;                                                                                    \
    cudaError_t _e = cudaGetLastError();                                                                     \
    if (_e != cudaSuccess)                                                                                   \
      return nb::set_err(ctx, NB200_ERR_CUDA, std::string("kernel launch: ") + cudaGetErrorString(_e) + " @" + __FILE__ + ":" + std::to_string(__LINE__)); \
  } while (0)

#define NB_ARG(ctx, cond, msg)                                                   \
  do {                                                                           \
    if (!(cond)) return nb::set_err(ctx, NB200_ERR_ARG, std::string(msg));       \
  } while (0)

#define NB_TRY(expr)                          \
  do {                                        \
    nb200_status _s = (expr);                 \
    if (_s != NB200_OK) return _s;            \
  } while (0)

// NB200_TRACE stage timer: prints the time since the previous mark (stream drained first)
void trace_mark(nb200_ctx* ctx, const char* stage);

// Stream-ordered device allocation from the device's default memory pool (release threshold raised at ctx
// creation, so steady-state alloc/free never reaches the driver).
inline cudaError_t dmalloc(nb200_ctx* ctx, void** p, size_t bytes) { return cudaMallocAsync(p, bytes ? bytes : 16, ctx->stream); }
inline void dfree(nb200_ctx* ctx, void* p) { if (p) cudaFreeAsync(p, ctx->stream); }

// Owning handles: an error return frees what a function still holds, in the stream order of its other frees.
// Batches and trees carry their ctx, so the deleters need none.
struct ColsDeleter { void operator()(nb200_cols* c) const { nb200_cols_free(c->ctx, c); } };
struct TreeDeleter { void operator()(nb200_tree* t) const { nb200_tree_free(t->ctx, t); } };
using ColsPtr = std::unique_ptr<nb200_cols, ColsDeleter>;
using TreePtr = std::unique_ptr<nb200_tree, TreeDeleter>;
// one dmalloc buffer of u32 words, freed on ctx->stream
struct DevBuf {
  nb200_ctx* ctx = nullptr;
  u32* p = nullptr;
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : ctx(o.ctx), p(o.p) { o.p = nullptr; }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { dfree(ctx, p); }
};
// fill an empty handle; on failure it stays empty
inline nb200_status alloc(nb200_ctx* ctx, ColsPtr& out, size_t n_cols, u32 log_size) {
  nb200_cols* c = nullptr;
  NB_TRY(nb200_cols_alloc(ctx, n_cols, log_size, &c));
  out.reset(c);
  return NB200_OK;
}
inline nb200_status alloc(nb200_ctx* ctx, DevBuf& out, size_t words) {
  u32* p = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&p, words * 4));
  out.ctx = ctx; out.p = p;
  return NB200_OK;
}

// ---- internal launchers (implemented in the .cu files) ----
nb200_status twiddles_prepare(nb200_ctx* ctx, u32 max_domain_log);
// Circle iFFT in place over a batch (evaluations -> coefficients)
// tw_log = log_size + 1 selects the HALF-DOMAIN transform: the domain is the first half (rows [0, 2^log_size) in bit-reversed order) of
// CanonicCoset(log_size + 1).circle_domain() instead of CanonicCoset(log_size).circle_domain(); 0 = the canonic domain.
nb200_status fft_interpolate(nb200_ctx* ctx, const u32* src, u32* dst, size_t n_cols, u32 log_size, u32 tw_log = 0);
// Circle FFT: coefficients (src, log src_log) zero-extended to dst (log dst_log); src may equal dst if logs match
nb200_status fft_evaluate(nb200_ctx* ctx, const u32* src, u32 src_log, u32* dst, u32 dst_log, size_t n_cols, u32 tw_log = 0);
// evaluations -> coefficients + LDE (+ optionally the half-coset extension the quotient step needs) for one batch (fft_fused.cu)
// destination of a row-sharded commitment: rank q's row-slice buffers (2^log_slice rows of every column) as mapped in THIS process
struct RowScatter { int world = 1; u32 log_slice = 0; size_t col0 = 0; u32* lde_rows[16] = {nullptr}; u32* hx_rows[16] = {nullptr}; };
nb200_status commit_transforms(nb200_ctx* ctx, const u32* evals, u32* coeffs, u32* lde, u32* half_ext, size_t n_cols, u32 log_size, u32 log_blowup,
                               const RowScatter* scatter = nullptr, bool* scattered = nullptr);
bool commit_transforms_can_scatter(u32 n, u32 bl, u32 log_slice, int world);
// ---- multi-GPU plumbing (comm.cu): NCCL over the ranks that prove one trace together; all no-ops / local copies without a communicator
void comm_release(nb200_ctx* ctx);
int comm_rank(const nb200_ctx* ctx);
int comm_world(const nb200_ctx* ctx);
int comm_log_world(const nb200_ctx* ctx);
void comm_shard_range(size_t total, int world, int rank, size_t* first, size_t* count);
nb200_status exchange_rows_to_cols(nb200_ctx* ctx, const u32* src_rows, size_t total, size_t LEN, u32* dst);
nb200_status comm_all_gather_dev(nb200_ctx* ctx, const u32* mine, size_t words, u32* out);
// symmetric peer heap (CUDA IPC over NVLink): see comm.cu
struct PeerBuf { u32* d = nullptr; int seg = -1; size_t off = 0; };
nb200_status peer_alloc(nb200_ctx* ctx, const void* owner, size_t words, PeerBuf* out);
u32* peer_ptr(nb200_ctx* ctx, const PeerBuf& b, int q);
void peer_heap_release(nb200_ctx* ctx, const void* owner);
nb200_status peer_cols_to_rows_chunk(nb200_ctx* ctx, cudaStream_t st, const u32* src, size_t total, size_t LEN, const PeerBuf& dst_rows, int j, int nch);
nb200_status peer_rows_to_cols(nb200_ctx* ctx, cudaStream_t st, const u32* src_rows, size_t total, size_t LEN, const PeerBuf& dst_shard);
nb200_status comm_barrier_stream(nb200_ctx* ctx);
cudaStream_t comm_side_stream(nb200_ctx* ctx);
nb200_status comm_fork(nb200_ctx* ctx);
nb200_status comm_join(nb200_ctx* ctx);
nb200_status exchange_cols_to_rows_chunk(nb200_ctx* ctx, cudaStream_t st, const u32* src, size_t total, size_t LEN, u32* dst_rows, u32* pack, int j, int nch);
nb200_status comm_all_reduce_sum_host(nb200_ctx* ctx, u32* host, size_t words);
nb200_status reorder_coset_to_bitrev(nb200_ctx* ctx, const u32* src, u32* dst, size_t n_cols, u32 log_size);
nb200_status expand_reorder(nb200_ctx* ctx, const void* src, u32 elem_bytes, u32* dst, size_t n_cols, u32 log_size, int coset_order);
// Host columns -> device evaluations -> coefficients -> LDE, in column chunks: the H2D copy of chunk k+1 (side stream)
// overlaps the transforms of chunk k.  `host` is n_cols x 2^log_size words (pinned memory for real overlap).
struct LeafSink { nb200_tree* tree = nullptr; };  // set for the one batch that holds all the largest columns of a tree (incremental leaf hashing)
// elem_bytes: width of a host word (4 = u32; 1 / 2 = the packed formats for byte- / halfword-valued columns, expanded on the device)
nb200_status upload_transform_pipelined(nb200_ctx* ctx, const void* host, size_t n_cols, u32 log_size, int coset_order, u32 log_blowup,
                                        u32* d_evals, u32* d_coeffs, u32* d_lde, u32* d_half_ext = nullptr, LeafSink* leaf = nullptr, u32 elem_bytes = 4);

struct ColRef { const u32* d; u32 log_size; };
nb200_status merkle_commit(nb200_ctx* ctx, const std::vector<ColRef>& cols, nb200_tree** out, nb200_tree* pre_leaf = nullptr);
// incremental leaf hashing while column chunks arrive from the host (merkle.cu)
nb200_status merkle_tree_alloc(nb200_ctx* ctx, u32 max_log, nb200_tree** out);
nb200_status merkle_leaf_absorb(nb200_ctx* ctx, nb200_tree* tree, const u32* d_cols, size_t stride, size_t n_cols, size_t cols_before, size_t total_cols, bool final);
long leaf_sink_batch(const size_t* n_cols, const u32* log_sizes, size_t n_batches);  // set for the one batch that holds all the largest columns of a tree
// The top log2(world) = k levels of a row-sharded tree (comm.cu), hashed on the host, identically on every rank: layers[k] holds the world
// sub-tree roots (the caps) on entry; layers[k-1] .. layers[0] are filled, mixing in the columns of 2^l < world LDE values at layer l.
struct TopCol { u32 log; std::vector<u32> vals; };
nb200_status hash_top_layers(nb200_ctx* ctx, u32 k, const std::vector<TopCol>& top, std::vector<std::vector<uint8_t>>& layers);

}  // namespace nb
