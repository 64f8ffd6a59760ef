// One commitment over N GPUs, inside the library (SURVEY.md §8e; BASELINE configs[3]): the ranks that prove ONE trace together share an
// NCCL communicator owned by the nb200_ctx.  The commit of a tree (TreeBuilder::extend_evals + commit, nexus-zkvm
// prover/src/machine.rs:208-263) shards at two granularities with one exchange between them:
//   1. column-sharded  rank r runs the fused iFFT + LDE pipeline (fft_fused.cu) on its column range nb200_shard_range(total, world, r)
//                      (multiples of 16 columns = one 64-byte Blake2s block);
//   2. exchange        grouped ncclSend/ncclRecv over NVLink: rank q receives rows [q * 2^(m-k), (q+1) * 2^(m-k)) of every column
//                      (m = LDE log size, world = 2^k).  In bit-reversed order that contiguous slice of a column is one depth-k sub-tree's
//                      leaves.  The sender packs its (own columns x peer's rows) block with one strided D2D copy; the receiver needs no
//                      unpacking: a peer's columns are adjacent in the row-slice batch;
//   3. row-sharded     rank q hashes its sub-tree over ALL columns of its rows (merkle.cu), the world 32-byte caps are all-gathered
//                      (ncclAllGather) and every rank finishes the top k levels on the host — the root is bit-identical to the one-GPU root.
// LDE VALUES are exchanged, not coefficients: evaluating every column on a rank's sub-coset from coefficients would need every column's full
// coefficient vector on every rank (world x the memory), which the 2^24-row configuration cannot afford.
//
// NCCL is bound with dlopen (no link-time dependency: the library still loads on a box without NCCL, and inside a PyTorch process it shares
// the libnccl that torch already loaded instead of bringing a second copy).
#include "common.cuh"
#include "blake2s.cuh"
#include <dlfcn.h>
#include <nccl.h>
#include <cstring>
#include <algorithm>

extern "C" nb200_status nb200_comm_all_gather(nb200_ctx* ctx, const uint8_t* mine, size_t bytes, uint8_t* out);

namespace nb {

struct NcclApi {
  void* h = nullptr;
  bool ok = false;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi& nccl() {
  static NcclApi a;
  static bool tried = false;
  if (tried) return a;
  tried = true;
  // a copy already mapped into the process (PyTorch's) wins; then $NB200_NCCL_LIB; then the system library
  const char* env = getenv("NB200_NCCL_LIB");
  a.h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
  if (!a.h && env && env[0]) a.h = dlopen(env, RTLD_NOW | RTLD_GLOBAL);
  if (!a.h) a.h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!a.h) a.h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!a.h) return a;
#define NB_SYM(f) a.f = (decltype(a.f))dlsym(a.h, "nccl" #f); if (!a.f) return a;
  NB_SYM(GetUniqueId) NB_SYM(CommInitRank) NB_SYM(CommDestroy) NB_SYM(AllGather) NB_SYM(Send) NB_SYM(Recv) NB_SYM(AllReduce) NB_SYM(GroupStart) NB_SYM(GroupEnd) NB_SYM(GetErrorString)
#undef NB_SYM
  a.ok = true;
  return a;
}

struct Comm {
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1, log_world = 0;
  cudaStream_t side = nullptr;                 // exchanges that overlap the transforms run here (comm_fork / comm_join order it against ctx->stream)
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  // symmetric peer heap: cudaMalloc'd segments whose CUDA-IPC handles every rank has opened; all ranks allocate the same sizes in the same order, so
  // a buffer has the same (segment, offset) everywhere and rank q's copy is reachable as seg.peer[q] + offset (NVLink peer stores / copy engines)
  struct Seg { u32* base = nullptr; size_t words = 0, used = 0; std::vector<u32*> peer; };
  std::vector<Seg> heap;
  int peer_state = -1;                         // -1 not tried, 0 unavailable (exchanges go through NCCL), 1 in use
  const void* heap_owner = nullptr;            // the scheme whose sharded trees live in the heap (one sharded proof at a time per context)
  u32* d_flag = nullptr;                       // 1-word buffer of the stream-ordered barrier
};

#define NB_NCCL(ctx, call)                                                                                                        \
  do {                                                                                                                            \
    ncclResult_t _r = (call);                                                                                                     \
    if (_r != ncclSuccess) return set_err(ctx, NB200_ERR_CUDA, std::string(#call) + ": " + nccl().GetErrorString(_r));            \
  } while (0)

void comm_release(nb200_ctx* ctx) {
  Comm* c = (Comm*)ctx->comm;
  if (!c) return;
  if (c->comm && nccl().ok) nccl().CommDestroy(c->comm);
  for (auto& sg : c->heap) {
    for (int q = 0; q < (int)sg.peer.size(); ++q) if (q != c->rank && sg.peer[q]) cudaIpcCloseMemHandle(sg.peer[q]);
    if (sg.base) cudaFree(sg.base);
  }
  if (c->d_flag) cudaFree(c->d_flag);
  if (c->side) cudaStreamDestroy(c->side);
  if (c->ev_fork) cudaEventDestroy(c->ev_fork);
  if (c->ev_join) cudaEventDestroy(c->ev_join);
  delete c;
  ctx->comm = nullptr;
}

// contiguous, 16-column-aligned column ranges, as even as possible (the last ranks may be empty for tiny trees)
static void shard_range(size_t total, int world, int rank, size_t* first, size_t* count) {
  const size_t align = 16, blocks = (total + align - 1) / align;
  size_t start = 0;
  for (int r = 0; r <= rank; ++r) {
    size_t nb = blocks / world + ((size_t)r < blocks % world ? 1 : 0);
    size_t end = std::min(total, start + nb * align);
    if (r == rank) { *first = start; *count = end - start; return; }
    start = end;
  }
}


int comm_rank(const nb200_ctx* ctx) { return ctx->comm ? ((Comm*)ctx->comm)->rank : 0; }
int comm_world(const nb200_ctx* ctx) { return ctx->comm ? ((Comm*)ctx->comm)->world : 1; }
int comm_log_world(const nb200_ctx* ctx) { return ctx->comm ? ((Comm*)ctx->comm)->log_world : 0; }
void comm_shard_range(size_t total, int world, int rank, size_t* first, size_t* count) { shard_range(total, world, rank, first, count); }

// ---- side stream: the row re-shard of column chunk j travels over NVLink while chunk j + 1 is being transformed on ctx->stream ----
cudaStream_t comm_side_stream(nb200_ctx* ctx) {
  Comm* c = (Comm*)ctx->comm;
  if (!c) return ctx->stream;
  if (!c->side) {
    if (cudaStreamCreateWithFlags(&c->side, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming) != cudaSuccess) { cudaGetLastError(); c->side = nullptr; return ctx->stream; }
  }
  return c->side;
}
// work enqueued on the side stream after this call sees everything enqueued on ctx->stream before it
nb200_status comm_fork(nb200_ctx* ctx) {
  cudaStream_t s = comm_side_stream(ctx);
  if (s == ctx->stream) return NB200_OK;
  Comm* c = (Comm*)ctx->comm;
  NB_CUDA(ctx, cudaEventRecord(c->ev_fork, ctx->stream));
  NB_CUDA(ctx, cudaStreamWaitEvent(s, c->ev_fork, 0));
  return NB200_OK;
}
// ... and the reverse: ctx->stream continues after everything enqueued on the side stream so far
nb200_status comm_join(nb200_ctx* ctx) {
  cudaStream_t s = comm_side_stream(ctx);
  if (s == ctx->stream) return NB200_OK;
  Comm* c = (Comm*)ctx->comm;
  NB_CUDA(ctx, cudaEventRecord(c->ev_join, s));
  NB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, c->ev_join, 0));
  return NB200_OK;
}

// stream-ordered barrier: when it completes on this rank's ctx->stream, every rank's stream has reached its own call (all earlier work there is done)
nb200_status comm_barrier_stream(nb200_ctx* ctx) {
  Comm* c = (Comm*)ctx->comm;
  if (!c || c->world == 1) return NB200_OK;
  if (!c->d_flag) { NB_CUDA(ctx, cudaMalloc((void**)&c->d_flag, 256)); NB_CUDA(ctx, cudaMemsetAsync(c->d_flag, 0, 256, ctx->stream)); }
  NB_NCCL(ctx, nccl().AllReduce(c->d_flag, c->d_flag, 1, ncclUint32, ncclSum, c->comm, ctx->stream));
  return NB200_OK;
}

// ---- symmetric peer heap -------------------------------------------------------------------------------------------------------------------
static bool all_ranks_agree(nb200_ctx* ctx, Comm* c, int mine) {
  std::vector<uint8_t> all((size_t)c->world * 4);
  int32_t v = mine;
  if (nb200_comm_all_gather(ctx, (const uint8_t*)&v, 4, all.data()) != NB200_OK) return false;
  for (int q = 0; q < c->world; ++q) { int32_t x; memcpy(&x, &all[(size_t)q * 4], 4); if (!x) return false; }
  return true;
}
// collective: every rank creates a segment of `words`, the IPC handles are all-gathered and opened; on any failure anywhere ALL ranks give the heap up
static bool peer_new_segment(nb200_ctx* ctx, Comm* c, size_t words) {
  Comm::Seg sg;
  sg.words = words;
  sg.peer.assign(c->world, nullptr);
  struct Msg { cudaIpcMemHandle_t h; int32_t ok; int32_t pad[3]; } mine;
  memset(&mine, 0, sizeof mine);
  bool ok = cudaMalloc((void**)&sg.base, words * 4) == cudaSuccess && cudaIpcGetMemHandle(&mine.h, sg.base) == cudaSuccess;
  if (!ok) cudaGetLastError();
  mine.ok = ok ? 1 : 0;
  std::vector<uint8_t> all((size_t)c->world * sizeof(Msg));
  bool gathered = nb200_comm_all_gather(ctx, (const uint8_t*)&mine, sizeof mine, all.data()) == NB200_OK;
  bool everyone = gathered;
  for (int q = 0; q < c->world && everyone; ++q) { Msg m; memcpy(&m, &all[(size_t)q * sizeof(Msg)], sizeof m); if (!m.ok) everyone = false; }
  bool opened = everyone;
  if (everyone) {
    sg.peer[c->rank] = sg.base;
    for (int q = 0; q < c->world && opened; ++q) {
      if (q == c->rank) continue;
      Msg m; memcpy(&m, &all[(size_t)q * sizeof(Msg)], sizeof m);
      if (cudaIpcOpenMemHandle((void**)&sg.peer[q], m.h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); sg.peer[q] = nullptr; opened = false; }
    }
  }
  const bool agreed = gathered && all_ranks_agree(ctx, c, opened ? 1 : 0);
  if (!agreed) {
    for (int q = 0; q < c->world; ++q) if (q != c->rank && sg.peer[q]) cudaIpcCloseMemHandle(sg.peer[q]);
    if (sg.base) cudaFree(sg.base);
    return false;
  }
  c->heap.push_back(std::move(sg));
  return true;
}
// Bump allocation of `words` (the same on every rank, collective when a new segment is needed).  out->d == nullptr: no peer heap (single rank,
// NB200_PEER_HEAP=0, or CUDA IPC unavailable between the ranks) — the caller uses the NCCL exchange instead; the answer is the same on every rank.
nb200_status peer_alloc(nb200_ctx* ctx, const void* owner, size_t words, PeerBuf* out) {
  *out = PeerBuf();
  Comm* c = (Comm*)ctx->comm;
  static const bool enabled = [] { const char* e = getenv("NB200_PEER_HEAP"); return !(e && e[0] == '0'); }();
  if (!c || c->world == 1 || !enabled || c->peer_state == 0) return NB200_OK;
  if (c->heap_owner && c->heap_owner != owner) {
    bool any = false;
    for (auto& sg : c->heap) any = any || sg.used;
    NB_ARG(ctx, !any, "peer heap: one sharded proof at a time per context (free the previous scheme first)");
  }
  c->heap_owner = owner;
  words = (words + 63) & ~(size_t)63;                    // 256-byte granules
  for (size_t i = 0; i < c->heap.size(); ++i) {
    auto& sg = c->heap[i];
    if (sg.words - sg.used >= words) { out->d = sg.base + sg.used; out->seg = (int)i; out->off = sg.used; sg.used += words; return NB200_OK; }
  }
  static const size_t min_seg = [] { const char* e = getenv("NB200_PEER_SEG_MIB"); size_t v = e ? (size_t)atoll(e) : 4096; return (v < 64 ? 64 : v) << 18; }();   // words
  if (!peer_new_segment(ctx, c, std::max(words, min_seg))) { c->peer_state = 0; return NB200_OK; }
  c->peer_state = 1;
  auto& sg = c->heap.back();
  out->d = sg.base; out->seg = (int)c->heap.size() - 1; out->off = 0; sg.used = words;
  return NB200_OK;
}
u32* peer_ptr(nb200_ctx* ctx, const PeerBuf& b, int q) {
  Comm* c = (Comm*)ctx->comm;
  return c->heap[b.seg].peer[q] + b.off;
}
// every allocation of `owner` is released (the memory stays mapped for the next proof)
void peer_heap_release(nb200_ctx* ctx, const void* owner) {
  Comm* c = ctx ? (Comm*)ctx->comm : nullptr;
  if (!c || c->heap_owner != owner) return;
  for (auto& sg : c->heap) sg.used = 0;
  c->heap_owner = nullptr;
}

// columns -> rows straight into the owners' row-slice buffers (peer heap): one strided 2-D copy per destination rank — no pack buffer, no NCCL
// staging, no SMs (copy engines over NVLink), so it overlaps the transforms of the next column chunk for real.  Chunking as in the NCCL variant.
nb200_status peer_cols_to_rows_chunk(nb200_ctx* ctx, cudaStream_t st, const u32* src, size_t total, size_t LEN, const PeerBuf& dst_rows, int j, int nch) {
  Comm* c = (Comm*)ctx->comm;
  const int world = c->world, rank = c->rank;
  const size_t S = LEN / world;
  size_t first = 0, count = 0;
  shard_range(total, world, rank, &first, &count);
  const size_t c0 = count * j / nch, c1 = count * (j + 1) / nch, nc = c1 - c0;
  if (!nc) return NB200_OK;
  for (int d = 0; d < world; ++d) {
    const int q = (rank + d) % world;                    // own slice first, then the peers in a rotated order (spreads the NVLink targets)
    NB_CUDA(ctx, cudaMemcpy2DAsync(peer_ptr(ctx, dst_rows, q) + (first + c0) * S, S * 4, src + c0 * LEN + (size_t)q * S, LEN * 4, S * 4, nc, cudaMemcpyDefault, st));
  }
  return NB200_OK;
}
// rows -> columns: this rank's S rows of rank q's columns go into q's column shard (peer heap) at row offset rank * S
nb200_status peer_rows_to_cols(nb200_ctx* ctx, cudaStream_t st, const u32* src_rows, size_t total, size_t LEN, const PeerBuf& dst_shard) {
  Comm* c = (Comm*)ctx->comm;
  const int world = c->world, rank = c->rank;
  const size_t S = LEN / world;
  for (int d = 0; d < world; ++d) {
    const int q = (rank + d) % world;
    size_t qf = 0, qc = 0;
    shard_range(total, world, q, &qf, &qc);
    if (qc) NB_CUDA(ctx, cudaMemcpy2DAsync(peer_ptr(ctx, dst_shard, q) + (size_t)rank * S, LEN * 4, src_rows + qf * S, S * 4, S * 4, qc, cudaMemcpyDefault, st));
  }
  return NB200_OK;
}

// columns -> rows, column chunk j of nch (every rank splits ITS column range into the same number of chunks, so the grouped send / recv pairs match):
// `src` = base of this rank's columns, `pack` = scratch of (world - 1) x (chunk columns) x (LEN / world) words, everything enqueued on `st`.
nb200_status exchange_cols_to_rows_chunk(nb200_ctx* ctx, cudaStream_t st, const u32* src, size_t total, size_t LEN, u32* dst_rows, u32* pack, int j, int nch) {
  Comm* c = (Comm*)ctx->comm;
  const int world = c ? c->world : 1, rank = c ? c->rank : 0;
  const size_t S = LEN / world;
  size_t first = 0, count = 0;
  shard_range(total, world, rank, &first, &count);
  const size_t c0 = count * j / nch, c1 = count * (j + 1) / nch, nc = c1 - c0;
  if (nc) NB_CUDA(ctx, cudaMemcpy2DAsync(dst_rows + (first + c0) * S, S * 4, src + c0 * LEN + (size_t)rank * S, LEN * 4, S * 4, nc, cudaMemcpyDeviceToDevice, st));
  if (world == 1) return NB200_OK;
  size_t slot = 0;
  for (int q = 0; q < world; ++q) {
    if (q == rank || !nc) continue;
    NB_CUDA(ctx, cudaMemcpy2DAsync(pack + slot * nc * S, S * 4, src + c0 * LEN + (size_t)q * S, LEN * 4, S * 4, nc, cudaMemcpyDeviceToDevice, st));
    ++slot;
  }
  ncclResult_t r = nccl().GroupStart();
  slot = 0;
  for (int q = 0; q < world && r == ncclSuccess; ++q) {
    if (q == rank) continue;
    size_t qf = 0, qc = 0;
    shard_range(total, world, q, &qf, &qc);
    const size_t q0 = qc * j / nch, q1 = qc * (j + 1) / nch;
    if (nc) { r = nccl().Send(pack + slot * nc * S, nc * S, ncclUint32, q, c->comm, st); ++slot; }
    if (r == ncclSuccess && q1 > q0) r = nccl().Recv(dst_rows + (qf + q0) * S, (q1 - q0) * S, ncclUint32, q, c->comm, st);
  }
  ncclResult_t r2 = nccl().GroupEnd();
  if (r != ncclSuccess || r2 != ncclSuccess) return set_err(ctx, NB200_ERR_CUDA, std::string("exchange cols->rows (chunk): ") + nccl().GetErrorString(r != ncclSuccess ? r : r2));
  return NB200_OK;
}

// rows -> columns (the inverse): `src_rows` = all `total` columns x this rank's S rows; `dst` = this rank's columns, LEN words each.
nb200_status exchange_rows_to_cols(nb200_ctx* ctx, const u32* src_rows, size_t total, size_t LEN, u32* dst) {
  Comm* c = (Comm*)ctx->comm;
  const int world = c ? c->world : 1, rank = c ? c->rank : 0;
  const size_t S = LEN / world;
  size_t first = 0, count = 0;
  shard_range(total, world, rank, &first, &count);
  if (count) NB_CUDA(ctx, cudaMemcpy2DAsync(dst + (size_t)rank * S, LEN * 4, src_rows + first * S, S * 4, S * 4, count, cudaMemcpyDeviceToDevice, ctx->stream));
  if (world == 1) return NB200_OK;
  u32* stage = nullptr;
  if (count) NB_CUDA(ctx, dmalloc(ctx, (void**)&stage, (size_t)(world - 1) * count * S * 4));
  nb200_status st = NB200_OK;
  ncclResult_t r = nccl().GroupStart();
  size_t slot = 0;
  for (int q = 0; q < world && r == ncclSuccess; ++q) {
    if (q == rank) continue;
    size_t qf = 0, qc = 0;
    shard_range(total, world, q, &qf, &qc);
    if (qc) r = nccl().Send(src_rows + qf * S, qc * S, ncclUint32, q, c->comm, ctx->stream);        // q's columns, my rows: contiguous
    if (r == ncclSuccess && count) { r = nccl().Recv(stage + slot * count * S, count * S, ncclUint32, q, c->comm, ctx->stream); ++slot; }
  }
  ncclResult_t r2 = nccl().GroupEnd();
  if (r != ncclSuccess || r2 != ncclSuccess) st = set_err(ctx, NB200_ERR_CUDA, std::string("exchange rows->cols: ") + nccl().GetErrorString(r != ncclSuccess ? r : r2));
  slot = 0;
  for (int q = 0; q < world && st == NB200_OK; ++q) {
    if (q == rank || !count) continue;
    if (cudaMemcpy2DAsync(dst + (size_t)q * S, LEN * 4, stage + slot * count * S, S * 4, S * 4, count, cudaMemcpyDeviceToDevice, ctx->stream) != cudaSuccess) st = set_err(ctx, NB200_ERR_CUDA, "exchange: unpack");
    ++slot;
  }
  dfree(ctx, stage);
  return st;
}

// device all-gather of `words` u32 per rank into out[world * words] (rank order); in place allowed when mine == out + rank * words
nb200_status comm_all_gather_dev(nb200_ctx* ctx, const u32* mine, size_t words, u32* out) {
  Comm* c = (Comm*)ctx->comm;
  if (!c) { if (mine != out) NB_CUDA(ctx, cudaMemcpyAsync(out, mine, words * 4, cudaMemcpyDeviceToDevice, ctx->stream)); return NB200_OK; }
  NB_NCCL(ctx, nccl().AllGather(mine, out, words, ncclUint32, c->comm, ctx->stream));
  return NB200_OK;
}
// element-wise sum of u32 words over the ranks (used where exactly one rank contributes a non-zero word: gathers of owned values)
nb200_status comm_all_reduce_sum_host(nb200_ctx* ctx, u32* host, size_t words) {
  Comm* c = (Comm*)ctx->comm;
  if (!c || words == 0) return NB200_OK;
  u32* d = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d, words * 4));
  nb200_status st = NB200_OK;
  if (cudaMemcpyAsync(d, host, words * 4, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) st = set_err(ctx, NB200_ERR_CUDA, "all_reduce: h2d");
  if (st == NB200_OK) { ncclResult_t r = nccl().AllReduce(d, d, words, ncclUint32, ncclSum, c->comm, ctx->stream); if (r != ncclSuccess) st = set_err(ctx, NB200_ERR_CUDA, nccl().GetErrorString(r)); }
  if (st == NB200_OK && cudaMemcpyAsync(host, d, words * 4, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) st = set_err(ctx, NB200_ERR_CUDA, "all_reduce: d2h");
  if (st == NB200_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess) st = set_err(ctx, NB200_ERR_CUDA, "all_reduce: sync");
  dfree(ctx, d);
  return st;
}

nb200_status hash_top_layers(nb200_ctx* ctx, u32 k, const std::vector<TopCol>& top, std::vector<std::vector<uint8_t>>& layers) {
  for (u32 l = k; l-- > 0;) {
    layers[l].resize((size_t)32 << l);
    for (size_t i = 0; i < ((size_t)1 << l); ++i) {
      std::vector<u32> vals;
      for (auto& tc : top) if (tc.log == l) vals.push_back(tc.vals[i]);
      NB_TRY(nb200_hash_node(ctx->merkle_hash, &layers[l + 1][64 * i], &layers[l + 1][64 * i + 32], vals.data(), vals.size(), &layers[l][32 * i]));
    }
  }
  return NB200_OK;
}

}  // namespace nb
using namespace nb;

extern "C" {

size_t nb200_comm_unique_id_bytes(void) { return sizeof(ncclUniqueId); }

nb200_status nb200_comm_get_unique_id(uint8_t* id_out) {
  if (!id_out) return NB200_ERR_ARG;
  if (!nccl().ok) { global_err() = "NCCL is not available (libnccl.so.2 could not be loaded)"; return NB200_ERR_STATE; }
  ncclUniqueId id;
  if (nccl().GetUniqueId(&id) != ncclSuccess) { global_err() = "ncclGetUniqueId failed"; return NB200_ERR_CUDA; }
  memcpy(id_out, &id, sizeof(id));
  return NB200_OK;
}

nb200_status nb200_comm_init(nb200_ctx* ctx, int rank, int world, const uint8_t* unique_id) {
  if (!ctx || !unique_id) return NB200_ERR_ARG;
  NB_ARG(ctx, world >= 1 && rank >= 0 && rank < world && (world & (world - 1)) == 0, "comm_init: world must be a power of two, 0 <= rank < world");
  NB_ARG(ctx, nccl().ok, "comm_init: NCCL is not available (libnccl.so.2 could not be loaded)");
  comm_release(ctx);
  NB_CUDA(ctx, cudaSetDevice(ctx->device));
  Comm* c = new Comm();
  c->rank = rank; c->world = world;
  while ((1 << c->log_world) < world) ++c->log_world;
  ncclUniqueId id;
  memcpy(&id, unique_id, sizeof(id));
  ncclResult_t r = nccl().CommInitRank(&c->comm, world, id, rank);
  if (r != ncclSuccess) { delete c; return set_err(ctx, NB200_ERR_CUDA, std::string("ncclCommInitRank: ") + nccl().GetErrorString(r)); }
  ctx->comm = c;
  return NB200_OK;
}
void nb200_comm_destroy(nb200_ctx* ctx) { if (ctx) comm_release(ctx); }
int nb200_comm_rank(const nb200_ctx* ctx) { return (ctx && ctx->comm) ? ((Comm*)ctx->comm)->rank : 0; }
int nb200_comm_world(const nb200_ctx* ctx) { return (ctx && ctx->comm) ? ((Comm*)ctx->comm)->world : 1; }

nb200_status nb200_shard_range(size_t total_cols, int world, int rank, size_t* first, size_t* count) {
  if (!first || !count || world < 1 || rank < 0 || rank >= world) return NB200_ERR_ARG;
  shard_range(total_cols, world, rank, first, count);
  return NB200_OK;
}

// all-gather of small host blobs through the communicator (caps, claimed sums, sampled values): out = world x bytes
nb200_status nb200_comm_all_gather(nb200_ctx* ctx, const uint8_t* mine, size_t bytes, uint8_t* out) {
  if (!ctx || !mine || !out) return NB200_ERR_ARG;
  Comm* c = (Comm*)ctx->comm;
  if (!c) { memcpy(out, mine, bytes); return NB200_OK; }
  uint8_t* d = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d, bytes * (c->world + 1)));
  nb200_status st = NB200_OK;
  if (cudaMemcpyAsync(d, mine, bytes, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) st = set_err(ctx, NB200_ERR_CUDA, "all_gather: h2d");
  if (st == NB200_OK) { ncclResult_t r = nccl().AllGather(d, d + bytes, bytes, ncclUint8, c->comm, ctx->stream); if (r != ncclSuccess) st = set_err(ctx, NB200_ERR_CUDA, nccl().GetErrorString(r)); }
  if (st == NB200_OK && cudaMemcpyAsync(out, d + bytes, bytes * c->world, cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess) st = set_err(ctx, NB200_ERR_CUDA, "all_gather: d2h");
  if (st == NB200_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess) st = set_err(ctx, NB200_ERR_CUDA, "all_gather: sync");
  dfree(ctx, d);
  return st;
}

// One tree over all ranks.  shard_evals: this rank's columns [first, first+count) = nb200_shard_range(total_cols, world, rank) of the 2^n-row
// columns, finalized order.  replicated: batches of SMALLER columns that follow them in commitment order (the reference's extension
// components), passed identically on every rank.  Out: coeffs (this rank's columns), rows (total_cols x 2^(n+blow-k): every column, this rank's
// row slice of the LDE), the rank's sub-tree, the caps (world x 32 bytes, optional) and the root (the same on every rank).
nb200_status nb200_commit_sharded(nb200_ctx* ctx, const nb200_cols* shard_evals, size_t total_cols, uint32_t log_size, uint32_t log_blowup,
                                  const nb200_cols* const* replicated, size_t n_replicated,
                                  nb200_cols** coeffs_out, nb200_cols** rows_out, nb200_tree** subtree_out, uint8_t* caps_out, uint8_t root[32]) {
  if (!ctx || !coeffs_out || !rows_out || !subtree_out || !root || (n_replicated && !replicated)) return NB200_ERR_ARG;
  Comm* c = (Comm*)ctx->comm;
  NB_ARG(ctx, c != nullptr, "commit_sharded: nb200_comm_init first");
  const int world = c->world, rank = c->rank;
  const u32 k = (u32)c->log_world, n = log_size, m = n + log_blowup;
  NB_ARG(ctx, m >= k, "commit_sharded: fewer LDE rows than ranks");
  size_t first = 0, count = 0;
  shard_range(total_cols, world, rank, &first, &count);
  NB_ARG(ctx, (count == 0 && (!shard_evals || shard_evals->n_cols == 0)) || (shard_evals && shard_evals->n_cols == count && shard_evals->log_size == n),
         "commit_sharded: the column shard must be nb200_shard_range(total_cols, world, rank) columns of 2^log_size rows");
  for (size_t b = 0; b < n_replicated; ++b) NB_ARG(ctx, replicated[b] && replicated[b]->log_size < n, "commit_sharded: replicated batches must be smaller than the sharded columns");
  NB_TRY(twiddles_prepare(ctx, std::max<u32>(m, 1)));
  const size_t len = (size_t)1 << n, mlen = (size_t)1 << m, S = mlen >> k;   // S = rows per rank
  ColsPtr co, rows;
  NB_TRY(alloc(ctx, co, count, n));
  {
    ColsPtr lde;
    DevBuf pack;
    // 1. column-sharded transforms
    NB_TRY(alloc(ctx, lde, count, m));
    if (count) NB_TRY(commit_transforms(ctx, shard_evals->d, co->d, lde->d, nullptr, count, n, log_blowup));
    // 2. exchange: my columns' rows of peer q -> q; every peer's columns' rows of mine <- that peer
    NB_TRY(alloc(ctx, rows, total_cols, m - k));
    if (world > 1 && count) NB_TRY(alloc(ctx, pack, (size_t)(world - 1) * count * S));
    if (count) NB_CUDA(ctx, cudaMemcpy2DAsync(rows->d + first * S, S * 4, lde->d + (size_t)rank * S, mlen * 4, S * 4, count, cudaMemcpyDeviceToDevice, ctx->stream));
    if (world > 1) {
      size_t slot = 0;
      for (int q = 0; q < world; ++q) {
        if (q == rank || !count) continue;
        NB_CUDA(ctx, cudaMemcpy2DAsync(pack.p + slot * count * S, S * 4, lde->d + (size_t)q * S, mlen * 4, S * 4, count, cudaMemcpyDeviceToDevice, ctx->stream));
        ++slot;
      }
      NB_NCCL(ctx, nccl().GroupStart());
      slot = 0;
      for (int q = 0; q < world; ++q) {
        if (q == rank) continue;
        size_t qf = 0, qc = 0;
        shard_range(total_cols, world, q, &qf, &qc);
        if (count) { NB_NCCL(ctx, nccl().Send(pack.p + slot * count * S, count * S, ncclUint32, q, c->comm, ctx->stream)); ++slot; }
        if (qc) NB_NCCL(ctx, nccl().Recv(rows->d + qf * S, qc * S, ncclUint32, q, c->comm, ctx->stream));
      }
      NB_NCCL(ctx, nccl().GroupEnd());
    }
  }
  // 3. row-sharded sub-tree (+ the replicated smaller columns: each rank takes its slice; columns with fewer than `world` LDE rows
  //    live above the cap layer and are hashed on the host below)
  std::vector<ColRef> refs;
  for (size_t g = 0; g < total_cols; ++g) refs.push_back(ColRef{rows->col(g), m - k});
  std::vector<TopCol> top;
  std::vector<ColsPtr> small_lde;
  for (size_t b = 0; b < n_replicated; ++b) {
    const nb200_cols* ev = replicated[b];
    const u32 sl = ev->log_size + log_blowup;
    ColsPtr sco, sld;
    NB_TRY(alloc(ctx, sco, ev->n_cols, ev->log_size));
    NB_TRY(alloc(ctx, sld, ev->n_cols, sl));
    NB_TRY(commit_transforms(ctx, ev->d, sco->d, sld->d, nullptr, ev->n_cols, ev->log_size, log_blowup));
    for (size_t g = 0; g < ev->n_cols; ++g) {
      if (sl >= k) refs.push_back(ColRef{sld->col(g) + ((size_t)rank << (sl - k)), sl - k});
      else {
        TopCol t; t.log = sl; t.vals.resize((size_t)1 << sl);
        NB_CUDA(ctx, cudaMemcpyAsync(t.vals.data(), sld->col(g), t.vals.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
        top.push_back(std::move(t));
      }
    }
    small_lde.push_back(std::move(sco));
    small_lde.push_back(std::move(sld));
  }
  nb200_tree* sub_raw = nullptr;
  NB_TRY(merkle_commit(ctx, refs, &sub_raw));
  TreePtr sub(sub_raw);
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  // caps exchange + top k levels on the host (identical on every rank)
  std::vector<std::vector<uint8_t>> layers(k + 1);
  layers[k].resize((size_t)32 * world);
  NB_TRY(nb200_comm_all_gather(ctx, sub->root, 32, layers[k].data()));
  if (caps_out) memcpy(caps_out, layers[k].data(), layers[k].size());
  NB_TRY(hash_top_layers(ctx, k, top, layers));
  memcpy(root, layers[0].data(), 32);
  *coeffs_out = co.release(); *rows_out = rows.release(); *subtree_out = sub.release();
  return NB200_OK;
}

}  // extern "C"
