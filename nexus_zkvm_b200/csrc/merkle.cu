// Blake2s Merkle commitment of mixed-size column sets (MerkleOps<Blake2sMerkleHasher>::commit_on_layer,
// MerkleProver::commit / decommit).  Replaces the SimdBackend path reached from TreeBuilder::commit at
// nexus-zkvm prover/src/machine.rs:228,237,263 and from FRI layer commits inside stwo::prover::prove
// (machine.rs:286-290).
//
// node(layer l, row r) = H( child(2r) || child(2r+1) [if a deeper layer exists] || v_c[r] for every column c of
// length 2^l, in the stable length-descending order of the input ).  Two hash constructions are supported
// (DESIGN.md "parity risk switches"): 0 = chained raw Blake2s compressions from the zero state (what stwo's SIMD
// compress16 path computes), 1 = RFC 7693 Blake2s-256 of the byte string.
//
// Kernel: one thread per node.  A warp reads 32 consecutive rows of each column (128-byte coalesced segments);
// 16 column words form one 64-byte message block held in registers, so no transposition is ever materialised.
// The work is integer-ALU bound (~1.2k ops per 64-byte block), not HBM bound.
#include "pcs.h"
#include "blake2s.cuh"
#include <algorithm>

namespace nb {

template <int VARIANT>
__global__ void __launch_bounds__(128) merkle_layer_kernel(const uint4* __restrict__ prev, const u32* const* __restrict__ cols,
                                                            u32 n_cols, u32 log_size, uint4* __restrict__ out, const u32 one) {
  const size_t row = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= ((size_t)1 << log_size)) return;
  u32 h[8];
  u32 m[16];
  u64 t = 0;
  const u32 total_words = (prev ? 16u : 0u) + n_cols;
  const u64 total_bytes = (u64)total_words * 4;
  if (VARIANT == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) h[i] = 0;
  } else {
    b2s_init(h);
  }
  if (prev) {
    const uint4* p = prev + 4 * row;  // two 32-byte children = 4 x uint4
    uint4 a = __ldg(p), b = __ldg(p + 1), c = __ldg(p + 2), d = __ldg(p + 3);
    m[0] = a.x; m[1] = a.y; m[2] = a.z; m[3] = a.w; m[4] = b.x; m[5] = b.y; m[6] = b.z; m[7] = b.w;
    m[8] = c.x; m[9] = c.y; m[10] = c.z; m[11] = c.w; m[12] = d.x; m[13] = d.y; m[14] = d.z; m[15] = d.w;
    if (VARIANT == 0) {
      b2s_compress_fma(h, m, 0, 0, 0, 0, one);
    } else {
      t = 64;
      bool last = (n_cols == 0);
      b2s_compress_fma(h, m, (u32)t, 0, last ? 0xFFFFFFFFu : 0u, 0, one);
    }
  } else if (VARIANT == 1 && n_cols == 0) {
#pragma unroll
    for (int i = 0; i < 16; ++i) m[i] = 0;
    b2s_compress_fma(h, m, 0, 0, 0xFFFFFFFFu, 0, one);
  }
  for (u32 c0 = 0; c0 < n_cols; c0 += 16) {
    if (c0 + 16 <= n_cols) {
#pragma unroll
      for (int j = 0; j < 16; ++j) m[j] = __ldg(cols[c0 + j] + row);
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j) m[j] = (c0 + j < n_cols) ? __ldg(cols[c0 + j] + row) : 0u;
    }
    if (VARIANT == 0) {
      b2s_compress_fma(h, m, 0, 0, 0, 0, one);
    } else {
      bool last = (c0 + 16 >= n_cols);
      t = last ? total_bytes : t + 64;
      b2s_compress_fma(h, m, (u32)t, (u32)(t >> 32), last ? 0xFFFFFFFFu : 0u, 0, one);
    }
  }
  uint4* o = out + 2 * row;
  o[0] = make_uint4(h[0], h[1], h[2], h[3]);
  o[1] = make_uint4(h[4], h[5], h[6], h[7]);
}

// Incremental leaf hashing: the largest columns of a tree arrive from the host in chunks (commitment order, whole 16-column message
// blocks); each chunk continues the per-row Blake2s state kept in the tree's leaf layer, so that when the last chunk has been
// transformed only the inner layers are left.  The work hides in the shadow of the PCIe copy of the next chunk (api.cu).
// Same bytes as merkle_layer_kernel with prev == nullptr over all the columns at once.
template <int VARIANT>
__global__ void __launch_bounds__(128) merkle_leaf_absorb_kernel(uint4* __restrict__ state, const u32* __restrict__ cols, size_t stride, u32 n_cols,
                                                                 u32 log_size, u64 bytes_before, u64 total_bytes, int first, int final, const u32 one) {
  const size_t row = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= ((size_t)1 << log_size)) return;
  u32 h[8], m[16];
  uint4* st = state + 2 * row;
  if (first) {
    if (VARIANT == 0) {
#pragma unroll
      for (int i = 0; i < 8; ++i) h[i] = 0;
    } else {
      b2s_init(h);
    }
  } else {
    uint4 a = st[0], b = st[1];
    h[0] = a.x; h[1] = a.y; h[2] = a.z; h[3] = a.w; h[4] = b.x; h[5] = b.y; h[6] = b.z; h[7] = b.w;
  }
  for (u32 c0 = 0; c0 < n_cols; c0 += 16) {
    if (c0 + 16 <= n_cols) {
#pragma unroll
      for (int j = 0; j < 16; ++j) m[j] = __ldg(cols + (size_t)(c0 + j) * stride + row);
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j) m[j] = (c0 + j < n_cols) ? __ldg(cols + (size_t)(c0 + j) * stride + row) : 0u;
    }
    if (VARIANT == 0) {
      b2s_compress_fma(h, m, 0, 0, 0, 0, one);
    } else {
      const bool last = final && (c0 + 16 >= n_cols);
      const u64 t = last ? total_bytes : bytes_before + (u64)(c0 + 16) * 4;
      b2s_compress_fma(h, m, (u32)t, (u32)(t >> 32), last ? 0xFFFFFFFFu : 0u, 0, one);
    }
  }
  st[0] = make_uint4(h[0], h[1], h[2], h[3]);
  st[1] = make_uint4(h[4], h[5], h[6], h[7]);
}

static nb200_status tree_alloc(nb200_ctx* ctx, u32 max_log, nb200_tree** out) {
  NB_ARG(ctx, max_log <= 30, "merkle: column too large");
  nb200_tree* tree = new nb200_tree();
  tree->ctx = ctx;
  tree->max_log = max_log;
  size_t total_nodes = ((size_t)2 << max_log) - 1;
  cudaError_t e = dmalloc(ctx, (void**)&tree->d_pool, total_nodes * 32);
  if (e != cudaSuccess) { delete tree; return set_err(ctx, NB200_ERR_OOM, std::string("merkle pool: ") + cudaGetErrorString(e)); }
  tree->layer.resize(max_log + 1);
  size_t off = 0;
  for (u32 l = 0; l <= max_log; ++l) { tree->layer[l] = tree->d_pool + off * 32; off += (size_t)1 << l; }
  *out = tree;
  return NB200_OK;
}
nb200_status merkle_tree_alloc(nb200_ctx* ctx, u32 max_log, nb200_tree** out) { return tree_alloc(ctx, max_log, out); }

// absorb columns [cols_before, cols_before + n_cols) of the tree's `total_cols` leaf-level columns; n_cols must be a multiple of 16 unless final
nb200_status merkle_leaf_absorb(nb200_ctx* ctx, nb200_tree* tree, const u32* d_cols, size_t stride, size_t n_cols, size_t cols_before, size_t total_cols, bool final) {
  NB_ARG(ctx, tree && n_cols > 0 && cols_before % 16 == 0 && (final || n_cols % 16 == 0) && cols_before + n_cols <= total_cols, "merkle_leaf_absorb: chunking");
  const size_t rows = (size_t)1 << tree->max_log;
  const u32 threads = 128, blocks = (u32)((rows + threads - 1) / threads);
  uint4* st = (uint4*)tree->layer[tree->max_log];
  if (ctx->merkle_hash == 0)
    merkle_leaf_absorb_kernel<0><<<blocks, threads, 0, ctx->stream>>>(st, d_cols, stride, (u32)n_cols, tree->max_log, (u64)cols_before * 4, (u64)total_cols * 4, cols_before == 0, final, 1u);
  else
    merkle_leaf_absorb_kernel<1><<<blocks, threads, 0, ctx->stream>>>(st, d_cols, stride, (u32)n_cols, tree->max_log, (u64)cols_before * 4, (u64)total_cols * 4, cols_before == 0, final, 1u);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

// The last layers of a tree (no more columns to inject, <= 2^TAIL_LOG nodes) in ONE launch: a single CTA walks them with a barrier
// per layer.  A proof commits ~25 trees (4 trace trees + one per FRI layer); their small layers are pure launch latency otherwise.
static constexpr u32 TAIL_LOG = 9;
template <int VARIANT>
__global__ void __launch_bounds__(256) merkle_tail_kernel(uint4* __restrict__ pool, u32 top_log, const u32 one) {
  for (int l = (int)top_log; l >= 0; --l) {
    const uint4* prev = pool + 2 * (((size_t)1 << (l + 1)) - 1);   // layer l + 1 (written by the previous launch or iteration)
    uint4* outl = pool + 2 * (((size_t)1 << l) - 1);
    for (u32 row = threadIdx.x; row < (1u << l); row += blockDim.x) {
      u32 h[8], m[16];
      const uint4* p = prev + 4 * row;
      uint4 a = p[0], b = p[1], c = p[2], d = p[3];                 // plain loads: the data may come from this very kernel
      m[0] = a.x; m[1] = a.y; m[2] = a.z; m[3] = a.w; m[4] = b.x; m[5] = b.y; m[6] = b.z; m[7] = b.w;
      m[8] = c.x; m[9] = c.y; m[10] = c.z; m[11] = c.w; m[12] = d.x; m[13] = d.y; m[14] = d.z; m[15] = d.w;
      if (VARIANT == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) h[i] = 0;
        b2s_compress_fma(h, m, 0, 0, 0, 0, one);
      } else {
        b2s_init(h);
        b2s_compress_fma(h, m, 64u, 0, 0xFFFFFFFFu, 0, one);
      }
      outl[2 * row] = make_uint4(h[0], h[1], h[2], h[3]);
      outl[2 * row + 1] = make_uint4(h[4], h[5], h[6], h[7]);
    }
    __syncthreads();
  }
}

// pre_leaf: a tree from merkle_tree_alloc whose leaf layer already holds the hashes of ALL the largest columns (merkle_leaf_absorb);
// it is consumed (becomes *out, or is freed on failure)
nb200_status merkle_commit(nb200_ctx* ctx, const std::vector<ColRef>& cols_in, nb200_tree** out, nb200_tree* pre_leaf, bool root_to_host) {
  // stable sort by length, descending (MerkleProver::commit)
  std::vector<ColRef> cols = cols_in;
  std::stable_sort(cols.begin(), cols.end(), [](const ColRef& a, const ColRef& b) { return a.log_size > b.log_size; });
  u32 max_log = cols.empty() ? 0 : cols[0].log_size;
  nb200_tree* tree = pre_leaf;
  cudaError_t e = cudaSuccess;
  if (tree) {
    if (tree->max_log != max_log) { dfree(ctx, tree->d_pool); delete tree; return set_err(ctx, NB200_ERR_ARG, "merkle: precomputed leaf layer of the wrong size"); }
  } else {
    NB_TRY(tree_alloc(ctx, max_log, &tree));
  }
  // device array of column pointers in sorted order
  const u32** d_ptrs = nullptr;
  std::vector<const u32*> h_ptrs(cols.size());
  for (size_t i = 0; i < cols.size(); ++i) h_ptrs[i] = cols[i].d;
  if (!cols.empty()) {
    e = dmalloc(ctx, (void**)&d_ptrs, cols.size() * sizeof(u32*));
    if (e != cudaSuccess) { dfree(ctx, tree->d_pool); delete tree; return set_err(ctx, NB200_ERR_OOM, "merkle ptrs"); }
    e = cudaMemcpyAsync(d_ptrs, h_ptrs.data(), cols.size() * sizeof(u32*), cudaMemcpyHostToDevice, ctx->stream);
    if (e != cudaSuccess) { dfree(ctx, (void*)d_ptrs); dfree(ctx, tree->d_pool); delete tree; return set_err(ctx, NB200_ERR_CUDA, cudaGetErrorString(e)); }
  }
  size_t ci = 0;
  int l_start = (int)max_log;
  if (pre_leaf) {  // the leaf layer is done: skip its columns
    while (ci < cols.size() && cols[ci].log_size == max_log) ++ci;
    l_start = (int)max_log - 1;
  }
  for (int l = l_start; l >= 0; --l) {
    size_t first = ci;
    while (ci < cols.size() && cols[ci].log_size == (u32)l) ++ci;
    u32 n_here = (u32)(ci - first);
    if (n_here == 0 && ci == cols.size() && l < (int)max_log && l <= (int)TAIL_LOG) {
      // nothing but inner nodes from here to the root
      if (ctx->merkle_hash == 0) merkle_tail_kernel<0><<<1, 256, 0, ctx->stream>>>((uint4*)tree->d_pool, (u32)l, 1u);
      else merkle_tail_kernel<1><<<1, 256, 0, ctx->stream>>>((uint4*)tree->d_pool, (u32)l, 1u);
      ctx->launches += 1;
      break;
    }
    const uint4* prev = (l == (int)max_log) ? nullptr : (const uint4*)tree->layer[l + 1];
    size_t rows = (size_t)1 << l;
    u32 threads = 128;
    u32 blocks = (u32)((rows + threads - 1) / threads);
    if (ctx->merkle_hash == 0)
      merkle_layer_kernel<0><<<blocks, threads, 0, ctx->stream>>>(prev, d_ptrs + first, n_here, (u32)l, (uint4*)tree->layer[l], 1u);
    else
      merkle_layer_kernel<1><<<blocks, threads, 0, ctx->stream>>>(prev, d_ptrs + first, n_here, (u32)l, (uint4*)tree->layer[l], 1u);
    ctx->launches += 1;
  }
  e = cudaGetLastError();
  // (without the sync, h_ptrs may go: a copy from pageable host memory has been staged by the time cudaMemcpyAsync returns)
  if (root_to_host) {
    if (e == cudaSuccess) e = cudaMemcpyAsync(tree->root, tree->layer[0], 32, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  } else {
    memset(tree->root, 0, 32);
  }
  if (d_ptrs) dfree(ctx, (void*)d_ptrs);
  if (e != cudaSuccess) { dfree(ctx, tree->d_pool); delete tree; return set_err(ctx, NB200_ERR_CUDA, std::string("merkle commit: ") + cudaGetErrorString(e)); }
  *out = tree;
  return NB200_OK;
}

// ---- gathers used by decommit / query openings ----
__global__ void gather_u32_kernel(const u32* const* __restrict__ addrs, size_t n, u32* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = *addrs[i];
}
__global__ void gather_hash_kernel(const uint4* const* __restrict__ addrs, size_t n, uint4* __restrict__ out) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { out[2 * i] = addrs[i][0]; out[2 * i + 1] = addrs[i][1]; }
}

nb200_status gather_u32(nb200_ctx* ctx, const std::vector<const u32*>& addrs, u32* host_out) {
  if (addrs.empty()) return NB200_OK;
  const u32** d_a = nullptr; u32* d_o = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_a, addrs.size() * sizeof(u32*)));
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_o, addrs.size() * 4));
  NB_CUDA(ctx, cudaMemcpyAsync(d_a, addrs.data(), addrs.size() * sizeof(u32*), cudaMemcpyHostToDevice, ctx->stream));
  gather_u32_kernel<<<(u32)((addrs.size() + 255) / 256), 256, 0, ctx->stream>>>(d_a, addrs.size(), d_o);
  NB_LAUNCH_CHECK(ctx);
  NB_CUDA(ctx, cudaMemcpyAsync(host_out, d_o, addrs.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  dfree(ctx, (void*)d_a); dfree(ctx, (void*)d_o);
  return NB200_OK;
}
nb200_status gather_hash(nb200_ctx* ctx, const std::vector<const uint8_t*>& addrs, uint8_t* host_out) {
  if (addrs.empty()) return NB200_OK;
  const uint4** d_a = nullptr; uint4* d_o = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_a, addrs.size() * sizeof(void*)));
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d_o, addrs.size() * 32));
  NB_CUDA(ctx, cudaMemcpyAsync(d_a, addrs.data(), addrs.size() * sizeof(void*), cudaMemcpyHostToDevice, ctx->stream));
  gather_hash_kernel<<<(u32)((addrs.size() + 255) / 256), 256, 0, ctx->stream>>>(d_a, addrs.size(), d_o);
  NB_LAUNCH_CHECK(ctx);
  NB_CUDA(ctx, cudaMemcpyAsync(host_out, d_o, addrs.size() * 32, cudaMemcpyDeviceToHost, ctx->stream));
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  dfree(ctx, (void*)d_a); dfree(ctx, (void*)d_o);
  return NB200_OK;
}

// Hashes and words from anywhere in device memory in ONE round trip: one upload of the address list, one launch, one copy back, one sync.
// Thread i < n_hash copies the 32-byte node at hash_addrs[i]; the threads after it copy one word each.
__global__ void gather_batch_kernel(const void* const* __restrict__ addrs, size_t n_hash, size_t n_val, uint4* __restrict__ hashes_out, u32* __restrict__ vals_out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_hash) {
    const uint4* a = (const uint4*)addrs[i];
    hashes_out[2 * i] = a[0]; hashes_out[2 * i + 1] = a[1];
  } else if (i < n_hash + n_val) {
    vals_out[i - n_hash] = *(const u32*)addrs[i];
  }
}

nb200_status gather_batch(nb200_ctx* ctx, const std::vector<const uint8_t*>& hash_addrs, const std::vector<const u32*>& val_addrs, uint8_t* hashes_out, u32* vals_out) {
  const size_t nh = hash_addrs.size(), nv = val_addrs.size(), n = nh + nv;
  if (n == 0) return NB200_OK;
  std::vector<const void*> addrs(n);
  std::copy(hash_addrs.begin(), hash_addrs.end(), addrs.begin());
  std::copy(val_addrs.begin(), val_addrs.end(), addrs.begin() + nh);
  // one device buffer: the hashes (32 bytes each, 16-byte aligned for the vector stores), the words, then the addresses (8-byte aligned)
  const size_t out_bytes = nh * 32 + nv * 4, a_off = (out_bytes + 7) & ~(size_t)7;
  uint8_t* d = nullptr;
  NB_CUDA(ctx, dmalloc(ctx, (void**)&d, a_off + n * sizeof(void*)));
  uint8_t* d_o = d;
  const void** d_a = (const void**)(d + a_off);
  std::vector<uint8_t> host(out_bytes);
  cudaError_t e = cudaMemcpyAsync(d_a, addrs.data(), n * sizeof(void*), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) {
    gather_batch_kernel<<<(u32)((n + 255) / 256), 256, 0, ctx->stream>>>(d_a, nh, nv, (uint4*)d_o, (u32*)(d_o + nh * 32));
    ctx->launches += 1;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(host.data(), d_o, out_bytes, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  dfree(ctx, d);
  if (e != cudaSuccess) return set_err(ctx, NB200_ERR_CUDA, std::string("gather: ") + cudaGetErrorString(e));
  if (nh) memcpy(hashes_out, host.data(), nh * 32);
  if (nv) memcpy(vals_out, host.data() + nh * 32, nv * 4);
  return NB200_OK;
}

// MerkleProver::decommit (stwo prover/vcs/prover.rs), the walk alone: which column values (in walk order, each marked queried or
// witness) and which nodes of the layers below each layer (the hash witness, in order) the decommitment names.
void merkle_decommit_plan(u32 max_log, const std::vector<u32>& col_logs, const std::vector<std::pair<u32, std::vector<u64>>>& queries, DecommitPlan& plan) {
  plan = DecommitPlan();
  std::vector<u32> order(col_logs.size());   // stable length-descending order of the columns, as committed
  for (size_t i = 0; i < order.size(); ++i) order[i] = (u32)i;
  std::stable_sort(order.begin(), order.end(), [&](u32 a, u32 b) { return col_logs[a] > col_logs[b]; });
  size_t ci = 0;
  std::vector<u64> last_layer_queries;
  for (int l = (int)max_log; l >= 0; --l) {
    std::vector<u64> layer_total;
    size_t first = ci;
    while (ci < order.size() && col_logs[order[ci]] == (u32)l) ++ci;
    const bool has_prev = (u32)l < max_log;
    const std::vector<u64>* lq = nullptr;
    for (auto& q : queries) if (q.first == (u32)l) lq = &q.second;
    size_t pq = 0, cq = 0;
    size_t nlq = lq ? lq->size() : 0;
    while (true) {
      bool has_p = pq < last_layer_queries.size(), has_c = cq < nlq;
      if (!has_p && !has_c) break;
      u64 node;
      if (has_p && has_c) node = std::min(last_layer_queries[pq] / 2, (*lq)[cq]);
      else if (has_p) node = last_layer_queries[pq] / 2;
      else node = (*lq)[cq];
      if (has_prev) {
        if (pq < last_layer_queries.size() && last_layer_queries[pq] == 2 * node) ++pq;
        else plan.hashes.push_back({(u32)l + 1, 2 * node});
        if (pq < last_layer_queries.size() && last_layer_queries[pq] == 2 * node + 1) ++pq;
        else plan.hashes.push_back({(u32)l + 1, 2 * node + 1});
      }
      bool queried = cq < nlq && (*lq)[cq] == node;
      if (queried) ++cq;
      for (size_t c = first; c < ci; ++c) { plan.vals.push_back({order[c], node}); plan.val_is_query.push_back(queried ? 1 : 0); }
      layer_total.push_back(node);
    }
    last_layer_queries.swap(layer_total);
  }
}

// the device addresses a plan names in `tree` and `cols` (the caller's column order), appended to the two lists
void merkle_decommit_addrs(const DecommitPlan& plan, const nb200_tree* tree, const std::vector<ColRef>& cols,
                           std::vector<const uint8_t*>& hash_addrs, std::vector<const u32*>& val_addrs) {
  for (auto& h : plan.hashes) hash_addrs.push_back(tree->layer[h.first] + 32 * h.second);
  for (auto& v : plan.vals) val_addrs.push_back(cols[v.first].d + v.second);
}

// the gathered hashes and words of one plan, in its order, sorted into the decommitment's three lists
void merkle_decommit_fill(const DecommitPlan& plan, const uint8_t* hashes, const u32* vals,
                          std::vector<u32>& queried_values, std::vector<uint8_t>& hash_witness, std::vector<u32>& column_witness) {
  hash_witness.assign(hashes, hashes + plan.hashes.size() * 32);
  queried_values.clear(); column_witness.clear();
  for (size_t i = 0; i < plan.vals.size(); ++i) (plan.val_is_query[i] ? queried_values : column_witness).push_back(vals[i]);
}

// MerkleProver::decommit of one tree: plan, one gather, fill
nb200_status merkle_decommit(nb200_ctx* ctx, const nb200_tree* tree, const std::vector<ColRef>& cols,
                             const std::vector<std::pair<u32, std::vector<u64>>>& queries,
                             std::vector<u32>& queried_values, std::vector<uint8_t>& hash_witness, std::vector<u32>& column_witness) {
  std::vector<u32> logs(cols.size());
  for (size_t i = 0; i < cols.size(); ++i) logs[i] = cols[i].log_size;
  DecommitPlan plan;
  merkle_decommit_plan(tree->max_log, logs, queries, plan);
  std::vector<const uint8_t*> ha;
  std::vector<const u32*> va;
  merkle_decommit_addrs(plan, tree, cols, ha, va);
  std::vector<uint8_t> hashes(ha.size() * 32);
  std::vector<u32> vals(va.size());
  NB_TRY(gather_batch(ctx, ha, va, hashes.data(), vals.data()));
  merkle_decommit_fill(plan, hashes.data(), vals.data(), queried_values, hash_witness, column_witness);
  return NB200_OK;
}

}  // namespace nb
