// Proving orchestrator: CommitmentSchemeProver / TreeBuilder and stwo::prover::prove + prove_values, FRI prover,
// proof assembly and postcard serialisation — the host logic that sequences the CUDA kernels between Fiat-Shamir
// round trips.  Replaces everything the reference reaches through
//   CommitmentSchemeProver::<SimdBackend, Blake2sMerkleChannel>::new / tree_builder / commit   prover/src/machine.rs:202-263
//   stwo::prover::prove::<SimdBackend, Blake2sMerkleChannel>(components, channel, scheme)         prover/src/machine.rs:286-290
// (stwo @0790eba prover/mod.rs, prover/pcs/mod.rs, prover/fri.rs, prover/air/accumulation.rs, core/proof.rs).
// The transcript (channel) is host-side, except between FRI's inner layers (device_channel.cuh); every data-parallel step is a kernel
// launch on ctx->stream.
#include "pcs.h"
#include "host_channel.h"
#include "circle_host.h"
#include <algorithm>
#include <map>
#include <set>
#include <memory>
#include <cstring>

struct nb200_channel { nb::HostChannel ch; };
struct nb200_air {
  nb::AirProgram prog;
  // per kind and component, compiled on first use (NVRTC); empty kernel = bytecode interpreter
  std::vector<nb::JitKernel> jit[nb::JIT_KINDS];
  std::vector<std::vector<nb::AirFrac>> fracs;   // every component's fractions as tables, lookups or neither (air_lookup_tables)
  ~nb200_air() { for (auto& v : jit) for (auto& j : v) nb::jit_release(j); }
};

namespace nb {

struct SchemeTree {
  std::vector<ColsPtr> coeffs, ldes;      // batches, commitment order
  std::vector<ColsPtr> half_ext;          // per batch or empty: the polynomials on the first half of CanonicCoset(lde log + 1).circle_domain(),
                                          // precomputed by the sharded commit when the scheme was told the AIR's degree bound (see component_quotients)
  struct ColLoc { u32 batch, idx, log; };
  std::vector<ColLoc> cols;               // global column index -> (batch, index in batch, polynomial log size)
  TreePtr merkle;
  const u32* coeff_ptr(size_t g) const { return coeffs[cols[g].batch]->col(cols[g].idx); }
  const u32* lde_ptr(size_t g) const { return ldes[cols[g].batch]->col(cols[g].idx); }
  // ---- one proof over N GPUs (nb200_scheme_commit_sharded): the tree's FIRST `big_total` columns (2^big_log rows each: the main component's)
  // are sharded — this rank holds the coefficients of its own column range and, for ALL of them, its slice of the LDE rows (and of the D2 rows);
  // the smaller columns that follow are replicated in coeffs / ldes / half_ext as usual.  cols[g].batch == BIG marks a sharded column.
  static constexpr u32 BIG = 0xffffffffu;
  bool sharded = false;
  int rank = 0;
  size_t big_total = 0, own_first = 0, own_count = 0;
  u32 big_log = 0;                              // polynomial log size n; LDE log m = n + blow-up; rows per rank S = 2^m / world
  ColsPtr big_coeffs;                           // own_count x 2^n
  ColsPtr big_rows;                             // big_total x S: LDE rows [rank * S, (rank + 1) * S)
  ColsPtr big_rows_hx;                          // big_total x S: the same rows of the half-coset extension D2 (or empty)
  ColsPtr big_eval_rows;                        // big_total x 2^n / world: trace-domain rows (kept for the interaction trace of trees 0 / 1)
  std::map<size_t, ColsPtr> full_lde, full_hx;  // columns read at a row offset: full LDE / D2 copies on every rank
  std::vector<std::vector<uint8_t>> top_layers; // host copies of the Merkle layers 0..k (layer k = the world caps); `merkle` is this rank's sub-tree
  // sharded column idx on the LDE domain / on D2, indexed by the GLOBAL row: only this rank's rows [row0(), row0() + S) may be read
  size_t row0() const { return (size_t)rank << big_rows->log_size; }
  const u32* lde_rows(size_t idx) const { return big_rows->col(idx) - row0(); }
  const u32* hx_rows(size_t idx) const { return big_rows_hx->col(idx) - row0(); }
};

}  // namespace nb

struct nb200_scheme {
  nb200_ctx* ctx = nullptr;
  uint32_t pow_bits = 5, log_blowup = 1, log_last = 0, n_queries = 3;  // PcsConfig::default() [risk A.4]
  std::vector<nb::SchemeTree> trees;
  uint32_t hint_log_expand = 0;  // nb200_scheme_set_constraint_log_degree: 0 = unknown
};

namespace nb {

nb200_status gather_hash(nb200_ctx* ctx, const std::vector<const uint8_t*>& addrs, uint8_t* host_out);

// the parameter table (QM31 values, 16 bytes each) in device memory, for the constraint and LogUp kernels
static nb200_status upload_params(nb200_ctx* ctx, const void* params, size_t n_params, DevBuf& out) {
  NB_TRY(alloc(ctx, out, std::max<size_t>(n_params, 1) * 4));
  if (n_params) NB_CUDA(ctx, cudaMemcpyAsync(out.p, params, n_params * 16, cudaMemcpyHostToDevice, ctx->stream));
  return NB200_OK;
}

// The component's specialised kernel, compiled on first use; nullptr = none.
// `interp_fallback`: the caller can run the bytecode interpreter, so only the kinds jit_specialised names are compiled and a failed
// compile is only logged (NB200_TRACE).  The sharded row kernels, the constraint check and the count have no interpreter: they try every
// program and reject a nullptr.
static const JitKernel* ensure_jit(nb200_ctx* ctx, nb200_air* air_h, size_t comp_idx, JitKind kind, bool interp_fallback) {
  std::vector<JitKernel>& v = air_h->jit[kind];
  if (v.size() != air_h->prog.comps.size()) v.resize(air_h->prog.comps.size());
  JitKernel& jk = v[comp_idx];
  if (!jk.tried) {
    jk.tried = true;
    const AirComponent& c = air_h->prog.comps[comp_idx];
    if ((!interp_fallback || jit_specialised(kind, c, air_h->fracs[comp_idx])) && jit_enabled()) {
      nb200_status st = jit_compile(ctx, kind, c, air_h->fracs[comp_idx], &jk);
      if (st != NB200_OK) jk.err = ctx->err;   // kept with the kernel: a later call that finds it missing reports why
      if (interp_fallback) {
        static const char* what[] = {"component", "logup program", "component (D2)", "constraint check"};
        if (st != NB200_OK && ctx->trace) fprintf(stderr, "[nb200] jit unavailable for %s: %s\n", what[kind], ctx->err.c_str());
        trace_mark(ctx, kind == JIT_LOGUP ? "jit: compile logup (one-time)" : "jit: compile (one-time)");
      }
    }
  }
  return jk.kernel ? &jk : nullptr;
}

static nb200_status finish_tree(nb200_ctx* ctx, SchemeTree& t, HostChannel& ch, nb200_tree* pre_leaf = nullptr) {
  std::vector<ColRef> refs;
  t.cols.clear();
  for (size_t b = 0; b < t.ldes.size(); ++b)
    for (size_t c = 0; c < t.ldes[b]->n_cols; ++c) {
      refs.push_back(ColRef{t.ldes[b]->col(c), t.ldes[b]->log_size});
      t.cols.push_back(SchemeTree::ColLoc{(u32)b, (u32)c, t.coeffs[b]->log_size});
    }
  nb200_tree* tree = nullptr;
  NB_TRY(merkle_commit(ctx, refs, &tree, pre_leaf));
  t.merkle.reset(tree);
  ch.mix_root(t.merkle->root);
  return NB200_OK;
}

// TreeBuilder::extend_evals + commit
nb200_status scheme_commit_evals(nb200_scheme* s, const nb200_cols* const* evals, size_t n, HostChannel& ch, uint8_t root[32]) {
  nb200_ctx* ctx = s->ctx;
  u32 max_log = 0;
  for (size_t b = 0; b < n; ++b) max_log = std::max(max_log, evals[b]->log_size + s->log_blowup);
  if (max_log >= 1) NB_TRY(twiddles_prepare(ctx, max_log));
  trace_mark(ctx, nullptr);
  SchemeTree t;
  // (the half coset D2 is not evaluated here: the quotient step extends only the few columns its high-degree constraints read)
  for (size_t b = 0; b < n; ++b) {
    ColsPtr co, lde;
    NB_TRY(alloc(ctx, co, evals[b]->n_cols, evals[b]->log_size));
    NB_TRY(alloc(ctx, lde, evals[b]->n_cols, evals[b]->log_size + s->log_blowup));
    NB_TRY(commit_transforms(ctx, evals[b]->d, co->d, lde->d, nullptr, co->n_cols, co->log_size, s->log_blowup));
    t.coeffs.push_back(std::move(co));
    t.ldes.push_back(std::move(lde));
  }
  trace_mark(ctx, "commit: ifft+lde");
  NB_TRY(finish_tree(ctx, t, ch));
  trace_mark(ctx, "commit: merkle");
  if (root) memcpy(root, t.merkle->root, 32);
  s->trees.push_back(std::move(t));
  return NB200_OK;
}

// The same, from HOST columns (the reference hands over host `Vec<BaseColumn>`s, trace_builder.rs:156-164): upload,
// finalize_columns on the device when `coset_order`, transforms — pipelined chunk by chunk — then Merkle + mix_root.
// On failure nothing is handed to the caller (every evals_out[b] is nullptr) and nothing stays allocated.
nb200_status scheme_commit_host(nb200_scheme* s, const void* const* host, const u32* elem_bytes, const size_t* n_cols, const u32* log_sizes, size_t n, int coset_order,
                                HostChannel& ch, uint8_t root[32], nb200_cols** evals_out) {
  nb200_ctx* ctx = s->ctx;
  for (size_t b = 0; b < n; ++b) evals_out[b] = nullptr;
  u32 max_log = 0;
  for (size_t b = 0; b < n; ++b) max_log = std::max(max_log, log_sizes[b] + s->log_blowup);
  if (max_log >= 1) NB_TRY(twiddles_prepare(ctx, max_log));
  trace_mark(ctx, nullptr);
  SchemeTree t;
  std::vector<ColsPtr> evals(n);
  // leaf hashes are continued chunk by chunk under the PCIe copy when one batch holds all the largest columns
  LeafSink sink;
  TreePtr pre_leaf;
  const long leaf_batch = leaf_sink_batch(n_cols, log_sizes, n);
  if (leaf_batch >= 0) {
    NB_TRY(merkle_tree_alloc(ctx, max_log, &sink.tree));
    pre_leaf.reset(sink.tree);
  }
  for (size_t b = 0; b < n; ++b) {
    ColsPtr co, lde;
    NB_TRY(alloc(ctx, evals[b], n_cols[b], log_sizes[b]));
    NB_TRY(alloc(ctx, co, n_cols[b], log_sizes[b]));
    NB_TRY(alloc(ctx, lde, n_cols[b], log_sizes[b] + s->log_blowup));
    NB_TRY(upload_transform_pipelined(ctx, host[b], n_cols[b], log_sizes[b], coset_order, s->log_blowup, evals[b]->d, co->d, lde->d, nullptr,
                                      (long)b == leaf_batch ? &sink : nullptr, elem_bytes ? elem_bytes[b] : 4u));
    t.coeffs.push_back(std::move(co));
    t.ldes.push_back(std::move(lde));
  }
  trace_mark(ctx, "commit(host): h2d+ifft+lde");
  NB_TRY(finish_tree(ctx, t, ch, pre_leaf.release()));   // merkle_commit consumes the leaf layer, also when it fails
  trace_mark(ctx, "commit: merkle");
  if (root) memcpy(root, t.merkle->root, 32);
  s->trees.push_back(std::move(t));
  for (size_t b = 0; b < n; ++b) evals_out[b] = evals[b].release();
  return NB200_OK;
}

// ======================================================================================================================================
// One PROOF over N GPUs (SURVEY §8e, BASELINE configs[3]).  Every rank calls the same sequence; transcript, roots and proof bytes are
// identical on all ranks and identical to the single-GPU proof.  Sharding: the main component's columns (the tree's first, largest batch) are
// column-sharded for the transforms and OODS evaluation and row-sharded for hashing, constraint rows and DEEP quotients, with one NVLink
// exchange per committed tree and evaluation set (comm.cu); the few columns read at a row offset (`Pc`, `IsPadding`, the last LogUp column) are
// replicated; everything small (extension components, composition tree, FRI) is computed redundantly on every rank.
// ======================================================================================================================================
// a column the constraints read at a row offset: every rank needs all of it — the all-gather of its row slices (contiguous row ranges in rank order)
static nb200_status replicate_from_rows(nb200_ctx* ctx, const nb200_cols* rows, size_t g, u32 log_len, ColsPtr& out) {
  NB_TRY(alloc(ctx, out, 1, log_len));
  return comm_all_gather_dev(ctx, rows->col(g), (size_t)1 << rows->log_size, out->d);
}

nb200_status scheme_commit_sharded(nb200_scheme* s, const nb200_cols* big_shard, size_t total_big, u32 n, const nb200_cols* const* small, size_t n_small,
                                   const u32* replicate, size_t n_replicate, int keep_eval_rows, HostChannel& ch, uint8_t root[32]) {
  nb200_ctx* ctx = s->ctx;
  const int world = comm_world(ctx), rank = comm_rank(ctx);
  const u32 k = (u32)comm_log_world(ctx), bl = s->log_blowup, m = n + bl;
  NB_ARG(ctx, m >= k + 10, "commit_sharded: the sharded columns need at least 1024 LDE rows per rank");
  for (size_t b = 0; b < n_small; ++b) NB_ARG(ctx, small[b] && small[b]->log_size < n, "commit_sharded: replicated batches must be smaller than the sharded columns");
  size_t first = 0, count = 0;
  comm_shard_range(total_big, world, rank, &first, &count);
  NB_ARG(ctx, (count == 0 && (!big_shard || big_shard->n_cols == 0)) || (big_shard && big_shard->n_cols == count && big_shard->log_size == n),
         "commit_sharded: the column shard must be nb200_shard_range(total, world, rank) columns of 2^log_size rows");
  const bool want_hx = (s->hint_log_expand == bl + 1);
  NB_TRY(twiddles_prepare(ctx, want_hx ? m + 1 : m));
  trace_mark(ctx, nullptr);
  SchemeTree t;
  t.sharded = true; t.rank = rank; t.big_total = total_big; t.own_first = first; t.own_count = count; t.big_log = n;
  // 1-3. column-sharded transforms of this rank's columns, pipelined with the exchange: the columns are transformed in `nch` chunks on ctx->stream;
  // as soon as a chunk is done its row slices (LDE, D2, trace rows) travel to their owners on the communicator's side stream while the next
  // chunk is being transformed.  Every rank uses the same chunk count, so the grouped send / recv pairs of chunk j match.
  NB_TRY(alloc(ctx, t.big_coeffs, count, n));
  {
    ColsPtr lde_full, hx_full;
    NB_TRY(alloc(ctx, lde_full, count, m));
    if (want_hx) NB_TRY(alloc(ctx, hx_full, count, m));
    // the row-slice buffers: in the symmetric peer heap when CUDA IPC links the ranks (the owners of the columns then write their rows straight into
    // them over NVLink with the copy engines), else ordinary allocations filled by grouped ncclSend / ncclRecv
    PeerBuf pb_rows, pb_hx, pb_ev;
    NB_TRY(peer_alloc(ctx, s, total_big << (m - k), &pb_rows));
    const bool peer = pb_rows.d != nullptr;
    if (peer) {
      nb200_cols* c = nullptr;
      NB_TRY(nb200_cols_from_device(ctx, pb_rows.d, total_big, m - k, &c));
      t.big_rows.reset(c);
      if (want_hx) {
        NB_TRY(peer_alloc(ctx, s, total_big << (m - k), &pb_hx));
        NB_ARG(ctx, pb_hx.d, "peer heap");
        NB_TRY(nb200_cols_from_device(ctx, pb_hx.d, total_big, m - k, &c));
        t.big_rows_hx.reset(c);
      }
      if (keep_eval_rows) {
        NB_TRY(peer_alloc(ctx, s, total_big << (n - k), &pb_ev));
        NB_ARG(ctx, pb_ev.d, "peer heap");
        NB_TRY(nb200_cols_from_device(ctx, pb_ev.d, total_big, n - k, &c));
        t.big_eval_rows.reset(c);
      }
      NB_TRY(comm_barrier_stream(ctx));     // every rank has reached this commit: nobody still reads what these buffers held in the previous proof
    } else {
      NB_TRY(alloc(ctx, t.big_rows, total_big, m - k));
      if (want_hx) NB_TRY(alloc(ctx, t.big_rows_hx, total_big, m - k));
      if (keep_eval_rows) NB_TRY(alloc(ctx, t.big_eval_rows, total_big, n - k));
    }
    static const int xchg_chunks = [] { const char* e = getenv("NB200_XCHG_CHUNKS"); int v = e ? atoi(e) : 4; return v < 1 ? 1 : (v > 64 ? 64 : v); }();
    // with the peer heap and a fused-pipeline size the LAST PASS of the transforms stores every finished tile into its owner's row-slice buffer (NVLink
    // peer stores from the kernel: compute and exchange are one launch); otherwise the columns are transformed in chunks and re-sharded by copies /
    // NCCL on the side stream while the next chunk is transformed
    const bool scatter_ok = peer && commit_transforms_can_scatter(n, bl, m - k, world);
    RowScatter sc;
    if (scatter_ok) {
      sc.world = world; sc.log_slice = m - k; sc.col0 = first;
      for (int q = 0; q < world; ++q) { sc.lde_rows[q] = peer_ptr(ctx, pb_rows, q); sc.hx_rows[q] = want_hx ? peer_ptr(ctx, pb_hx, q) : nullptr; }
    }
    const int nch = (!scatter_ok && world > 1 && total_big / world >= 64) ? xchg_chunks : 1;
    DevBuf pack;
    {
      size_t maxc = 0;
      for (int r = 0; r < world; ++r) { size_t f, c; comm_shard_range(total_big, world, r, &f, &c); maxc = std::max(maxc, c); }
      const size_t chunk_cols = (maxc + nch - 1) / nch + 1;
      if (world > 1 && !peer) NB_TRY(alloc(ctx, pack, (size_t)(world - 1) * chunk_cols << (m - k)));
    }
    cudaStream_t xs = comm_side_stream(ctx);
    // Until the exchange is joined and the stream drained, the side stream may still read pack, lde_full and hx_full. On an error return this
    // guard, destroyed before them, joins it and drains the stream so that their memory is not freed under a running copy.
    struct JoinOnError {
      nb200_ctx* ctx; bool armed = true;
      ~JoinOnError() { if (armed) { comm_join(ctx); cudaStreamSynchronize(ctx->stream); } }
    } join{ctx};
    for (int j = 0; j < nch; ++j) {
      const size_t c0 = count * j / nch, c1 = count * (j + 1) / nch;
      bool scattered = false;
      if (c1 > c0) {
        RowScatter scj = sc;
        scj.col0 = first + c0;
        NB_TRY(commit_transforms(ctx, big_shard->d + (c0 << n), t.big_coeffs->d + (c0 << n), lde_full->d + (c0 << m), hx_full ? hx_full->d + (c0 << m) : nullptr, c1 - c0, n, bl,
                                 scatter_ok ? &scj : nullptr, &scattered));
        if (scatter_ok && !scattered) return set_err(ctx, NB200_ERR_STATE, "commit_sharded: the fused pipeline refused the row scatter");
      }
      NB_TRY(comm_fork(ctx));
      if (peer) {
        if (!scatter_ok) {
          NB_TRY(peer_cols_to_rows_chunk(ctx, xs, lde_full->d, total_big, (size_t)1 << m, pb_rows, j, nch));
          if (want_hx) NB_TRY(peer_cols_to_rows_chunk(ctx, xs, hx_full->d, total_big, (size_t)1 << m, pb_hx, j, nch));
        }
        if (keep_eval_rows && count) NB_TRY(peer_cols_to_rows_chunk(ctx, xs, big_shard->d, total_big, (size_t)1 << n, pb_ev, j, nch));
      } else {
        NB_TRY(exchange_cols_to_rows_chunk(ctx, xs, lde_full->d, total_big, (size_t)1 << m, t.big_rows->d, pack.p, j, nch));
        if (want_hx) NB_TRY(exchange_cols_to_rows_chunk(ctx, xs, hx_full->d, total_big, (size_t)1 << m, t.big_rows_hx->d, pack.p, j, nch));
        if (keep_eval_rows) NB_TRY(exchange_cols_to_rows_chunk(ctx, xs, count ? big_shard->d : nullptr, total_big, (size_t)1 << n, t.big_eval_rows->d, pack.p, j, nch));
      }
    }
    trace_mark(ctx, "sharded commit: ifft+lde (own columns; exchange overlapped)");
    NB_TRY(comm_join(ctx));
    if (peer) NB_TRY(comm_barrier_stream(ctx));   // my copies are done AND (the barrier completing) so are everybody's into my buffers
    // columns that constraints read at a row offset: full copies everywhere
    for (size_t i = 0; i < n_replicate; ++i) {
      const size_t g = replicate[i];
      NB_ARG(ctx, g < total_big, "commit_sharded: replicate index out of range");
      if (t.full_lde.count(g)) continue;
      NB_TRY(replicate_from_rows(ctx, t.big_rows.get(), g, m, t.full_lde[g]));
      if (want_hx) NB_TRY(replicate_from_rows(ctx, t.big_rows_hx.get(), g, m, t.full_hx[g]));
    }
    NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    join.armed = false;
  }
  trace_mark(ctx, "sharded commit: exchange tail + replicated columns");
  // 4. the smaller batches: computed in full by every rank
  for (size_t b = 0; b < n_small; ++b) {
    ColsPtr co, lde, hx;
    NB_TRY(alloc(ctx, co, small[b]->n_cols, small[b]->log_size));
    NB_TRY(alloc(ctx, lde, small[b]->n_cols, small[b]->log_size + bl));
    if (want_hx && lde->log_size > 8) NB_TRY(alloc(ctx, hx, small[b]->n_cols, lde->log_size));
    NB_TRY(commit_transforms(ctx, small[b]->d, co->d, lde->d, hx ? hx->d : nullptr, co->n_cols, co->log_size, bl));
    t.coeffs.push_back(std::move(co));
    t.ldes.push_back(std::move(lde));
    t.half_ext.push_back(std::move(hx));
  }
  // 5. row-sharded sub-tree, caps, top levels
  std::vector<ColRef> refs;
  t.cols.clear();
  for (size_t g = 0; g < total_big; ++g) { refs.push_back(ColRef{t.big_rows->col(g), m - k}); t.cols.push_back(SchemeTree::ColLoc{SchemeTree::BIG, (u32)g, n}); }
  std::vector<TopCol> top;
  for (size_t b = 0; b < t.ldes.size(); ++b)
    for (size_t c2 = 0; c2 < t.ldes[b]->n_cols; ++c2) {
      const u32 sl = t.ldes[b]->log_size;
      t.cols.push_back(SchemeTree::ColLoc{(u32)b, (u32)c2, t.coeffs[b]->log_size});
      if (sl >= k) refs.push_back(ColRef{t.ldes[b]->col(c2) + ((size_t)rank << (sl - k)), sl - k});
      else {
        TopCol tc; tc.log = sl; tc.vals.resize((size_t)1 << sl);
        NB_CUDA(ctx, cudaMemcpyAsync(tc.vals.data(), t.ldes[b]->col(c2), tc.vals.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
        top.push_back(std::move(tc));
      }
    }
  nb200_tree* sub = nullptr;
  NB_TRY(merkle_commit(ctx, refs, &sub));
  t.merkle.reset(sub);
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  t.top_layers.assign(k + 1, {});
  t.top_layers[k].resize((size_t)32 << k);
  {
    DevBuf d;
    NB_TRY(alloc(ctx, d, (size_t)8 * (world + 1)));
    NB_CUDA(ctx, cudaMemcpyAsync(d.p, t.merkle->root, 32, cudaMemcpyHostToDevice, ctx->stream));
    NB_TRY(comm_all_gather_dev(ctx, d.p, 8, d.p + 8));
    NB_CUDA(ctx, cudaMemcpyAsync(t.top_layers[k].data(), d.p + 8, (size_t)32 * world, cudaMemcpyDeviceToHost, ctx->stream));
    NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  NB_TRY(hash_top_layers(ctx, k, top, t.top_layers));
  memcpy(t.merkle->root, t.top_layers[0].data(), 32);   // from here on `merkle->root` is the root of the WHOLE tree (the sub-tree's own root is top_layers[k][rank])
  trace_mark(ctx, "sharded commit: merkle + caps");
  ch.mix_root(t.merkle->root);
  if (root) memcpy(root, t.merkle->root, 32);
  s->trees.push_back(std::move(t));
  return NB200_OK;
}

// MerkleProver::decommit of a sharded tree: the same walk as merkle_decommit; every value / hash it names is owned by exactly one rank (a row
// slice, a sub-tree node) or known to all (replicated columns, the top layers): owners fill their words, one all-reduce merges them.
static nb200_status merkle_decommit_sharded(nb200_ctx* ctx, const SchemeTree& t, u32 blow, const std::vector<std::pair<u32, std::vector<u64>>>& queries,
                                            std::vector<u32>& queried_values, std::vector<uint8_t>& hash_witness, std::vector<u32>& column_witness) {
  const u32 k = (u32)comm_log_world(ctx);
  const int rank = comm_rank(ctx);
  const u32 m = t.big_log + blow;
  struct CRef { const u32* d; u32 log; bool big; };   // d is indexed by the global row; big: only this rank's rows, else a full replicated column
  std::vector<CRef> cols;
  for (size_t g = 0; g < t.cols.size(); ++g) {
    if (t.cols[g].batch == SchemeTree::BIG) cols.push_back(CRef{t.lde_rows(t.cols[g].idx), m, true});
    else cols.push_back(CRef{t.ldes[t.cols[g].batch]->col(t.cols[g].idx), t.ldes[t.cols[g].batch]->log_size, false});
  }
  std::stable_sort(cols.begin(), cols.end(), [](const CRef& a, const CRef& b) { return a.log > b.log; });
  std::vector<const u32*> val_addrs; std::vector<size_t> val_slot; std::vector<uint8_t> val_is_query;
  std::vector<const uint8_t*> hash_addrs; std::vector<size_t> hash_slot;
  std::vector<u32> vals; std::vector<uint8_t> hashes;
  size_t ci = 0;
  std::vector<u64> last_layer_queries;
  for (int l = (int)m; l >= 0; --l) {
    std::vector<u64> layer_total;
    size_t firstc = ci;
    while (ci < cols.size() && cols[ci].log == (u32)l) ++ci;
    const std::vector<u64>* lq = nullptr;
    for (auto& q : queries) if (q.first == (u32)l) lq = &q.second;
    size_t pq = 0, cq = 0;
    size_t nlq = lq ? lq->size() : 0;
    auto want_hash = [&](u64 child) {   // node `child` of layer l + 1
      const u32 cl = (u32)l + 1;
      const size_t slot = hashes.size() / 32;
      hashes.resize(hashes.size() + 32, 0);
      if (cl <= k) { if (rank == 0) memcpy(&hashes[32 * slot], &t.top_layers[cl][32 * child], 32); }      // known to all: rank 0 contributes
      else if ((child >> (cl - k)) == (u64)rank) { hash_addrs.push_back(t.merkle->layer[cl - k] + 32 * (child & (((u64)1 << (cl - k)) - 1))); hash_slot.push_back(slot); }
    };
    while (true) {
      bool has_p = pq < last_layer_queries.size(), has_c = cq < nlq;
      if (!has_p && !has_c) break;
      u64 node;
      if (has_p && has_c) node = std::min(last_layer_queries[pq] / 2, (*lq)[cq]);
      else if (has_p) node = last_layer_queries[pq] / 2;
      else node = (*lq)[cq];
      if ((u32)l < m) {
        if (pq < last_layer_queries.size() && last_layer_queries[pq] == 2 * node) ++pq; else want_hash(2 * node);
        if (pq < last_layer_queries.size() && last_layer_queries[pq] == 2 * node + 1) ++pq; else want_hash(2 * node + 1);
      }
      bool queried = cq < nlq && (*lq)[cq] == node;
      if (queried) ++cq;
      for (size_t c = firstc; c < ci; ++c) {
        const size_t slot = vals.size();
        vals.push_back(0u); val_is_query.push_back(queried ? 1 : 0);
        if (cols[c].big) { if ((node >> (m - k)) == (u64)rank) { val_addrs.push_back(cols[c].d + node); val_slot.push_back(slot); } }
        else if (rank == 0) { val_addrs.push_back(cols[c].d + node); val_slot.push_back(slot); }
      }
      layer_total.push_back(node);
    }
    last_layer_queries.swap(layer_total);
  }
  std::vector<u32> got(val_addrs.size());
  NB_TRY(gather_u32(ctx, val_addrs, got.data()));
  for (size_t i = 0; i < got.size(); ++i) vals[val_slot[i]] = got[i];
  std::vector<uint8_t> goth(hash_addrs.size() * 32);
  NB_TRY(gather_hash(ctx, hash_addrs, goth.data()));
  for (size_t i = 0; i < hash_addrs.size(); ++i) memcpy(&hashes[32 * hash_slot[i]], &goth[32 * i], 32);
  // merge: exactly one rank filled each word
  std::vector<u32> buf(vals.size() + hashes.size() / 4);
  memcpy(buf.data(), vals.data(), vals.size() * 4);
  if (!hashes.empty()) memcpy(buf.data() + vals.size(), hashes.data(), hashes.size());
  NB_TRY(comm_all_reduce_sum_host(ctx, buf.data(), buf.size()));
  queried_values.clear(); column_witness.clear();
  for (size_t i = 0; i < vals.size(); ++i) (val_is_query[i] ? queried_values : column_witness).push_back(buf[i]);
  hash_witness.resize(hashes.size());
  if (!hashes.empty()) memcpy(hash_witness.data(), buf.data() + vals.size(), hashes.size());
  return NB200_OK;
}

// ---- host-side point-mode interpreter (PointEvaluator) for the prover's sanity check ----
static qm31 from_partial_evals(const qm31 v[4]) {
  qm31 I = qm31_make(0, 1, 0, 0), U = qm31_make(0, 0, 1, 0), IU = qm31_make(0, 0, 0, 1);
  return qm31_add(qm31_add(v[0], qm31_mul(v[1], I)), qm31_add(qm31_mul(v[2], U), qm31_mul(v[3], IU)));
}
template <class OnC>
static void run_point(const std::vector<AirInstr>& prog, const qm31* mask, const std::vector<qm31>& params, std::vector<qm31>& br, std::vector<qm31>& er, OnC on_c) {
  for (const AirInstr& in : prog) {
    switch (in.op) {
      case OP_LOADM: br[in.dst] = mask[in.a]; break;
      case OP_CONSTB: br[in.dst] = qm31_from_m31(in.a); break;
      case OP_ADDB: br[in.dst] = qm31_add(br[in.a], br[in.b]); break;
      case OP_SUBB: br[in.dst] = qm31_sub(br[in.a], br[in.b]); break;
      case OP_MULB: br[in.dst] = qm31_mul(br[in.a], br[in.b]); break;
      case OP_NEGB: br[in.dst] = qm31_neg(br[in.a]); break;
      case OP_PARAME: er[in.dst] = params[in.a]; break;
      case OP_ADDE: er[in.dst] = qm31_add(er[in.a], er[in.b]); break;
      case OP_SUBE: er[in.dst] = qm31_sub(er[in.a], er[in.b]); break;
      case OP_MULE: er[in.dst] = qm31_mul(er[in.a], er[in.b]); break;
      case OP_NEGE: er[in.dst] = qm31_neg(er[in.a]); break;
      case OP_ADDEB: er[in.dst] = qm31_add(er[in.a], br[in.b]); break;
      case OP_SUBEB: er[in.dst] = qm31_sub(er[in.a], br[in.b]); break;
      case OP_MULEB: er[in.dst] = qm31_mul(er[in.a], br[in.b]); break;
      case OP_BTOE: er[in.dst] = br[in.a]; break;
      case OP_LOADME: er[in.dst] = from_partial_evals(mask + in.a); break;
      case OP_CONSTRB: on_c(br[in.a]); break;
      case OP_CONSTRE: on_c(er[in.a]); break;
      default: break;
    }
  }
}
// coset_vanishing of CanonicCoset(log).coset at a QM31 point
static qm31 coset_vanishing_q(u32 log_size, qpoint p) {
  HCoset c = HCoset::odds(log_size);
  u32 shift = idx_add(idx_neg(c.initial_index), c.step_index >> 1);
  qpoint r = qp_add(p, qp_from_m31(index_to_point(shift)));
  qm31 x = r.x;
  for (u32 i = 1; i < log_size; ++i) x = qm31_double_x(x);
  return x;
}

// ---- postcard (serde) writer for StarkProof ----                                              [risk A.12]
struct Postcard {
  std::vector<uint8_t> out;
  void varint(uint64_t v) { while (v >= 0x80) { out.push_back((uint8_t)(v | 0x80)); v >>= 7; } out.push_back((uint8_t)v); }
  void q(const qm31& v) { for (int k = 0; k < 4; ++k) varint(v.c[k]); }
  void hash(const uint8_t* h) { out.insert(out.end(), h, h + 32); }
};
struct Decommitment { std::vector<uint8_t> hash_witness; std::vector<u32> column_witness; };
struct FriLayerProof { std::vector<qm31> fri_witness; Decommitment decommitment; uint8_t commitment[32]; };
static void put_decommitment(Postcard& pc, const Decommitment& d) {
  pc.varint(d.hash_witness.size() / 32); pc.out.insert(pc.out.end(), d.hash_witness.begin(), d.hash_witness.end());
  pc.varint(d.column_witness.size()); for (u32 v : d.column_witness) pc.varint(v);
}
static void put_fri_layer(Postcard& pc, const FriLayerProof& l) {
  pc.varint(l.fri_witness.size()); for (auto& v : l.fri_witness) pc.q(v);
  put_decommitment(pc, l.decommitment); pc.hash(l.commitment);
}

// ---- queries (core/queries.rs) ----
struct Queries {
  std::vector<u64> positions; u32 log_domain_size = 0;
  static Queries generate(HostChannel& ch, u32 log_domain_size, size_t n_queries) {
    std::set<u64> q; size_t cnt = 0; u64 mask = ((u64)1 << log_domain_size) - 1;
    while (true) {
      uint8_t r[32]; ch.draw_random_bytes(r);
      for (int k = 0; k < 8; ++k) {
        u32 w = (u32)r[4 * k] | ((u32)r[4 * k + 1] << 8) | ((u32)r[4 * k + 2] << 16) | ((u32)r[4 * k + 3] << 24);
        q.insert((u64)w & mask);
        if (++cnt == n_queries) { Queries o; o.positions.assign(q.begin(), q.end()); o.log_domain_size = log_domain_size; return o; }
      }
    }
  }
  Queries fold(u32 n) const {
    Queries o; o.log_domain_size = log_domain_size - n;
    for (u64 p : positions) { u64 f = p >> n; if (o.positions.empty() || o.positions.back() != f) o.positions.push_back(f); }
    return o;
  }
};

// decommitment positions of one FRI layer column (compute_decommitment_positions_and_witness_evals), and the positions whose values
// are its witness: the sibling of every query whose sibling is not queried itself
static void positions_and_witness_plan(const std::vector<u64>& queries, std::vector<u64>& positions, std::vector<u64>& need) {
  size_t i = 0;
  while (i < queries.size()) {
    size_t j = i; u64 key = queries[i] >> 1;
    while (j < queries.size() && (queries[j] >> 1) == key) ++j;
    size_t qi = i;
    for (u64 pos = key << 1; pos < (key << 1) + 2; ++pos) {
      positions.push_back(pos);
      if (qi < j && queries[qi] == pos) { ++qi; continue; }
      need.push_back(pos);
    }
    i = j;
  }
}

static qm31 load_param(const u32* p) { return qm31_make(p[0], p[1], p[2], p[3]); }

// How a component's quotients are evaluated (always the same polynomial, hence the same composition coefficients):
//   Q_FULL   on CanonicCoset(eval_log).circle_domain(), the reference's domain: every polynomial is extended to it
//            (or, when eval_log equals the committed LDE size, the committed evaluations are used as they are);
//   Q_HALF   when eval_log = LDE size + 1: on the committed LDE domain D1 = CanonicCoset(eval_log - 1).circle_domain() (no transform
//            at all) and on D2 = the first half of CanonicCoset(eval_log).circle_domain() (a half-size transform).  In the circle-FFT
//            basis a polynomial with coefficients [lo | hi] is lo + pi^(eval_log-2)(x) * hi, and pi^(eval_log-2)(x) vanishes on D1 and is
//            the constant top-layer twiddle t on D2, so  lo = interpolate_D1(q|D1)  and  hi = interpolate_D2((q|D2 - lo|D2) / t).
//            A constraint of degree d <= AIR_LOW_DEGREE (air.h) has a quotient of circle degree at most 2^(eval_log - 2): its hi part is
//            zero.  By linearity hi(q) = hi(q_high), q_high the sum over the constraints of higher degree only, so D2 needs only those
//            constraints and only the columns they read:  hi = interpolate_D2((q_high|D2 - lo(q_high)|D2) / t),  lo(q_high) taken from
//            q_high|D1, which the D1 kernel sums on the side.  (The bytecode interpreter evaluates every constraint on D2: q_high = q.)
enum QuotMode { Q_FULL = 0, Q_HALF = 1 };
static QuotMode quotient_mode(const nb200_scheme* s, const AirComponent& c) {
  const u32 lde = c.log_size + s->log_blowup;
  return (c.eval_log() == lde + 1 && lde > 8) ? Q_HALF : Q_FULL;   // the half-domain transforms need more than 2^8 points (fft.cu)
}

// ComponentProver::evaluate_constraint_quotients_on_domain for one component: bring every column the component reads onto
// the evaluation rows, run the (JIT-specialised or interpreted) constraint kernel, ADD into the accumulators.
//   Q_FULL: accum = 4 columns of 2^eval_log (evaluations on the canonic domain);
//   Q_HALF: accum = q on D1, accum_hi = q_high on D2, accum_sub = q_high on D1, each 4 columns of 2^(eval_log - 1).
nb200_status component_quotients(nb200_scheme* s, nb200_air* air_h, size_t comp_idx, const u32* d_params, const std::vector<qm31>& coeff,
                                 QuotMode mode, nb200_cols* accum, nb200_cols* accum_hi, nb200_cols* accum_sub) {
  nb200_ctx* ctx = s->ctx;
  const AirProgram& air = air_h->prog;
  NB_ARG(ctx, comp_idx < air.comps.size(), "constraint quotients: component index");
  const AirComponent& c = air.comps[comp_idx];
  const u32 elog = c.eval_log(), lde_log = c.log_size + s->log_blowup;
  auto half_acc = [&](const nb200_cols* a) { return a && a->n_cols == 4 && a->log_size == lde_log; };
  if (mode == Q_HALF) NB_ARG(ctx, elog == lde_log + 1 && half_acc(accum) && half_acc(accum_hi) && half_acc(accum_sub), "constraint quotients: half-domain accumulators");
  else NB_ARG(ctx, accum && accum->n_cols == 4 && accum->log_size == elog, "constraint quotients: accumulator must be 4 columns of the evaluation domain size");
  NB_ARG(ctx, coeff.size() == c.n_constraints, "constraint quotients: one coefficient per constraint");
  NB_TRY(twiddles_prepare(ctx, elog));
  const bool reuse_lde = (mode == Q_FULL && elog == lde_log);
  const JitKernel* jp = ensure_jit(ctx, air_h, comp_idx, JIT_CONSTRAINTS, true);
  // Q_HALF: with the specialised kernels D2 evaluates the high-degree constraints only (none: D2 is skipped), else every constraint
  const std::vector<char> high = high_constraints(c);
  const JitKernel* jd2 = nullptr;
  bool split = false;
  if (mode == Q_HALF && jit_usable(jp, c, lde_log)) {
    jd2 = count_high(high) ? ensure_jit(ctx, air_h, comp_idx, JIT_D2, true) : nullptr;
    split = !count_high(high) || jd2;
  }
  const std::vector<char> on_d2 = split ? masks_read_by(c, high) : std::vector<char>(c.masks.size(), mode == Q_HALF ? 1 : 0);
  std::map<std::pair<u32, u32>, ColsPtr> ext;
  std::map<std::pair<u32, u32>, u32> d2_slot;   // Q_HALF: (tree, column) -> its column in d2_ext
  std::vector<const u32*> mask_cols(c.masks.size(), nullptr), mask_lde(c.masks.size());
  for (size_t m = 0; m < c.masks.size(); ++m) {
    const AirMask& mk = c.masks[m];
    NB_ARG(ctx, mk.tree < s->trees.size() && mk.col < s->trees[mk.tree].cols.size(), "prove: AIR references a column that was not committed");
    const SchemeTree& tr = s->trees[mk.tree];
    const SchemeTree::ColLoc& loc = tr.cols[mk.col];
    // a sharded column has no batch in ldes / coeffs: only component_quotients_sharded can read it
    NB_ARG(ctx, loc.batch != SchemeTree::BIG, "constraint quotients: column " + std::to_string(mk.col) + " of tree " + std::to_string(mk.tree) +
                                              " is sharded; only the sharded route (the half-domain entry) evaluates this component");
    NB_ARG(ctx, loc.log == c.log_size, "prove: column size differs from its component's log_size");
    mask_lde[m] = tr.ldes[loc.batch]->col(loc.idx);
    if (reuse_lde) { mask_cols[m] = mask_lde[m]; continue; }
    if (mode == Q_HALF) {
      if (!on_d2[m]) continue;
      if (loc.batch < tr.half_ext.size() && tr.half_ext[loc.batch]) mask_cols[m] = tr.half_ext[loc.batch]->col(loc.idx);   // precomputed at commit time
      else d2_slot.emplace(std::make_pair(mk.tree, mk.col), (u32)d2_slot.size());
      continue;
    }
    ColsPtr& e = ext[std::make_pair(mk.tree, loc.batch)];
    if (!e) {
      const nb200_cols* co = tr.coeffs[loc.batch].get();
      NB_TRY(alloc(ctx, e, co->n_cols, elog));
      NB_TRY(fft_evaluate(ctx, co->d, co->log_size, e->d, elog, co->n_cols));
    }
    mask_cols[m] = e->col(loc.idx);
  }
  // Q_HALF: the columns D2 reads, gathered from the committed coefficients into one batch and evaluated on the first half of canonic(elog)
  ColsPtr d2_ext;
  if (!d2_slot.empty()) {
    ColsPtr gathered;
    NB_TRY(alloc(ctx, gathered, d2_slot.size(), c.log_size));
    for (auto& kv : d2_slot)
      NB_CUDA(ctx, cudaMemcpyAsync(gathered->col(kv.second), s->trees[kv.first.first].coeff_ptr(kv.first.second), (size_t)4 << c.log_size,
                                   cudaMemcpyDeviceToDevice, ctx->stream));
    NB_TRY(alloc(ctx, d2_ext, d2_slot.size(), lde_log));
    NB_TRY(fft_evaluate(ctx, gathered->d, c.log_size, d2_ext->d, lde_log, d2_slot.size(), elog));
    for (size_t m = 0; m < c.masks.size(); ++m) {
      auto it = d2_slot.find(std::make_pair(c.masks[m].tree, c.masks[m].col));
      if (on_d2[m] && it != d2_slot.end()) mask_cols[m] = d2_ext->col(it->second);
    }
  }
  trace_mark(ctx, "constraints: extend columns");
  if (mode == Q_HALF) {
    u32* lo[4] = {accum->col(0), accum->col(1), accum->col(2), accum->col(3)};
    u32* hi[4] = {accum_hi->col(0), accum_hi->col(1), accum_hi->col(2), accum_hi->col(3)};
    u32* sub[4] = {accum_sub->col(0), accum_sub->col(1), accum_sub->col(2), accum_sub->col(3)};
    if (split) {
      NB_TRY(constraint_eval(ctx, c, mask_lde, d_params, coeff, lo, jp, lde_log, lde_log, 0, 0, sub));   // D1: the committed LDE; q and q_high
      if (jd2) NB_TRY(constraint_eval(ctx, c, mask_cols, d_params, coeff, hi, jd2, lde_log, elog));      // D2: first half of canonic(elog)
    } else {
      NB_TRY(constraint_eval(ctx, c, mask_lde, d_params, coeff, lo, jp, lde_log, lde_log));
      NB_TRY(constraint_eval(ctx, c, mask_lde, d_params, coeff, sub, jp, lde_log, lde_log));
      NB_TRY(constraint_eval(ctx, c, mask_cols, d_params, coeff, hi, jp, lde_log, elog));
    }
  } else {
    u32* accp[4] = {accum->col(0), accum->col(1), accum->col(2), accum->col(3)};
    NB_TRY(constraint_eval(ctx, c, mask_cols, d_params, coeff, accp, jp, elog, elog));
  }
  trace_mark(ctx, "constraints: row kernel");
  return NB200_OK;
}

static bool component_is_sharded(const nb200_scheme* s, const AirComponent& c) {
  for (const AirMask& mk : c.masks)
    if (mk.tree < s->trees.size() && s->trees[mk.tree].sharded && mk.col < s->trees[mk.tree].cols.size() && s->trees[mk.tree].cols[mk.col].batch == SchemeTree::BIG) return true;
  return false;
}

// evaluate_constraint_quotients_on_domain of the sharded (main) component: this rank evaluates ITS rows of D1 (from the LDE row slices) and of D2
// (from the D2 row slices) — masks at a row offset read the replicated full columns — and the accumulator columns are all-gathered in place.
static nb200_status component_quotients_sharded(nb200_scheme* s, nb200_air* air_h, size_t comp_idx, const u32* d_params, const std::vector<qm31>& coeff,
                                                nb200_cols* accum, nb200_cols* accum_hi, nb200_cols* accum_sub) {
  nb200_ctx* ctx = s->ctx;
  const AirComponent& c = air_h->prog.comps[comp_idx];
  const u32 elog = c.eval_log(), lde_log = c.log_size + s->log_blowup, k = (u32)comm_log_world(ctx);
  auto half_acc = [&](const nb200_cols* a) { return a && a->n_cols == 4 && a->log_size == lde_log; };
  NB_ARG(ctx, elog == lde_log + 1 && half_acc(accum) && half_acc(accum_hi) && half_acc(accum_sub),
         "sharded constraint quotients: the component must use the half-domain route");
  NB_ARG(ctx, coeff.size() == c.n_constraints, "constraint quotients: one coefficient per constraint");
  const size_t S = (size_t)1 << (lde_log - k);
  const u32 row0 = (u32)(comm_rank(ctx) * S);
  std::vector<const u32*> m_lde(c.masks.size()), m_hx(c.masks.size());
  for (size_t m = 0; m < c.masks.size(); ++m) {
    const AirMask& mk = c.masks[m];
    NB_ARG(ctx, mk.tree < s->trees.size() && mk.col < s->trees[mk.tree].cols.size(), "prove: AIR references a column that was not committed");
    const SchemeTree& tr = s->trees[mk.tree];
    const SchemeTree::ColLoc& loc = tr.cols[mk.col];
    NB_ARG(ctx, tr.sharded && loc.batch == SchemeTree::BIG && loc.log == c.log_size && tr.big_rows_hx, "sharded constraint quotients: the component may only read sharded columns of its own size");
    if (mk.off == 0) { m_lde[m] = tr.lde_rows(loc.idx); m_hx[m] = tr.hx_rows(loc.idx); }
    else {
      auto f = tr.full_lde.find(loc.idx); auto h = tr.full_hx.find(loc.idx);
      NB_ARG(ctx, f != tr.full_lde.end() && h != tr.full_hx.end(), "sharded constraint quotients: column " + std::to_string(mk.col) + " of tree " + std::to_string(mk.tree) +
                                                                   " is read at a row offset but was not listed for replication at commit time");
      m_lde[m] = f->second->d; m_hx[m] = h->second->d;
    }
  }
  // the same split as component_quotients: D1 sums q and q_high, D2 evaluates the high-degree constraints only (from every column's D2 rows,
  // which the sharded commit still computes)
  const JitKernel* jk = ensure_jit(ctx, air_h, comp_idx, JIT_CONSTRAINTS, false);
  const bool any_high = count_high(high_constraints(c)) > 0;
  const JitKernel* jd2 = any_high ? ensure_jit(ctx, air_h, comp_idx, JIT_D2, false) : nullptr;
  NB_ARG(ctx, jk != nullptr && (!any_high || jd2 != nullptr), "sharded constraint quotients need the specialised kernel");
  const std::vector<char> on_d2 = masks_read_by(c, high_constraints(c));
  for (size_t m = 0; m < c.masks.size(); ++m) if (!on_d2[m]) m_hx[m] = nullptr;
  u32* lo[4] = {accum->col(0), accum->col(1), accum->col(2), accum->col(3)};
  u32* hi[4] = {accum_hi->col(0), accum_hi->col(1), accum_hi->col(2), accum_hi->col(3)};
  u32* sub[4] = {accum_sub->col(0), accum_sub->col(1), accum_sub->col(2), accum_sub->col(3)};
  NB_TRY(constraint_eval(ctx, c, m_lde, d_params, coeff, lo, jk, lde_log, lde_log, row0, S, sub));
  if (jd2) NB_TRY(constraint_eval(ctx, c, m_hx, d_params, coeff, hi, jd2, lde_log, elog, row0, S));
  for (int q = 0; q < 4; ++q)
    for (u32* a : {lo[q], hi[q], sub[q]}) NB_TRY(comm_all_gather_dev(ctx, a + row0, S, a));
  trace_mark(ctx, "constraints: row kernel (sharded) + all-gather");
  return NB200_OK;
}

// coefficients (4 columns of 2^elog, circle-FFT basis) of the quotient polynomial held by a Q_HALF accumulator triple (q|D1, q_high|D2,
// q_high|D1: see quotient_mode); they are consumed
static nb200_status half_to_coeffs(nb200_ctx* ctx, nb200_cols* lo, nb200_cols* hi, nb200_cols* sub, u32 elog, u32* out /* 4 columns */, size_t out_stride /* >= 2^elog */) {
  const u32 h = elog - 1;
  const size_t hl = (size_t)1 << h;
  NB_TRY(fft_interpolate(ctx, lo->d, lo->d, 4, h));                 // lo = coefficients of q mod pi^(elog-2)
  NB_TRY(fft_interpolate(ctx, sub->d, sub->d, 4, h));               // lo(q_high)
  ColsPtr t;
  NB_TRY(alloc(ctx, t, 4, h));
  NB_TRY(fft_evaluate(ctx, sub->d, h, t->d, h, 4, elog));           // lo(q_high) evaluated on D2
  NB_TRY(sub_scale_top_twiddle(ctx, hi->d, t->d, 4 * hl, elog));    // (q_high|D2 - lo(q_high)|D2) / t
  NB_TRY(fft_interpolate(ctx, hi->d, hi->d, 4, h, elog));           // hi coefficients
  // the composition's coefficient columns are 2^comp_log apart; this accumulator's polynomial may be smaller (a machine whose largest
  // evaluation domain belongs to another component): found by the prover2-shaped machine, tests/test_gpu_prove_parity.py
  NB_TRY(add_cols_strided(ctx, out, out_stride, lo->d, hl, hl, 4));
  NB_TRY(add_cols_strided(ctx, out + hl, out_stride, hi->d, hl, hl, 4));
  return NB200_OK;
}

// QuotientOps::accumulate_quotients on CanonicCoset(log_size).circle_domain(): out (4 columns) = sum over the sample batches
struct SampleBatch { qpoint p; std::vector<std::pair<const u32*, qm31>> cols; };
nb200_status accumulate_quotients(nb200_ctx* ctx, u32 lg, const std::vector<SampleBatch>& hb, qm31 q_coeff, u32* out, u32 row0 = 0, size_t n_rows = 0) {
  std::vector<QBatchDev> qb(hb.size()); std::vector<QEntryDev> qe;
  for (size_t b = 0; b < hb.size(); ++b) {
    QBatchDev& B = qb[b];
    const qpoint& p = hb[b].p;
    B.prx[0] = p.x.c[0]; B.prx[1] = p.x.c[1]; B.pix[0] = p.x.c[2]; B.pix[1] = p.x.c[3];
    B.pry[0] = p.y.c[0]; B.pry[1] = p.y.c[1]; B.piy[0] = p.y.c[2]; B.piy[1] = p.y.c[3];
    qm31 alpha = qm31_one(), sa = qm31_zero(), sb = qm31_zero();
    B.first = (u32)qe.size(); B.count = (u32)hb[b].cols.size();
    for (auto& cv : hb[b].cols) {
      alpha = qm31_mul(alpha, q_coeff);
      // complex_conjugate_line_coeffs
      qm31 a = qm31_sub(qm31_conj(cv.second), cv.second);
      qm31 c = qm31_sub(qm31_conj(p.y), p.y);
      qm31 bq = qm31_sub(qm31_mul(cv.second, c), qm31_mul(a, p.y));
      sa = qm31_add(sa, qm31_mul(alpha, a)); sb = qm31_add(sb, qm31_mul(alpha, bq));
      qm31 ac = qm31_mul(alpha, c);
      QEntryDev e; e.col = cv.first; memcpy(e.c, ac.c, 16); e.pad[0] = e.pad[1] = 0;
      qe.push_back(e);
    }
    memcpy(B.A, sa.c, 16); memcpy(B.B, sb.c, 16);
    qm31 bc = qm31_pow(q_coeff, hb[b].cols.size());
    memcpy(B.coeff, bc.c, 16);
  }
  ColsPtr dom;
  NB_TRY(alloc(ctx, dom, 2, lg));
  NB_TRY(domain_points(ctx, lg, dom->col(0), dom->col(1)));
  return quotients_launch(ctx, qb.data(), qb.size(), qe.data(), qe.size(), dom->col(0), dom->col(1), lg, out, row0, n_rows);
}

// The host tables of the combined route (quotients_from_coeffs): per batch, its columns with their alphas (q_coeff^1, ^2, ... in batch
// order, as accumulate_quotients numbers them) as deep_combine entries, the entry range, and the line descriptor whose numerator is
// c G(x) - (A y + B).  A and B are accumulate_quotients' sums; c = conj(p.y) - p.y takes the place of its per-entry alpha c.
void deep_plan(const std::vector<SampleBatch>& hb, qm31 q_coeff, std::vector<QLineDev>& lines, std::vector<QEntryDev>& entries, std::vector<uint2>& ranges) {
  lines.assign(hb.size(), QLineDev{}); entries.clear(); ranges.assign(hb.size(), uint2{0, 0});
  for (size_t b = 0; b < hb.size(); ++b) {
    QLineDev& L = lines[b];
    const qpoint& p = hb[b].p;
    L.prx[0] = p.x.c[0]; L.prx[1] = p.x.c[1]; L.pix[0] = p.x.c[2]; L.pix[1] = p.x.c[3];
    L.pry[0] = p.y.c[0]; L.pry[1] = p.y.c[1]; L.piy[0] = p.y.c[2]; L.piy[1] = p.y.c[3];
    const qm31 c = qm31_sub(qm31_conj(p.y), p.y);
    qm31 alpha = qm31_one(), sa = qm31_zero(), sb = qm31_zero();
    ranges[b] = uint2{(u32)entries.size(), (u32)hb[b].cols.size()};
    for (auto& cv : hb[b].cols) {
      alpha = qm31_mul(alpha, q_coeff);
      // complex_conjugate_line_coeffs
      qm31 a = qm31_sub(qm31_conj(cv.second), cv.second);
      qm31 bq = qm31_sub(qm31_mul(cv.second, c), qm31_mul(a, p.y));
      sa = qm31_add(sa, qm31_mul(alpha, a)); sb = qm31_add(sb, qm31_mul(alpha, bq));
      QEntryDev e; e.col = cv.first; memcpy(e.c, alpha.c, 16); e.pad[0] = e.pad[1] = 0;
      entries.push_back(e);
    }
    memcpy(L.A, sa.c, 16); memcpy(L.B, sb.c, 16); memcpy(L.c, c.c, 16);
    qm31 bc = qm31_pow(q_coeff, hb[b].cols.size());
    memcpy(L.coeff, bc.c, 16);
  }
}

// accumulate_quotients over the LDEs (2^lg rows) of the columns whose coefficients (2^(lg - blow) each) the batches name: each batch's
// combination G_b = sum_k alpha_k f_k is formed on the coefficients, the 4 x n_batches combination columns are extended to 2^lg rows
// (LDE evaluation is linear and exact, so these are G_b's values on the LDE), and the row kernel reads them instead of every column.
nb200_status quotients_from_coeffs(nb200_ctx* ctx, u32 lg, u32 blow, const std::vector<SampleBatch>& hc, qm31 q_coeff, u32* out) {
  NB_ARG(ctx, !hc.empty() && lg >= blow + 2, "quotients_from_coeffs: at least one batch and 4 coefficients per column");
  std::vector<QLineDev> lines; std::vector<QEntryDev> entries; std::vector<uint2> ranges;
  deep_plan(hc, q_coeff, lines, entries, ranges);
  const u32 n = lg - blow;
  const size_t nb = hc.size();
  ColsPtr ext;
  NB_TRY(alloc(ctx, ext, 4 * nb, lg));
  {
    ColsPtr g;
    NB_TRY(alloc(ctx, g, 4 * nb, n));
    NB_TRY(deep_combine(ctx, ranges.data(), nb, entries.data(), entries.size(), n, g->d));
    NB_TRY(fft_evaluate(ctx, g->d, n, ext->d, lg, 4 * nb));
  }
  ColsPtr dom;
  NB_TRY(alloc(ctx, dom, 2, lg));
  NB_TRY(domain_points(ctx, lg, dom->col(0), dom->col(1)));
  return quotients_combined(ctx, lines.data(), nb, ext->d, dom->col(0), dom->col(1), lg, out);
}

// ---- stwo::prover::prove, one function per stage; prove_impl runs them in order ----

static nb200_status zeroed(nb200_ctx* ctx, u32 lg, ColsPtr& out) {
  NB_TRY(alloc(ctx, out, 4, lg));
  NB_CUDA(ctx, cudaMemsetAsync(out->d, 0, ((size_t)16) << lg, ctx->stream));
  return NB200_OK;
}

// composition polynomial: every component's constraint quotients, combined by the powers of random_coeff, committed as tree 3
static nb200_status commit_composition(nb200_scheme* s, nb200_air* air_h, const std::vector<qm31>& params, qm31 random_coeff, size_t n_total, HostChannel& ch) {
  nb200_ctx* ctx = s->ctx;
  const AirProgram& air = air_h->prog;
  const u32 blow = s->log_blowup;
  u32 comp_log = 0;
  for (auto& c : air.comps) comp_log = std::max(comp_log, c.eval_log());
  NB_TRY(twiddles_prepare(ctx, comp_log + blow));
  std::vector<qm31> powers(n_total);
  { qm31 a = qm31_one(); for (size_t i = 0; i < n_total; ++i) { powers[i] = a; a = qm31_mul(a, random_coeff); } }
  DevBuf d_params;
  NB_TRY(upload_params(ctx, params.data(), params.size(), d_params));

  // accumulators per (evaluation log, mode): Q_FULL -> {evals on canonic(elog), -, -}; Q_HALF -> {q on D1, q_high on D2, q_high on D1}
  struct Acc { ColsPtr a, b, c; };
  std::map<std::pair<u32, int>, Acc> acc;
  size_t g0 = 0;
  for (const AirComponent& c : air.comps) {
    const u32 elog = c.eval_log();
    const QuotMode mode = quotient_mode(s, c);
    Acc& a = acc[std::make_pair(elog, (int)mode)];
    if (!a.a) {
      NB_TRY(zeroed(ctx, mode == Q_HALF ? elog - 1 : elog, a.a));
      if (mode == Q_HALF) { NB_TRY(zeroed(ctx, elog - 1, a.b)); NB_TRY(zeroed(ctx, elog - 1, a.c)); }
    }
    std::vector<qm31> coeff(c.n_constraints);
    for (u32 k = 0; k < c.n_constraints; ++k) coeff[k] = powers[n_total - 1 - (g0 + k)];
    const size_t comp_idx = &c - &air.comps[0];
    if (component_is_sharded(s, c)) NB_TRY(component_quotients_sharded(s, air_h, comp_idx, d_params.p, coeff, a.a.get(), a.b.get(), a.c.get()));
    else NB_TRY(component_quotients(s, air_h, comp_idx, d_params.p, coeff, mode, a.a.get(), a.b.get(), a.c.get()));
    g0 += c.n_constraints;
  }
  // DomainEvaluationAccumulator::finalize.  Upstream folds the per-size accumulators upwards (evaluate the running polynomial on the next
  // size, add, interpolate); interpolation is linear, so the result is the sum of the zero-extended coefficient vectors — computed here.
  ColsPtr cur;  // coefficients of the composition (4 columns of 2^comp_log)
  NB_TRY(zeroed(ctx, comp_log, cur));
  for (auto& kv : acc) {
    const u32 elog = kv.first.first;
    nb200_cols* a = kv.second.a.get();
    if (kv.first.second == Q_HALF) NB_TRY(half_to_coeffs(ctx, a, kv.second.b.get(), kv.second.c.get(), elog, cur->d, (size_t)1 << comp_log));
    else {
      NB_TRY(fft_interpolate(ctx, a->d, a->d, 4, elog));
      NB_TRY(add_cols_strided(ctx, cur->d, (size_t)1 << comp_log, a->d, (size_t)1 << elog, (size_t)1 << elog, 4));
    }
  }
  acc.clear();   // before tree 3 is allocated
  // tree 3: the composition's 4 coordinate polynomials
  SchemeTree t;
  ColsPtr lde;
  NB_TRY(alloc(ctx, lde, 4, comp_log + blow));
  NB_TRY(fft_evaluate(ctx, cur->d, comp_log, lde->d, comp_log + blow, 4));
  t.coeffs.push_back(std::move(cur));
  t.ldes.push_back(std::move(lde));
  NB_TRY(finish_tree(ctx, t, ch));
  s->trees.push_back(std::move(t));
  trace_mark(ctx, "composition: coefficients + commit");
  return NB200_OK;
}

// the out-of-domain point, the points each committed column is sampled at and the values there (tree / column / offset order)
struct OodsSamples {
  qpoint point;
  std::vector<std::vector<std::vector<int32_t>>> offs;   // per tree / column: offsets in declaration order (Components::mask_points)
  std::vector<std::vector<std::vector<qpoint>>> points;
  std::vector<std::vector<std::vector<qm31>>> sampled;
};

static nb200_status sample_oods(nb200_scheme* s, const AirProgram& air, HostChannel& ch, OodsSamples& o) {
  nb200_ctx* ctx = s->ctx;
  {
    qm31 t = ch.draw_felt();
    qm31 t2 = qm31_sqr(t);
    qm31 ip = qm31_inv(qm31_add(t2, qm31_one()));
    o.point.x = qm31_mul(qm31_sub(qm31_one(), t2), ip);
    o.point.y = qm31_mul(qm31_add(t, t), ip);
  }
  auto& offs = o.offs;
  offs.resize(4);
  for (int t = 0; t < 4; ++t) offs[t].resize(s->trees[t].cols.size());
  for (const AirComponent& c : air.comps)
    for (const AirMask& m : c.masks) {
      auto& off = offs[m.tree][m.col];
      if (std::find(off.begin(), off.end(), m.off) == off.end()) off.push_back(m.off);
    }
  for (auto& off : offs[3]) off.assign(1, 0);
  auto mask_point = [&](u32 log_size, int32_t off) -> qpoint {
    if (off == 0) return o.point;
    u32 step = canonic_step_index(log_size);
    u32 idx = idx_mul(step, (u64)(off < 0 ? -off : off));
    if (off < 0) idx = idx_neg(idx);
    return qp_add(o.point, qp_from_m31(index_to_point(idx)));
  };
  auto& points = o.points;
  auto& sampled = o.sampled;
  points.resize(4); sampled.resize(4);
  std::vector<std::vector<qm31>*> sharded_samples;   // (multi-GPU) sampled-value lists of column-sharded columns, one entry per pushed value
  // every (column, point) pair of every tree is evaluated in one launch; a column-sharded column that this rank does not hold has no job
  // (its value stays zero until the all-reduce below)
  std::vector<EvalJob> jobs;
  std::vector<u32> pts;                                  // one point per distinct (tree, column offsets): 8 words each
  std::vector<std::vector<std::vector<long>>> job_of(4); // per tree / column / sample: its job, or -1
  for (int t = 0; t < 4; ++t) {
    const SchemeTree& tr = s->trees[t];
    points[t].resize(tr.cols.size()); sampled[t].resize(tr.cols.size()); job_of[t].resize(tr.cols.size());
    for (size_t g = 0; g < tr.cols.size(); ++g)
      for (int32_t off : offs[t][g]) points[t][g].push_back(mask_point(tr.cols[g].log, off));
    // groups of consecutive columns of one batch with the same offsets share their points
    size_t g = 0;
    while (g < tr.cols.size()) {
      size_t h = g + 1;
      while (h < tr.cols.size() && tr.cols[h].batch == tr.cols[g].batch && offs[t][h] == offs[t][g]) ++h;
      const size_t np = offs[t][g].size(), p0 = pts.size() / 8;
      for (size_t k = 0; k < np; ++k) {
        pts.insert(pts.end(), points[t][g][k].x.c, points[t][g][k].x.c + 4);
        pts.insert(pts.end(), points[t][g][k].y.c, points[t][g][k].y.c + 4);
      }
      const bool big = tr.sharded && tr.cols[g].batch == SchemeTree::BIG;
      for (size_t c = g; c < h; ++c) {
        const u32* co = nullptr;
        if (!big) co = tr.coeff_ptr(c);
        else if (c >= tr.own_first && c < tr.own_first + tr.own_count) co = tr.big_coeffs->col(c - tr.own_first);
        for (size_t k = 0; k < np; ++k) {
          job_of[t][c].push_back(co ? (long)jobs.size() : -1);
          if (co) jobs.push_back(EvalJob{co, tr.cols[c].log, (u32)(p0 + k)});
        }
      }
      g = h;
    }
  }
  std::vector<u32> out(jobs.size() * 4);
  NB_TRY(eval_at_points_multi(ctx, jobs, pts.data(), pts.size() / 8, out.data()));
  for (int t = 0; t < 4; ++t) {
    const SchemeTree& tr = s->trees[t];
    for (size_t c = 0; c < tr.cols.size(); ++c)
      for (long j : job_of[t][c]) {
        sampled[t][c].push_back(j >= 0 ? load_param(&out[4 * j]) : qm31_zero());
        if (tr.sharded && tr.cols[c].batch == SchemeTree::BIG) sharded_samples.push_back(&sampled[t][c]);
      }
  }
  if (!sharded_samples.empty()) {
    // every sampled value of a sharded column was computed by exactly one rank (zero elsewhere): one all-reduce completes them.  The list holds one
    // pointer per pushed value, in push order, so the k-th occurrence of a list is its k-th value.
    std::map<std::vector<qm31>*, size_t> seen;
    std::vector<u32> buf;
    for (auto* v : sharded_samples) { const qm31& q = (*v)[seen[v]++]; buf.insert(buf.end(), q.c, q.c + 4); }
    NB_TRY(comm_all_reduce_sum_host(ctx, buf.data(), buf.size()));
    seen.clear();
    size_t pos = 0;
    for (auto* v : sharded_samples) { (*v)[seen[v]++] = load_param(&buf[pos]); pos += 4; }
  }
  {
    std::vector<qm31> flat;
    for (auto& t : sampled) for (auto& c : t) for (auto& v : c) flat.push_back(v);
    ch.mix_felts(flat.data(), flat.size());
  }
  trace_mark(ctx, "oods eval_at_point");
  return NB200_OK;
}

// the columns FRI commits to and the layers it folds them into: held until their decommitments are taken
struct FriLayer { ColsPtr cols; TreePtr tree; u32 log; };
struct FriState {
  std::vector<ColsPtr> quotients;   // DEEP quotients, 4 coordinate columns each, largest first
  std::vector<u32> qlogs;
  TreePtr first_tree;
  std::vector<FriLayer> inner;
};

// Whether quotients_from_coeffs beats accumulate_quotients over the LDEs for these batches.  Each entry it combines on the coefficients
// saves reading half an LDE column (blow-up 2), and each of the 4 x n_batches combination columns it extends costs about as much as
// reading 6 LDE columns (H100, profiles/README.md: 12 columns extended to 2^21 rows in 0.20 ms; one such column read in 2.9 us).  A group
// breaks even at about 12 entries per extended column; the rule asks for 32.  The v1 main group (1395 entries at 3 points) passes; a
// group of a few columns, such as the composition's 4 at one point, stays on the LDEs.
static bool combine_pays(const std::vector<SampleBatch>& hc) {
  size_t entries = 0;
  for (auto& b : hc) entries += b.cols.size();
  return !hc.empty() && entries >= 32 * 4 * hc.size();
}

static nb200_status deep_quotients(nb200_scheme* s, const OodsSamples& o, HostChannel& ch, FriState& f) {
  nb200_ctx* ctx = s->ctx;
  qm31 q_coeff = ch.draw_felt();
  struct CRef { int t; size_t g; u32 log; };
  std::vector<CRef> all;
  for (int t = 0; t < 4; ++t) for (size_t g = 0; g < s->trees[t].cols.size(); ++g) all.push_back(CRef{t, g, s->trees[t].cols[g].log + s->log_blowup});
  std::stable_sort(all.begin(), all.end(), [](const CRef& a, const CRef& b) { return a.log > b.log; });
  for (size_t i = 0; i < all.size();) {
    size_t j = i; while (j < all.size() && all[j].log == all[i].log) ++j;
    const u32 lg = all[i].log;
    // ColumnSampleBatch::new_vec: group samples by point, first-seen order                   [risk: IndexMap vs BTreeMap]
    // hb names the columns' LDEs, hc the same batches with their coefficients (the combined route; unused when the group is sharded)
    std::vector<SampleBatch> hb, hc;
    const SchemeTree* sharded = nullptr;   // a tree whose row slices this group reads
    for (size_t k = i; k < j; ++k) {
      const CRef& r = all[k];
      for (size_t pi = 0; pi < o.points[r.t][r.g].size(); ++pi) {
        const qpoint& p = o.points[r.t][r.g][pi];
        size_t b = 0;
        for (; b < hb.size(); ++b) if (qm31_eq(hb[b].p.x, p.x) && qm31_eq(hb[b].p.y, p.y)) break;
        if (b == hb.size()) { hb.push_back(SampleBatch{p, {}}); hc.push_back(SampleBatch{p, {}}); }
        const SchemeTree& trr = s->trees[r.t];
        if (trr.sharded && trr.cols[r.g].batch == SchemeTree::BIG) {
          sharded = &trr;
          hb[b].cols.push_back({trr.lde_rows(trr.cols[r.g].idx), o.sampled[r.t][r.g][pi]});
        } else {
          hb[b].cols.push_back({trr.lde_ptr(r.g), o.sampled[r.t][r.g][pi]});
          hc[b].cols.push_back({trr.coeff_ptr(r.g), o.sampled[r.t][r.g][pi]});
        }
      }
    }
    ColsPtr q;
    NB_TRY(alloc(ctx, q, 4, lg));
    if (sharded) {   // this rank's rows of the quotient column, then an all-gather: FRI runs replicated on the whole column
      const size_t rows = sharded->big_rows->col_len();
      const u32 r0 = (u32)sharded->row0();
      NB_TRY(accumulate_quotients(ctx, lg, hb, q_coeff, q->d, r0, rows));
      for (int qq = 0; qq < 4; ++qq) NB_TRY(comm_all_gather_dev(ctx, q->col(qq) + r0, rows, q->col(qq)));
    } else if (combine_pays(hc) && lg >= s->log_blowup + 2) NB_TRY(quotients_from_coeffs(ctx, lg, s->log_blowup, hc, q_coeff, q->d));
    else NB_TRY(accumulate_quotients(ctx, lg, hb, q_coeff, q->d));
    f.quotients.push_back(std::move(q)); f.qlogs.push_back(lg);
    i = j;
  }
  trace_mark(ctx, "deep quotients");
  return NB200_OK;
}

static nb200_status fri_commit(nb200_scheme* s, HostChannel& ch, FriState& f, std::vector<qm31>& last_layer_poly) {
  nb200_ctx* ctx = s->ctx;
  {
    std::vector<ColRef> refs;
    for (size_t g = 0; g < f.quotients.size(); ++g) for (int k = 0; k < 4; ++k) refs.push_back(ColRef{f.quotients[g]->col(k), f.qlogs[g]});
    nb200_tree* tree = nullptr;
    NB_TRY(merkle_commit(ctx, refs, &tree));
    f.first_tree.reset(tree);
    ch.mix_root(tree->root);
  }
  qm31 circle_alpha = ch.draw_felt();
  const size_t last_domain = (size_t)1 << (s->log_last + s->log_blowup);
  u32 L = f.qlogs[0] - 1;
  u32 n_inner = 0;
  for (u32 l = L; ((size_t)1 << l) > last_domain && l > 0; --l) ++n_inner;
  // The inner layers run on the device channel (device_channel.cuh), seeded from the host channel's state: each layer's Merkle root is
  // mixed and the next alpha drawn by one device thread, so the layers are queued without waiting for the host.  chan = the channel
  // state (16 words), then per layer its root (8 words) and alpha (4 words).
  DevBuf chan;
  NB_TRY(alloc(ctx, chan, 16 + 12 * (size_t)n_inner));
  DevChannel seed{};
  for (int i = 0; i < 8; ++i) seed.digest[i] = (u32)ch.digest[4 * i] | ((u32)ch.digest[4 * i + 1] << 8) | ((u32)ch.digest[4 * i + 2] << 16) | ((u32)ch.digest[4 * i + 3] << 24);
  seed.n_sent[0] = (u32)ch.n_sent; seed.n_sent[1] = (u32)(ch.n_sent >> 32);
  NB_CUDA(ctx, cudaMemcpyAsync(chan.p, &seed, sizeof(seed), cudaMemcpyHostToDevice, ctx->stream));
  u32* rec = chan.p + 16;
  ColsPtr layer;
  NB_TRY(alloc(ctx, layer, 4, L));
  NB_CUDA(ctx, cudaMemsetAsync(layer->d, 0, (size_t)16 << L, ctx->stream));
  size_t ci = 0;
  while (((size_t)1 << L) > last_domain) {
    const size_t k = f.inner.size();
    if (k >= n_inner) return set_err(ctx, NB200_ERR_STATE, "fri: layer count");
    for (; ci < f.quotients.size() && f.qlogs[ci] - 1 == L; ++ci) NB_TRY(fold_circle_into_line(ctx, layer->d, f.quotients[ci]->d, f.qlogs[ci], circle_alpha));
    std::vector<ColRef> refs; for (int c = 0; c < 4; ++c) refs.push_back(ColRef{layer->col(c), L});
    const u32* folded = layer->d;
    f.inner.push_back(FriLayer{std::move(layer), nullptr, L});
    nb200_tree* tree = nullptr;
    NB_TRY(merkle_commit(ctx, refs, &tree, nullptr, false));
    f.inner.back().tree.reset(tree);
    NB_TRY(channel_mix_draw(ctx, (DevChannel*)chan.p, tree->layer[0], rec + 12 * k, ch.draw_domain_sep));
    NB_TRY(alloc(ctx, layer, 4, L - 1));
    NB_TRY(fold_line(ctx, layer->d, folded, L, rec + 12 * k + 8));
    L -= 1;
  }
  // circle columns that fold exactly into the last layer's size would be an upstream assertion failure
  if (ci != f.quotients.size()) return set_err(ctx, NB200_ERR_STATE, "fri: not all columns consumed");
  if (((size_t)1 << L) != last_domain) return set_err(ctx, NB200_ERR_STATE, "fri: last layer size");
  // one round trip for the whole FRI commit: every root and device-drawn alpha, and the last layer
  std::vector<u32> recs(12 * (size_t)n_inner);
  std::vector<u32> host((size_t)4 << L);
  if (!recs.empty()) NB_CUDA(ctx, cudaMemcpyAsync(recs.data(), rec, recs.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
  NB_CUDA(ctx, cudaMemcpyAsync(host.data(), layer->d, host.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  layer.reset();
  // the host channel replays the layers: the same state as a channel that mixed each root and drew each alpha itself
  for (size_t k = 0; k < f.inner.size(); ++k) {
    memcpy(f.inner[k].tree->root, &recs[12 * k], 32);
    ch.mix_root(f.inner[k].tree->root);
    const qm31 alpha = ch.draw_felt();
    if (memcmp(alpha.c, &recs[12 * k + 8], 16) != 0) return set_err(ctx, NB200_ERR_STATE, "fri: the device channel drew a different alpha than the host channel");
  }
  // LineEvaluation::interpolate on the host (the last layer has 2^(log_last + blowup) points)
  size_t n = (size_t)1 << L;
  std::vector<qm31> v(n);
  for (size_t i2 = 0; i2 < n; ++i2) v[bit_reverse_u32((u32)i2, L)] = qm31_make(host[i2], host[n + i2], host[2 * n + i2], host[3 * n + i2]);
  HLineDomain d = HLineDomain::make(HCoset::half_odds(L));
  while (d.size() > 1) {
    size_t ds = d.size();
    for (size_t c0 = 0; c0 < n; c0 += ds)
      for (size_t i2 = 0; i2 < ds / 2; ++i2) {
        u32 xi = m31_inv(d.at(i2));
        qm31 a = v[c0 + i2], b = v[c0 + ds / 2 + i2];
        v[c0 + i2] = qm31_add(a, b);
        v[c0 + ds / 2 + i2] = qm31_mul_m31(qm31_sub(a, b), xi);
      }
    d = d.dbl();
  }
  u32 sc = m31_inv((u32)(n % P31));
  for (auto& qv : v) qv = qm31_mul_m31(qv, sc);
  // v is the LinePoly storage order (bit-reversed); ordered coefficients = bit-reversed again
  std::vector<qm31> ordered(n);
  for (size_t i2 = 0; i2 < n; ++i2) ordered[bit_reverse_u32((u32)i2, L)] = v[i2];
  size_t bound = (size_t)1 << s->log_last;
  for (size_t i2 = bound; i2 < n; ++i2) if (!qm31_is_zero(ordered[i2])) return set_err(ctx, NB200_ERR_CONSTRAINTS, "fri: last layer has invalid degree (constraints not satisfied)");
  last_layer_poly.resize(bound);
  for (size_t i2 = 0; i2 < bound; ++i2) last_layer_poly[bit_reverse_u32((u32)i2, s->log_last)] = ordered[i2];
  ch.mix_felts(last_layer_poly.data(), last_layer_poly.size());
  trace_mark(ctx, "fri commit");
  return NB200_OK;
}

// the parts of the StarkProof that the proof-of-work, query and decommitment stage produces
struct Decommitments {
  uint64_t nonce = 0;
  FriLayerProof first_layer;
  std::vector<FriLayerProof> inner_layers;
  std::vector<std::vector<u32>> queried_values;   // per tree
  std::vector<Decommitment> trees;                // per tree
};

static nb200_status decommit(nb200_scheme* s, HostChannel& ch, const FriState& f, Decommitments& out) {
  nb200_ctx* ctx = s->ctx;
  const u32 blow = s->log_blowup;
  NB_TRY(grind(ctx, ch.digest.data(), s->pow_bits, &out.nonce));
  ch.mix_u64(out.nonce);
  const u32 max_log = f.qlogs[0];
  Queries queries = Queries::generate(ch, max_log, s->n_queries);
  std::vector<std::pair<u32, std::vector<u64>>> by_log;
  for (u32 lg : f.qlogs) by_log.push_back({lg, queries.fold(max_log - lg).positions});

  // Every position is known now: the walks of all the decommitments (first FRI layer, inner layers, trace trees) are planned on the host,
  // everything they name is fetched with ONE gather, and the results are sorted into the proof in the same order as a walk per tree.
  std::vector<const uint8_t*> ha;
  std::vector<const u32*> va;
  struct Wit { std::vector<qm31>* out; size_t v0, n; };                            // FRI witness values: n QM31s from va[v0]
  struct Part { DecommitPlan plan; size_t h0, v0; Decommitment* dec; std::vector<u32>* qv; };
  std::vector<Wit> wits;
  std::vector<Part> parts;
  auto plan_witness = [&](const nb200_cols* col4, const std::vector<u64>& q, std::vector<u64>& pos, std::vector<qm31>& w) {
    std::vector<u64> need;
    positions_and_witness_plan(q, pos, need);
    wits.push_back(Wit{&w, va.size(), need.size()});
    for (u64 p : need) for (int k = 0; k < 4; ++k) va.push_back(col4->col(k) + p);
  };
  auto plan_tree = [&](const nb200_tree* tree, const std::vector<ColRef>& refs, const std::vector<std::pair<u32, std::vector<u64>>>& q,
                       Decommitment& dec, std::vector<u32>* qv) {
    Part p;
    std::vector<u32> logs(refs.size());
    for (size_t i = 0; i < refs.size(); ++i) logs[i] = refs[i].log_size;
    merkle_decommit_plan(tree->max_log, logs, q, p.plan);
    p.h0 = ha.size(); p.v0 = va.size(); p.dec = &dec; p.qv = qv;
    merkle_decommit_addrs(p.plan, tree, refs, ha, va);
    parts.push_back(std::move(p));
  };
  {
    std::vector<std::pair<u32, std::vector<u64>>> dpos;
    for (size_t g = 0; g < f.quotients.size(); ++g) {
      std::vector<u64> pos;
      plan_witness(f.quotients[g].get(), queries.fold(max_log - f.qlogs[g]).positions, pos, out.first_layer.fri_witness);
      dpos.push_back({f.qlogs[g], pos});
    }
    std::vector<ColRef> refs;
    for (size_t g = 0; g < f.quotients.size(); ++g) for (int k = 0; k < 4; ++k) refs.push_back(ColRef{f.quotients[g]->col(k), f.qlogs[g]});
    plan_tree(f.first_tree.get(), refs, dpos, out.first_layer.decommitment, nullptr);
    memcpy(out.first_layer.commitment, f.first_tree->root, 32);
  }
  out.inner_layers.resize(f.inner.size());
  {
    Queries lq = queries.fold(1);
    for (size_t k = 0; k < f.inner.size(); ++k) {
      const FriLayer& ly = f.inner[k];
      FriLayerProof& lp = out.inner_layers[k];
      std::vector<u64> pos;
      plan_witness(ly.cols.get(), lq.positions, pos, lp.fri_witness);
      std::vector<std::pair<u32, std::vector<u64>>> dpos{{ly.log, pos}};
      std::vector<ColRef> refs; for (int c = 0; c < 4; ++c) refs.push_back(ColRef{ly.cols->col(c), ly.log});
      plan_tree(ly.tree.get(), refs, dpos, lp.decommitment, nullptr);
      memcpy(lp.commitment, ly.tree->root, 32);
      lq = lq.fold(1);
    }
  }
  out.queried_values.resize(4); out.trees.resize(4);
  for (int t = 0; t < 4; ++t) {
    const SchemeTree& tr = s->trees[t];
    if (tr.sharded) continue;   // below, with its own gathers and all-reduce
    std::vector<ColRef> refs;
    for (size_t g = 0; g < tr.cols.size(); ++g) refs.push_back(ColRef{tr.lde_ptr(g), tr.cols[g].log + blow});
    plan_tree(tr.merkle.get(), refs, by_log, out.trees[t], &out.queried_values[t]);
  }
  std::vector<uint8_t> hashes(ha.size() * 32);
  std::vector<u32> vals(va.size());
  NB_TRY(gather_batch(ctx, ha, va, hashes.data(), vals.data()));
  for (const Wit& w : wits)
    for (size_t i = 0; i < w.n; ++i) { const u32* v = &vals[w.v0 + 4 * i]; w.out->push_back(qm31_make(v[0], v[1], v[2], v[3])); }
  for (const Part& p : parts) {
    std::vector<u32> unused;   // a FRI layer's queried values are not part of the proof
    merkle_decommit_fill(p.plan, hashes.data() + 32 * p.h0, vals.data() + p.v0, p.qv ? *p.qv : unused, p.dec->hash_witness, p.dec->column_witness);
  }
  for (int t = 0; t < 4; ++t) {
    const SchemeTree& tr = s->trees[t];
    if (tr.sharded) NB_TRY(merkle_decommit_sharded(ctx, tr, blow, by_log, out.queried_values[t], out.trees[t].hash_witness, out.trees[t].column_witness));
  }
  return NB200_OK;
}

// sanity check: composition(oods) == recomputed from the sampled mask values
static nb200_status check_oods(nb200_ctx* ctx, const AirProgram& air, const std::vector<qm31>& params, qm31 random_coeff, const OodsSamples& o) {
  qm31 accumulation = qm31_zero();
  for (const AirComponent& c : air.comps) {
    std::vector<qm31> mask(c.masks.size());
    for (size_t m = 0; m < c.masks.size(); ++m) {
      const auto& off = o.offs[c.masks[m].tree][c.masks[m].col];
      size_t k = std::find(off.begin(), off.end(), c.masks[m].off) - off.begin();
      mask[m] = o.sampled[c.masks[m].tree][c.masks[m].col][k];
    }
    qm31 dinv = qm31_inv(coset_vanishing_q(c.log_size, o.point));
    std::vector<qm31> br(c.n_base_regs), er(c.n_ext_regs);
    run_point(c.prog, mask.data(), params, br, er, [&](qm31 v) { accumulation = qm31_add(qm31_mul(accumulation, random_coeff), qm31_mul(dinv, v)); });
  }
  const auto& comp = o.sampled[3];
  qm31 cv[4] = {comp[0][0], comp[1][0], comp[2][0], comp[3][0]};
  if (!qm31_eq(from_partial_evals(cv), accumulation)) return set_err(ctx, NB200_ERR_CONSTRAINTS, "ConstraintsNotSatisfied");
  return NB200_OK;
}

// StarkProof -> postcard
static std::vector<uint8_t> serialize_proof(const nb200_scheme* s, const OodsSamples& o, const std::vector<qm31>& last_layer_poly, const Decommitments& d) {
  Postcard pc;
  pc.varint(s->pow_bits); pc.varint(s->log_blowup); pc.varint(s->log_last); pc.varint(s->n_queries);
  pc.varint(4); for (int t = 0; t < 4; ++t) pc.hash(s->trees[t].merkle->root);
  pc.varint(4);
  for (int t = 0; t < 4; ++t) { pc.varint(o.sampled[t].size()); for (auto& c : o.sampled[t]) { pc.varint(c.size()); for (auto& v : c) pc.q(v); } }
  pc.varint(4); for (int t = 0; t < 4; ++t) put_decommitment(pc, d.trees[t]);
  pc.varint(4); for (int t = 0; t < 4; ++t) { pc.varint(d.queried_values[t].size()); for (u32 v : d.queried_values[t]) pc.varint(v); }
  pc.varint(d.nonce);
  put_fri_layer(pc, d.first_layer);
  pc.varint(d.inner_layers.size()); for (auto& l : d.inner_layers) put_fri_layer(pc, l);
  pc.varint(last_layer_poly.size()); for (auto& v : last_layer_poly) pc.q(v);
  pc.varint(s->log_last);
  return std::move(pc.out);
}

// stwo::prover::prove
nb200_status prove_impl(nb200_scheme* s, nb200_air* air_h, const std::vector<qm31>& params, HostChannel& ch, std::vector<uint8_t>& proof_bytes) {
  nb200_ctx* ctx = s->ctx;
  const AirProgram& air = air_h->prog;
  NB_ARG(ctx, s->trees.size() == 3, "prove: the preprocessed, main and interaction trees must be committed first");
  NB_ARG(ctx, params.size() == air.n_params, "prove: parameter table size");
  size_t n_total = 0;
  for (auto& c : air.comps) n_total += c.n_constraints;
  NB_ARG(ctx, n_total > 0, "prove: no constraints");

  trace_mark(ctx, nullptr);
  const qm31 random_coeff = ch.draw_felt();
  NB_TRY(commit_composition(s, air_h, params, random_coeff, n_total, ch));   // tree 3 stays in the scheme even if a later stage fails
  OodsSamples oods;
  NB_TRY(sample_oods(s, air, ch, oods));
  std::vector<qm31> last_layer_poly;
  Decommitments dec;
  {
    FriState fri;
    NB_TRY(deep_quotients(s, oods, ch, fri));
    NB_TRY(fri_commit(s, ch, fri, last_layer_poly));
    NB_TRY(decommit(s, ch, fri, dec));
  }
  trace_mark(ctx, "pow + decommit");
  NB_TRY(check_oods(ctx, air, params, random_coeff, oods));
  proof_bytes = serialize_proof(s, oods, last_layer_poly, dec);
  trace_mark(ctx, "sanity + serialize");
  return NB200_OK;
}

// LogupTraceGenerator over the committed trace (the trace evaluations are passed in by the caller, as in the reference
// where generate_interaction_trace reads the finalized traces — machine.rs:242-247)
nb200_status gen_interaction(nb200_ctx* ctx, nb200_air* air_h, u32 comp_idx, const nb200_cols* const* tree0, size_t n0, const nb200_cols* const* tree1, size_t n1,
                             const std::vector<qm31>& params, nb200_cols** out, qm31* claimed) {
  const AirProgram& air = air_h->prog;
  NB_ARG(ctx, comp_idx < air.comps.size(), "gen_interaction: component index");
  const AirComponent& c = air.comps[comp_idx];
  std::vector<std::vector<const u32*>> flat(2);
  std::vector<std::vector<u32>> flog(2);
  for (size_t b = 0; b < n0; ++b) for (size_t k = 0; k < tree0[b]->n_cols; ++k) { flat[0].push_back(tree0[b]->col(k)); flog[0].push_back(tree0[b]->log_size); }
  for (size_t b = 0; b < n1; ++b) for (size_t k = 0; k < tree1[b]->n_cols; ++k) { flat[1].push_back(tree1[b]->col(k)); flog[1].push_back(tree1[b]->log_size); }
  std::vector<const u32*> mask_cols(c.masks.size(), nullptr);
  for (size_t m = 0; m < c.masks.size(); ++m) {
    const AirMask& mk = c.masks[m];
    if (mk.tree == 2) continue;
    NB_ARG(ctx, mk.col < flat[mk.tree].size(), "gen_interaction: AIR references a missing trace column");
    NB_ARG(ctx, flog[mk.tree][mk.col] == c.log_size, "gen_interaction: column size differs from the component's log_size");
    mask_cols[m] = flat[mk.tree][mk.col];
  }
  DevBuf d_params;
  NB_TRY(upload_params(ctx, params.data(), params.size(), d_params));
  ColsPtr o;
  NB_TRY(alloc(ctx, o, (size_t)4 * c.n_logup_cols(), c.log_size));
  trace_mark(ctx, nullptr);
  const JitKernel* jk = ensure_jit(ctx, air_h, comp_idx, JIT_LOGUP, true);
  nb200_status st = logup_generate(ctx, c, mask_cols, d_params.p, o->d, claimed, jk);
  trace_mark(ctx, "logup interaction trace");
  cudaStreamSynchronize(ctx->stream);
  NB_TRY(st);
  *out = o.release();
  return NB200_OK;
}

// assert_constraints_on_polys for one component on the GPU: every constraint evaluated on every row of its trace domain, from the trace
// evaluations of the three committed trees (the caller's batches, commitment order).  Per constraint: the number of rows where it does not
// hold and the first of them in coset order (UINT64_MAX: none).
nb200_status check_constraints(nb200_ctx* ctx, nb200_air* air_h, u32 comp_idx, const nb200_cols* const* const trees[3], const size_t n_trees[3],
                               const u32* params, size_t n_params, uint64_t* n_failing, uint64_t* first_row, size_t n) {
  const AirProgram& air = air_h->prog;
  NB_ARG(ctx, comp_idx < air.comps.size(), "check_constraints: component index");
  const AirComponent& c = air.comps[comp_idx];
  NB_ARG(ctx, n == c.n_constraints, "check_constraints: n must be the component's constraint count");
  NB_ARG(ctx, n_params == air.n_params, "check_constraints: parameter table size");
  if (n == 0) return NB200_OK;   // nothing to check: an empty report
  std::vector<std::vector<const u32*>> flat(3);
  std::vector<std::vector<u32>> flog(3);
  for (int t = 0; t < 3; ++t)
    for (size_t b = 0; b < n_trees[t]; ++b) {
      NB_ARG(ctx, trees[t][b], "check_constraints: null batch");
      for (size_t k = 0; k < trees[t][b]->n_cols; ++k) { flat[t].push_back(trees[t][b]->col(k)); flog[t].push_back(trees[t][b]->log_size); }
    }
  std::vector<const u32*> mask_cols(c.masks.size(), nullptr);
  for (size_t m = 0; m < c.masks.size(); ++m) {
    const AirMask& mk = c.masks[m];
    NB_ARG(ctx, mk.col < flat[mk.tree].size(), "check_constraints: AIR references a missing trace column");
    NB_ARG(ctx, flog[mk.tree][mk.col] == c.log_size, "check_constraints: column size differs from the component's log_size");
    mask_cols[m] = flat[mk.tree][mk.col];
  }
  const JitKernel* jk = ensure_jit(ctx, air_h, comp_idx, JIT_CHECK, false);
  if (!jk)
    return set_err(ctx, NB200_ERR_STATE, jit_enabled() ? "check_constraints: the constraint-check kernel could not be compiled: " + air_h->jit[JIT_CHECK][comp_idx].err
                                                       : std::string("check_constraints: the constraint check runs only as a generated kernel (NB200_JIT=0)"));
  // device side: the parameter table and one count + one row per constraint
  DevBuf d_params, d_res;
  NB_TRY(upload_params(ctx, params, n_params, d_params));
  NB_TRY(alloc(ctx, d_res, 2 * n));
  NB_CUDA(ctx, cudaMemsetAsync(d_res.p, 0, n * 4, ctx->stream));
  NB_CUDA(ctx, cudaMemsetAsync(d_res.p + n, 0xff, n * 4, ctx->stream));
  trace_mark(ctx, nullptr);
  // one thread per trace row; a domain smaller than a CTA (MultiMachine has 2^4-row components) runs as one CTA of exactly its rows
  const size_t rows = (size_t)1 << jk->log_size;
  const u32 block = (u32)std::min<size_t>(rows, JIT_LAUNCH_BLOCK);
  u32* d_nfail = d_res.p; u32* d_first = d_res.p + n;
  void* args[] = {(void*)&d_params.p, (void*)&d_nfail, (void*)&d_first};
  NB_TRY(jit_launch(ctx, *jk, mask_cols.data(), mask_cols.size(), dim3((u32)((rows + block - 1) / block)), dim3(block), args));
  std::vector<u32> res(2 * n);
  NB_CUDA(ctx, cudaMemcpyAsync(res.data(), d_res.p, 2 * n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // also: the host tables above have been consumed
  trace_mark(ctx, "constraint check");
  for (size_t k = 0; k < n; ++k) {
    n_failing[k] = res[k];
    first_row[k] = res[n + k] == 0xffffffffu ? UINT64_MAX : (uint64_t)res[n + k];
  }
  return NB200_OK;
}

// Every table fraction's multiplicity column, counted on the GPU from the AIR's own lookups (air_lookup_tables, jit.cu gen_count_source).
// Each row of each table fraction is a bin (tables in component then fraction order, rows in finalized order).  The build kernels hash
// every table tuple to its bin, the probe kernels add every lookup's numerator to its tuple's bin, and the bins are written mod P into the
// multiplicity columns of tree 1, in place.  A tuple listed by two rows of one relation is refused, or with `first_row` credited to its
// first row (table_first_row.cuh, between build and probe): *n_repeated = the rows written as 0.
nb200_status table_multiplicities(nb200_ctx* ctx, nb200_air* air_h, const nb200_cols* const* const trees[2], const size_t n_trees[2],
                                  uint64_t* n_unmatched, uint32_t first[3], bool first_row = false, uint64_t* n_repeated = nullptr) {
  const AirProgram& air = air_h->prog;
  const std::vector<std::vector<AirFrac>>& fr = air_h->fracs;
  std::vector<std::vector<u32*>> flat(2);
  std::vector<std::vector<u32>> flog(2);
  for (int t = 0; t < 2; ++t)
    for (size_t b = 0; b < n_trees[t]; ++b) {
      NB_ARG(ctx, trees[t][b], "table_multiplicities: null batch");
      for (size_t k = 0; k < trees[t][b]->n_cols; ++k) { flat[t].push_back(trees[t][b]->col(k)); flog[t].push_back(trees[t][b]->log_size); }
    }
  NB_ARG(ctx, air.comps.size() < (1u << 16), "table_multiplicities: at most 2^16 - 1 components");
  std::vector<std::vector<u32>> tbase(air.comps.size());
  std::vector<std::pair<u32*, u32>> mult;      // bin order: (multiplicity column, log size) per table fraction
  std::set<const u32*> mult_seen;
  std::vector<char> builds(air.comps.size(), 0), probes(air.comps.size(), 0);
  uint64_t n_bins = 0, additions = 0;
  u32 max_len = 0;
  for (size_t k = 0; k < air.comps.size(); ++k) {
    const AirComponent& c = air.comps[k];
    for (size_t i = 0; i < fr[k].size(); ++i) {
      const AirFrac& f = fr[k][i];
      const std::string where = "table_multiplicities: component " + std::to_string(k) + ", fraction " + std::to_string(i) + ": ";
      NB_ARG(ctx, f.kind != FRAC_BAD, where + f.why);
      if (f.kind == FRAC_TABLE) {
        const AirMask& mk = c.masks[f.mult_mask];
        NB_ARG(ctx, mk.col < flat[1].size() && flog[1][mk.col] == c.log_size, where + "its multiplicity column is missing from tree 1 or has another size");
        NB_ARG(ctx, mult_seen.insert(flat[1][mk.col]).second, where + "two table fractions share a multiplicity column");
        tbase[k].push_back((u32)n_bins);
        mult.push_back({flat[1][mk.col], c.log_size});
        n_bins += (uint64_t)1 << c.log_size;
        builds[k] = 1;
      } else if (f.kind == FRAC_LOOKUP) {
        NB_ARG(ctx, i < (1u << 20), where + "at most 2^20 fractions per component");
        additions += (uint64_t)1 << c.log_size;
        probes[k] = 1;
      } else {
        continue;
      }
      max_len = std::max<u32>(max_len, (u32)f.tuple.size());
    }
  }
  *n_unmatched = 0;
  first[0] = first[1] = first[2] = UINT32_MAX;
  if (n_repeated) *n_repeated = 0;
  if (n_bins == 0) return NB200_OK;   // no table: nothing to count
  NB_ARG(ctx, n_bins <= (1ull << 30), "table_multiplicities: at most 2^30 table rows");
  // a numerator is below 2^31, so a u64 bin is exact for up to 2^33 additions: more lookups than that in one call could wrap it
  NB_ARG(ctx, additions <= (1ull << 33), "table_multiplicities: more than 2^33 lookups (rows x lookup fractions) could overflow a 64-bit counter");
  // the columns each component's count kernel reads (trees 0 and 1; the logup program reads nothing else)
  std::vector<const u32*> cols_all;
  std::vector<size_t> cols_at(air.comps.size(), 0);
  for (size_t k = 0; k < air.comps.size(); ++k) {
    const AirComponent& c = air.comps[k];
    cols_at[k] = cols_all.size();
    for (const AirMask& mk : c.masks) {
      const u32* p = nullptr;
      if ((builds[k] || probes[k]) && mk.tree < 2) {
        NB_ARG(ctx, mk.col < flat[mk.tree].size(), "table_multiplicities: AIR references a missing trace column");
        NB_ARG(ctx, flog[mk.tree][mk.col] == c.log_size, "table_multiplicities: column size differs from the component's log_size");
        p = flat[mk.tree][mk.col];
      }
      cols_all.push_back(p);
    }
  }
  std::vector<const JitKernel*> jk(air.comps.size(), nullptr);
  for (size_t k = 0; k < air.comps.size(); ++k) {
    if (!builds[k] && !probes[k]) continue;
    jk[k] = ensure_jit(ctx, air_h, k, JIT_COUNT, false);
    if (!jk[k])
      return set_err(ctx, NB200_ERR_STATE, jit_enabled() ? "table_multiplicities: the count kernel could not be compiled: " + air_h->jit[JIT_COUNT][k].err
                                                         : std::string("table_multiplicities: the count runs only as a generated kernel (NB200_JIT=0)"));
  }
  // hash: at most half full; keys: relation, length, values per bin
  uint64_t cap = 1024;   // <= 2^31: the slot index and its mask fit 32 bits
  while (cap < 2 * n_bins) cap <<= 1;
  const u32 kw = 2 + max_len;
  std::vector<u32> tb;
  std::vector<size_t> tb_at(air.comps.size(), 0);
  for (size_t k = 0; k < air.comps.size(); ++k) { tb_at[k] = tb.size(); tb.insert(tb.end(), tbase[k].begin(), tbase[k].end()); }
  DevBuf d_slots, d_keys, d_cnt, d_um, d_tb;
  NB_TRY(alloc(ctx, d_slots, cap));
  NB_TRY(alloc(ctx, d_keys, n_bins * kw));
  NB_TRY(alloc(ctx, d_cnt, 2 * n_bins));
  NB_TRY(alloc(ctx, d_um, 4 + 1));
  NB_TRY(alloc(ctx, d_tb, std::max<size_t>(tb.size(), 1)));
  NB_CUDA(ctx, cudaMemsetAsync(d_slots.p, 0xff, (size_t)cap * 4, ctx->stream));
  NB_CUDA(ctx, cudaMemsetAsync(d_cnt.p, 0, n_bins * 8, ctx->stream));
  const uint64_t um_init[2] = {0, UINT64_MAX};
  NB_CUDA(ctx, cudaMemcpyAsync(d_um.p, um_init, 16, cudaMemcpyHostToDevice, ctx->stream));
  NB_CUDA(ctx, cudaMemsetAsync(d_um.p + 4, 0, 4, ctx->stream));
  if (!tb.empty()) NB_CUDA(ctx, cudaMemcpyAsync(d_tb.p, tb.data(), tb.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
  // component k's count kernel in `mode` (jit.cu gen_count_source); rows by a grid-stride loop: at most 8 CTAs per SM, so that the probe's
  // private bins are zeroed and flushed a bounded number of times
  const u32 mask = (u32)(cap - 1);
  unsigned long long *cnt = (unsigned long long*)d_cnt.p, *um_dev = (unsigned long long*)d_um.p;
  u32* err = d_um.p + 4;
  auto count = [&](size_t k, u32 mode, const u32* tbase, u32 nsh) {
    const size_t rows = (size_t)1 << jk[k]->log_size;
    const u32 block = (u32)std::min<size_t>(rows, 256);
    const u32 grid = (u32)std::min<size_t>((rows + block - 1) / block, (size_t)ctx->sm_count * 8);
    u32 comp = (u32)k;
    void* args[] = {(void*)&mode, (void*)&comp, (void*)&tbase, (void*)&d_slots.p, (void*)&d_keys.p, (void*)&kw, (void*)&mask,
                    (void*)&cnt, (void*)&nsh, (void*)&um_dev, (void*)&err};
    return jit_launch(ctx, *jk[k], cols_all.data() + cols_at[k], air.comps[k].masks.size(), dim3(grid), dim3(block), args, mode ? (size_t)nsh * 8 : 0);
  };
  trace_mark(ctx, nullptr);
  for (size_t k = 0; k < air.comps.size(); ++k)
    if (builds[k]) NB_TRY(count(k, 0, d_tb.p + tb_at[k], 0));
  // first_row: the build's duplicate flag is ignored; each key's slot is pointed at its first bin (owner: one u64 claim per slot, then the
  // count of distinct keys)
  DevBuf d_owner;
  std::vector<u32> tables;   // (first bin, log size) per table fraction, bin order
  if (first_row) {
    for (size_t t = 0, b = 0; t < mult.size(); b += (size_t)1 << mult[t].second, ++t) { tables.push_back((u32)b); tables.push_back(mult[t].second); }
    NB_TRY(alloc(ctx, d_owner, 2 * cap + 1 + tables.size()));
    unsigned long long* owner = (unsigned long long*)d_owner.p;
    u32 *distinct = d_owner.p + 2 * cap, *d_tables = distinct + 1;
    NB_CUDA(ctx, cudaMemsetAsync(owner, 0xff, (size_t)cap * 8, ctx->stream));
    NB_CUDA(ctx, cudaMemsetAsync(distinct, 0, 4, ctx->stream));
    NB_CUDA(ctx, cudaMemcpyAsync(d_tables, tables.data(), tables.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    NB_TRY(table_first_row_resolve(ctx, d_slots.p, d_keys.p, kw, cap, (u32)n_bins, d_tables, (u32)mult.size(), owner, distinct));
  } else {
    u32 dup = 0;
    NB_CUDA(ctx, cudaMemcpyAsync(&dup, d_um.p + 4, 4, cudaMemcpyDeviceToHost, ctx->stream));
    NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // also: the host tables above have been consumed
    if (dup) return set_err(ctx, NB200_ERR_ARG, "table_multiplicities: a table lists the same tuple in two rows of one relation");
  }
  // bins privatised per CTA when they fit in 32 KB of shared memory (the v1 machine's Range256 + Range32: 288 bins)
  const u32 nsh = n_bins * 8 <= 32768 ? (u32)n_bins : 0u;
  for (size_t k = 0; k < air.comps.size(); ++k)
    if (probes[k]) NB_TRY(count(k, 1, d_tb.p, nsh));
  uint64_t bin = 0;
  for (auto& m : mult) {
    NB_TRY(table_mult_store(ctx, m.first, (const unsigned long long*)d_cnt.p + bin, (size_t)1 << m.second));
    bin += (uint64_t)1 << m.second;
  }
  uint64_t um[2];
  u32 distinct = 0;
  NB_CUDA(ctx, cudaMemcpyAsync(um, d_um.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
  if (first_row) NB_CUDA(ctx, cudaMemcpyAsync(&distinct, d_owner.p + 2 * cap, 4, cudaMemcpyDeviceToHost, ctx->stream));
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // also: the host tables above have been consumed
  trace_mark(ctx, "table multiplicities");
  if (n_repeated) *n_repeated = n_bins - distinct;
  *n_unmatched = um[0];
  if (um[0]) { first[0] = (uint32_t)(um[1] >> 48); first[1] = (uint32_t)((um[1] >> 28) & 0xFFFFF); first[2] = (uint32_t)(um[1] & 0xFFFFFFF); }
  return NB200_OK;
}

// LogupTraceGenerator of the sharded (main) component: this rank runs the row kernel on ITS trace rows (all columns: the row slices kept by
// nb200_scheme_commit_sharded), the last secure column is all-gathered for the global claimed sum / coset-order prefix sum (finalize_last),
// and one rows -> columns exchange hands every rank its COLUMN shard of the 4 * n_logup interaction columns, ready for the next sharded commit.
nb200_status gen_interaction_sharded(nb200_scheme* s, nb200_air* air_h, u32 comp_idx, const std::vector<qm31>& params, nb200_cols** shard_out, qm31* claimed) {
  nb200_ctx* ctx = s->ctx;
  const AirProgram& air = air_h->prog;
  NB_ARG(ctx, comp_idx < air.comps.size() && s->trees.size() >= 2, "gen_interaction_sharded: commit trees 0 and 1 first");
  const AirComponent& c = air.comps[comp_idx];
  const u32 n = c.log_size, k = (u32)comm_log_world(ctx);
  const int world = comm_world(ctx), rank = comm_rank(ctx);
  NB_ARG(ctx, n >= k + 10, "gen_interaction_sharded: at least 1024 trace rows per rank");
  const size_t Sn = (size_t)1 << (n - k), N = (size_t)1 << n;
  const size_t ncols = c.n_logup_cols(), total = 4 * ncols;
  std::vector<const u32*> mask_cols(c.masks.size(), nullptr);
  for (size_t m = 0; m < c.masks.size(); ++m) {
    const AirMask& mk = c.masks[m];
    if (mk.tree == 2 || mk.off != 0) continue;
    const SchemeTree& tr = s->trees[mk.tree];
    NB_ARG(ctx, tr.sharded && mk.col < tr.cols.size() && tr.cols[mk.col].batch == SchemeTree::BIG && tr.big_eval_rows, "gen_interaction_sharded: the component may only read sharded trace columns (commit with keep_eval_rows)");
    mask_cols[m] = tr.big_eval_rows->col(tr.cols[mk.col].idx);   // this rank's trace rows
  }
  const JitKernel* jk = ensure_jit(ctx, air_h, comp_idx, JIT_LOGUP, false);
  NB_ARG(ctx, jk != nullptr, "gen_interaction_sharded needs the specialised logup kernel");
  DevBuf d_params;
  NB_TRY(upload_params(ctx, params.data(), params.size(), d_params));
  ColsPtr rows, last, shard;
  NB_TRY(alloc(ctx, rows, total, n - k));
  trace_mark(ctx, nullptr);
  NB_TRY(logup_rows(ctx, c, mask_cols, d_params.p, rows->d, n - k, jk));
  // finalize_last on the whole last secure column (every rank, redundantly), then this rank's rows go back into the row batch
  NB_TRY(alloc(ctx, last, 4, n));
  for (int q = 0; q < 4; ++q) NB_TRY(comm_all_gather_dev(ctx, rows->col(total - 4 + q), Sn, last->col(q)));
  NB_TRY(logup_finalize_last(ctx, n, last->d, claimed));
  for (int q = 0; q < 4; ++q)
    NB_CUDA(ctx, cudaMemcpyAsync(rows->col(total - 4 + q), last->col(q) + (size_t)rank * Sn, Sn * 4, cudaMemcpyDeviceToDevice, ctx->stream));
  trace_mark(ctx, "logup interaction trace (sharded rows)");
  // rows -> this rank's column shard
  size_t first = 0, count = 0;
  comm_shard_range(total, world, rank, &first, &count);
  PeerBuf pb_shard;
  size_t maxc = 0;
  for (int r = 0; r < world; ++r) { size_t f, cn; comm_shard_range(total, world, r, &f, &cn); maxc = std::max(maxc, cn); }
  NB_TRY(peer_alloc(ctx, s, maxc << n, &pb_shard));      // the same size on every rank (symmetric offsets)
  if (pb_shard.d) {
    // peer heap: my rows of rank q's columns go straight into q's shard (copy engines over NVLink); valid until the scheme is freed
    nb200_cols* sc = nullptr;
    NB_TRY(nb200_cols_from_device(ctx, pb_shard.d, count, n, &sc));
    shard.reset(sc);
    NB_TRY(comm_barrier_stream(ctx));
    NB_TRY(peer_rows_to_cols(ctx, ctx->stream, rows->d, total, N, pb_shard));
    NB_TRY(comm_barrier_stream(ctx));
  } else {
    NB_TRY(alloc(ctx, shard, count, n));
    NB_TRY(exchange_rows_to_cols(ctx, rows->d, total, N, shard->d));
  }
  cudaStreamSynchronize(ctx->stream);
  trace_mark(ctx, "logup: rows -> columns exchange");
  *shard_out = shard.release();
  return NB200_OK;
}

// the sample batches of nb200_fri_quotients(_from_coeffs): columns numbered through the device batches, each of 2^col_log words
static nb200_status sample_batches_of(nb200_ctx* ctx, const nb200_cols* const* batches, size_t n_batches, u32 col_log,
                                      const nb200_sample_batch* sample_batches, size_t n_sample_batches, const nb200_sample_entry* entries,
                                      size_t n_entries, std::vector<SampleBatch>& hb) {
  std::vector<const u32*> cols;
  for (size_t b = 0; b < n_batches; ++b) {
    NB_ARG(ctx, batches[b] && batches[b]->log_size == col_log, "fri_quotients: every column must have 2^log_size rows (from coefficients: 2^(log_size - log_blowup) words)");
    for (size_t c = 0; c < batches[b]->n_cols; ++c) cols.push_back(batches[b]->col(c));
  }
  hb.assign(n_sample_batches, SampleBatch{});
  for (size_t b = 0; b < n_sample_batches; ++b) {
    const nb200_sample_batch& sb = sample_batches[b];
    NB_ARG(ctx, sb.first_entry <= n_entries && sb.n_entries <= n_entries - sb.first_entry, "fri_quotients: sample batch entry range");
    memcpy(hb[b].p.x.c, sb.point, 16); memcpy(hb[b].p.y.c, sb.point + 4, 16);
    for (size_t e = sb.first_entry; e < sb.first_entry + sb.n_entries; ++e) {
      NB_ARG(ctx, entries[e].column < cols.size(), "fri_quotients: column index out of range");
      qm31 v; memcpy(v.c, entries[e].value, 16);
      hb[b].cols.push_back({cols[entries[e].column], v});
    }
  }
  return NB200_OK;
}

}  // namespace nb

using namespace nb;

extern "C" {

// ---- one proof over N GPUs: commit / interaction trace (nb200_prove itself needs no sharded twin: it follows the trees it finds) ----
nb200_status nb200_scheme_commit_sharded(nb200_scheme* s, const nb200_cols* big_shard, size_t total_big, uint32_t log_size, const nb200_cols* const* small, size_t n_small,
                                         const uint32_t* replicate_cols, size_t n_replicate, int keep_eval_rows, nb200_channel* channel, uint8_t root[32]) {
  if (!s || !channel || (n_small && !small) || (n_replicate && !replicate_cols)) return NB200_ERR_ARG;
  return scheme_commit_sharded(s, big_shard, total_big, log_size, small, n_small, replicate_cols, n_replicate, keep_eval_rows, channel->ch, root);
}
nb200_status nb200_gen_interaction_trace_sharded(nb200_scheme* s, const nb200_air* air, uint32_t component, const uint32_t* params, size_t n_params,
                                                 nb200_cols** shard_out, uint32_t claimed_sum[4]) {
  if (!s || !air || !shard_out || !claimed_sum) return NB200_ERR_ARG;
  std::vector<qm31> p(n_params);
  if (n_params) memcpy(p.data(), params, n_params * 16);
  qm31 cs;
  NB_TRY(gen_interaction_sharded(s, const_cast<nb200_air*>(air), component, p, shard_out, &cs));
  memcpy(claimed_sum, cs.c, 16);
  return NB200_OK;
}

// ---- Blake2sChannel (stwo core/channel/blake2s.rs) — machine.rs:197-206,240,262 ----
nb200_status nb200_channel_new(nb200_ctx* ctx, nb200_channel** out) {
  if (!out) return NB200_ERR_ARG;
  nb200_channel* c = new nb200_channel();
  if (ctx) c->ch.draw_domain_sep = ctx->draw_domain_sep;
  *out = c;
  return NB200_OK;
}
nb200_status nb200_channel_clone(const nb200_channel* c, nb200_channel** out) { if (!c || !out) return NB200_ERR_ARG; *out = new nb200_channel(*c); return NB200_OK; }
void nb200_channel_free(nb200_channel* c) { delete c; }
void nb200_channel_digest(const nb200_channel* c, uint8_t out[32]) { memcpy(out, c->ch.digest.data(), 32); }
void nb200_channel_mix_u64(nb200_channel* c, uint64_t v) { c->ch.mix_u64(v); }
void nb200_channel_mix_u32s(nb200_channel* c, const uint32_t* w, size_t n) { c->ch.mix_u32s(w, n); }
void nb200_channel_mix_felts(nb200_channel* c, const uint32_t* felts, size_t n) { c->ch.mix_u32s(felts, 4 * n); }
void nb200_channel_mix_root(nb200_channel* c, const uint8_t root[32]) { c->ch.mix_root(root); }
void nb200_channel_draw_felt(nb200_channel* c, uint32_t out[4]) { qm31 q = c->ch.draw_felt(); memcpy(out, q.c, 16); }
void nb200_channel_draw_felts(nb200_channel* c, size_t n, uint32_t* out) { std::vector<qm31> v(n); c->ch.draw_felts(n, v.data()); if (n) memcpy(out, v.data(), n * 16); }
void nb200_channel_draw_random_bytes(nb200_channel* c, uint8_t out[32]) { c->ch.draw_random_bytes(out); }
nb200_status nb200_device_channel_draw(nb200_ctx* ctx, const uint8_t digest[32], uint64_t n_sent, const uint8_t* roots, size_t n,
                                       uint32_t* felts_out, uint8_t digest_out[32], uint64_t* n_sent_out) {
  if (!ctx || !digest || n == 0 || !felts_out || !digest_out || !n_sent_out) return NB200_ERR_ARG;
  DevChannel st{};
  for (int i = 0; i < 8; ++i) st.digest[i] = (u32)digest[4 * i] | ((u32)digest[4 * i + 1] << 8) | ((u32)digest[4 * i + 2] << 16) | ((u32)digest[4 * i + 3] << 24);
  st.n_sent[0] = (u32)n_sent; st.n_sent[1] = (u32)(n_sent >> 32);
  DevBuf d;   // the state (16 words), the roots (8 words each), the records (12 words each)
  NB_TRY(alloc(ctx, d, 16 + 8 * n + 12 * n));
  u32* d_roots = d.p + 16;
  u32* d_rec = d_roots + 8 * n;
  NB_CUDA(ctx, cudaMemcpyAsync(d.p, &st, sizeof(st), cudaMemcpyHostToDevice, ctx->stream));
  if (roots) NB_CUDA(ctx, cudaMemcpyAsync(d_roots, roots, 32 * n, cudaMemcpyHostToDevice, ctx->stream));
  for (size_t i = 0; i < n; ++i)
    NB_TRY(channel_mix_draw(ctx, (DevChannel*)d.p, roots ? (const uint8_t*)(d_roots + 8 * i) : nullptr, d_rec + 12 * i, ctx->draw_domain_sep));
  std::vector<u32> rec(12 * n);
  NB_CUDA(ctx, cudaMemcpyAsync(rec.data(), d_rec, rec.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
  NB_CUDA(ctx, cudaMemcpyAsync(&st, d.p, sizeof(st), cudaMemcpyDeviceToHost, ctx->stream));
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (size_t i = 0; i < n; ++i) memcpy(felts_out + 4 * i, &rec[12 * i + 8], 16);
  for (int i = 0; i < 8; ++i) for (int b = 0; b < 4; ++b) digest_out[4 * i + b] = (uint8_t)(st.digest[i] >> (8 * b));
  *n_sent_out = (uint64_t)st.n_sent[0] | ((uint64_t)st.n_sent[1] << 32);
  return NB200_OK;
}

// ---- AIR ----
nb200_status nb200_air_load(nb200_ctx* ctx, const uint32_t* words, size_t n_words, nb200_air** out) {
  if (!out) return NB200_ERR_ARG;
  nb200_air* a = new nb200_air();
  try { a->prog = air_parse(words, n_words); a->fracs = air_lookup_tables(a->prog); *out = a; return NB200_OK; }
  catch (std::exception& e) { delete a; return set_err(ctx, NB200_ERR_ARG, e.what()); }
}
void nb200_air_free(nb200_air* a) { delete a; }
uint32_t nb200_air_n_params(const nb200_air* a) { return a ? a->prog.n_params : 0; }
uint32_t nb200_air_n_components(const nb200_air* a) { return a ? (uint32_t)a->prog.comps.size() : 0; }
uint64_t nb200_kernel_source_key(const char* src) { return src ? jit_source_key(src) : 0; }
uint32_t nb200_air_n_constraints(const nb200_air* a, uint32_t component) {
  return a && component < a->prog.comps.size() ? a->prog.comps[component].n_constraints : 0;
}
nb200_status nb200_air_constraint_degrees(const nb200_air* a, uint32_t component, uint32_t* degrees, size_t n) {
  if (!a || component >= a->prog.comps.size() || (n && !degrees)) return NB200_ERR_ARG;
  const std::vector<u32> d = constraint_degrees(a->prog.comps[component]);
  if (n != d.size()) return NB200_ERR_ARG;
  std::copy(d.begin(), d.end(), degrees);
  return NB200_OK;
}
nb200_status nb200_air_d2_masks(const nb200_air* a, uint32_t component, uint8_t* flags, size_t n) {
  if (!a || component >= a->prog.comps.size()) return NB200_ERR_ARG;
  const AirComponent& c = a->prog.comps[component];
  if (n != c.masks.size() || (n && !flags)) return NB200_ERR_ARG;
  const std::vector<char> used = masks_read_by(c, high_constraints(c));
  for (size_t m = 0; m < n; ++m) flags[m] = used[m] ? 1 : 0;
  return NB200_OK;
}
// the source the prover compiles for this kind and component; NB200_ERR_STATE when it compiles none (the interpreter runs the program, or
// there is nothing to evaluate)
static nb200_status kernel_source(const nb200_air* a, uint32_t component, JitKind kind, char** out) {
  const AirComponent& c = a->prog.comps[component];
  if (!jit_specialised(kind, c, a->fracs[component])) return NB200_ERR_STATE;
  const std::string src = jit_kernel_source(kind, c, a->fracs[component]);
  char* o = (char*)malloc(src.size() + 1);
  if (!o) return NB200_ERR_OOM;
  memcpy(o, src.c_str(), src.size() + 1);
  *out = o;
  return NB200_OK;
}
nb200_status nb200_air_kernel_source(const nb200_air* a, uint32_t component, int which, char** out) {
  if (!a || !out || component >= a->prog.comps.size() || which < 0 || which > 3) return NB200_ERR_ARG;
  *out = nullptr;
  return kernel_source(a, component, (JitKind)which, out);
}

// ---- CommitmentSchemeProver ----
nb200_status nb200_scheme_new(nb200_ctx* ctx, uint32_t pow_bits, uint32_t log_blowup, uint32_t log_last_layer_degree_bound, uint32_t n_queries, nb200_scheme** out) {
  if (!ctx || !out) return NB200_ERR_ARG;
  NB_ARG(ctx, log_blowup >= 1 && log_blowup <= 4 && n_queries >= 1 && log_last_layer_degree_bound <= 10, "scheme: config out of range");
  nb200_scheme* s = new nb200_scheme();
  s->ctx = ctx; s->pow_bits = pow_bits; s->log_blowup = log_blowup; s->log_last = log_last_layer_degree_bound; s->n_queries = n_queries;
  *out = s;
  return NB200_OK;
}
nb200_status nb200_scheme_set_constraint_log_degree(nb200_scheme* s, uint32_t log_expand) {
  if (!s) return NB200_ERR_ARG;
  s->hint_log_expand = log_expand;
  return NB200_OK;
}
uint32_t nb200_air_max_log_expand(const nb200_air* a) {
  uint32_t m = 0;
  if (a) for (auto& c : a->prog.comps) m = std::max<uint32_t>(m, c.log_expand);
  return m;
}
void nb200_scheme_free(nb200_scheme* s) {
  if (!s) return;
  s->trees.clear();
  peer_heap_release(s->ctx, s);
  delete s;
}
nb200_status nb200_scheme_commit(nb200_scheme* s, const nb200_cols* const* eval_batches, size_t n_batches, nb200_channel* channel, uint8_t root[32]) {
  if (!s || !channel) return NB200_ERR_ARG;
  return scheme_commit_evals(s, eval_batches, n_batches, channel->ch, root);
}
nb200_status nb200_scheme_commit_host(nb200_scheme* s, const uint32_t* const* host_batches, const size_t* n_cols, const uint32_t* log_sizes, size_t n_batches,
                                      int coset_order, nb200_channel* channel, uint8_t root[32], nb200_cols** evals_out) {
  if (!s || !channel || !host_batches || !evals_out) return NB200_ERR_ARG;
  return scheme_commit_host(s, (const void* const*)host_batches, nullptr, n_cols, log_sizes, n_batches, coset_order, channel->ch, root, evals_out);
}
nb200_status nb200_scheme_commit_host_packed(nb200_scheme* s, const void* const* host_batches, const uint32_t* elem_bytes, const size_t* n_cols, const uint32_t* log_sizes,
                                             size_t n_batches, int coset_order, nb200_channel* channel, uint8_t root[32], nb200_cols** evals_out) {
  if (!s || !channel || !host_batches || !evals_out) return NB200_ERR_ARG;
  for (size_t b = 0; elem_bytes && b < n_batches; ++b)
    if (!(elem_bytes[b] == 1 || elem_bytes[b] == 2 || elem_bytes[b] == 4)) return nb::set_err(s->ctx, NB200_ERR_ARG, "scheme_commit_host: 1, 2 or 4 bytes per host word");
  return scheme_commit_host(s, host_batches, elem_bytes, n_cols, log_sizes, n_batches, coset_order, channel->ch, root, evals_out);
}
nb200_status nb200_gen_interaction_trace(nb200_ctx* ctx, const nb200_air* air, uint32_t component, const nb200_cols* const* tree0, size_t n0,
                                         const nb200_cols* const* tree1, size_t n1, const uint32_t* params, size_t n_params,
                                         nb200_cols** out, uint32_t claimed_sum[4]) {
  if (!ctx || !air || !out) return NB200_ERR_ARG;
  std::vector<qm31> p(n_params);
  if (n_params) memcpy(p.data(), params, n_params * 16);
  qm31 cs;
  NB_TRY(gen_interaction(ctx, const_cast<nb200_air*>(air), component, tree0, n0, tree1, n1, p, out, &cs));
  memcpy(claimed_sum, cs.c, 16);
  return NB200_OK;
}
nb200_status nb200_prove(nb200_scheme* s, const nb200_air* air, const uint32_t* params, size_t n_params, nb200_channel* channel,
                         uint8_t** proof_out, size_t* proof_len) {
  if (!s || !air || !channel || !proof_out || !proof_len) return NB200_ERR_ARG;
  std::vector<qm31> p(n_params);
  if (n_params) memcpy(p.data(), params, n_params * 16);
  std::vector<uint8_t> bytes;
  NB_TRY(prove_impl(s, const_cast<nb200_air*>(air), p, channel->ch, bytes));
  uint8_t* o = (uint8_t*)malloc(bytes.size() ? bytes.size() : 1);
  memcpy(o, bytes.data(), bytes.size());
  *proof_out = o; *proof_len = bytes.size();
  return NB200_OK;
}
nb200_status nb200_check_constraints(nb200_ctx* ctx, const nb200_air* air, uint32_t component, const nb200_cols* const* tree0, size_t n0,
                                     const nb200_cols* const* tree1, size_t n1, const nb200_cols* const* tree2, size_t n2, const uint32_t* params,
                                     size_t n_params, uint64_t* n_failing, uint64_t* first_row, size_t n) {
  if (!ctx || !air || (n0 && !tree0) || (n1 && !tree1) || (n2 && !tree2) || (n_params && !params) || (n && (!n_failing || !first_row))) return NB200_ERR_ARG;
  const nb200_cols* const* trees[3] = {tree0, tree1, tree2};
  const size_t n_trees[3] = {n0, n1, n2};
  return check_constraints(ctx, const_cast<nb200_air*>(air), component, trees, n_trees, params, n_params, n_failing, first_row, n);
}
nb200_status nb200_table_multiplicities(nb200_ctx* ctx, const nb200_air* air, const nb200_cols* const* tree0, size_t n0, nb200_cols* const* tree1, size_t n1,
                                        uint64_t* n_unmatched, uint32_t first_unmatched[3]) {
  if (!ctx || !air || (n0 && !tree0) || (n1 && !tree1) || !n_unmatched || !first_unmatched) return NB200_ERR_ARG;
  const nb200_cols* const* trees[2] = {tree0, (const nb200_cols* const*)tree1};
  const size_t n_trees[2] = {n0, n1};
  return table_multiplicities(ctx, const_cast<nb200_air*>(air), trees, n_trees, n_unmatched, first_unmatched);
}
nb200_status nb200_table_multiplicities_first_row(nb200_ctx* ctx, const nb200_air* air, const nb200_cols* const* tree0, size_t n0,
                                                  nb200_cols* const* tree1, size_t n1, uint64_t* n_unmatched, uint32_t first_unmatched[3],
                                                  uint64_t* n_repeated) {
  if (!ctx || !air || (n0 && !tree0) || (n1 && !tree1) || !n_unmatched || !first_unmatched || !n_repeated) return NB200_ERR_ARG;
  const nb200_cols* const* trees[2] = {tree0, (const nb200_cols* const*)tree1};
  const size_t n_trees[2] = {n0, n1};
  return table_multiplicities(ctx, const_cast<nb200_air*>(air), trees, n_trees, n_unmatched, first_unmatched, true, n_repeated);
}
nb200_status nb200_air_lookup_tables(const nb200_air* a, uint32_t component, uint32_t* kind, uint32_t* relation, uint32_t* arg, size_t n) {
  if (!a || component >= a->prog.comps.size()) return NB200_ERR_ARG;
  const std::vector<AirFrac>& fr = a->fracs[component];
  if (n != fr.size() || (n && (!kind || !relation || !arg))) return NB200_ERR_ARG;
  const AirComponent& c = a->prog.comps[component];
  for (size_t i = 0; i < n; ++i) {
    kind[i] = fr[i].kind;
    relation[i] = fr[i].rel;
    arg[i] = fr[i].kind == FRAC_TABLE ? c.masks[fr[i].mult_mask].col : (u32)fr[i].tuple.size();
  }
  return NB200_OK;
}
nb200_status nb200_air_count_kernel_source(const nb200_air* a, uint32_t component, char** out) {
  if (!a || !out || component >= a->prog.comps.size()) return NB200_ERR_ARG;
  *out = nullptr;
  for (const AirFrac& f : a->fracs[component])
    if (f.kind == FRAC_BAD) return NB200_ERR_ARG;
  return kernel_source(a, component, JIT_COUNT, out);
}

// ---- backend-trait level operations (the per-trait surface a `CudaBackend` shim binds; the coarse nb200_prove runs the same code) ----
static bool secure4(const nb200_cols* c, u32 log) { return c && c->n_cols == 4 && c->log_size == log; }

nb200_status nb200_fold_line(nb200_ctx* ctx, const nb200_cols* src, const uint32_t alpha[4], nb200_cols** dst_out) {
  if (!ctx || !src || !alpha || !dst_out) return NB200_ERR_ARG;
  NB_ARG(ctx, src->n_cols == 4 && src->log_size >= 1, "fold_line: src must be a secure column (4 coordinate columns) of at least 2 values");
  NB_TRY(twiddles_prepare(ctx, src->log_size + 1));
  ColsPtr d;
  NB_TRY(alloc(ctx, d, 4, src->log_size - 1));
  qm31 a; memcpy(a.c, alpha, 16);
  NB_TRY(fold_line(ctx, d->d, src->d, src->log_size, a));
  *dst_out = d.release();
  return NB200_OK;
}
nb200_status nb200_fold_circle_into_line(nb200_ctx* ctx, nb200_cols* dst, const nb200_cols* src, const uint32_t alpha[4]) {
  if (!ctx || !dst || !src || !alpha) return NB200_ERR_ARG;
  NB_ARG(ctx, src->n_cols == 4 && src->log_size >= 3 && secure4(dst, src->log_size - 1), "fold_circle_into_line: src = 4 columns of 2^k (k >= 3), dst = 4 columns of 2^(k-1)");
  NB_TRY(twiddles_prepare(ctx, src->log_size));
  qm31 a; memcpy(a.c, alpha, 16);
  return fold_circle_into_line(ctx, dst->d, src->d, src->log_size, a);
}
nb200_status nb200_accumulate(nb200_ctx* ctx, nb200_cols* a, const nb200_cols* b) {
  if (!ctx || !a || !b) return NB200_ERR_ARG;
  NB_ARG(ctx, a->n_cols == b->n_cols && a->log_size == b->log_size, "accumulate: shape mismatch");
  return add_inplace(ctx, a->d, b->d, a->n_cols << a->log_size);
}
nb200_status nb200_grind(nb200_ctx* ctx, const uint8_t digest[32], uint32_t pow_bits, uint64_t* nonce_out) {
  if (!ctx || !digest || !nonce_out) return NB200_ERR_ARG;
  return grind(ctx, digest, pow_bits, nonce_out);
}
nb200_status nb200_fri_quotients(nb200_ctx* ctx, const nb200_cols* const* batches, size_t n_batches, uint32_t log_size,
                                 const nb200_sample_batch* sample_batches, size_t n_sample_batches,
                                 const nb200_sample_entry* entries, size_t n_entries, const uint32_t random_coeff[4], nb200_cols** out) {
  if (!ctx || (!batches && n_batches) || (!sample_batches && n_sample_batches) || (!entries && n_entries) || !random_coeff || !out) return NB200_ERR_ARG;
  std::vector<SampleBatch> hb;
  NB_TRY(sample_batches_of(ctx, batches, n_batches, log_size, sample_batches, n_sample_batches, entries, n_entries, hb));
  qm31 rc; memcpy(rc.c, random_coeff, 16);
  ColsPtr q;
  NB_TRY(alloc(ctx, q, 4, log_size));
  NB_TRY(accumulate_quotients(ctx, log_size, hb, rc, q->d));
  *out = q.release();
  return NB200_OK;
}
nb200_status nb200_fri_quotients_from_coeffs(nb200_ctx* ctx, const nb200_cols* const* coeffs, size_t n_batches, uint32_t log_size, uint32_t log_blowup,
                                             const nb200_sample_batch* sample_batches, size_t n_sample_batches,
                                             const nb200_sample_entry* entries, size_t n_entries, const uint32_t random_coeff[4], nb200_cols** out) {
  if (!ctx || (!coeffs && n_batches) || (!sample_batches && n_sample_batches) || (!entries && n_entries) || !random_coeff || !out) return NB200_ERR_ARG;
  NB_ARG(ctx, log_size >= log_blowup + 2 && n_sample_batches > 0, "fri_quotients_from_coeffs: at least one sample batch and 4 coefficients per column");
  std::vector<SampleBatch> hc;
  NB_TRY(sample_batches_of(ctx, coeffs, n_batches, log_size - log_blowup, sample_batches, n_sample_batches, entries, n_entries, hc));
  NB_TRY(twiddles_prepare(ctx, log_size));
  qm31 rc; memcpy(rc.c, random_coeff, 16);
  ColsPtr q;
  NB_TRY(alloc(ctx, q, 4, log_size));
  NB_TRY(quotients_from_coeffs(ctx, log_size, log_blowup, hc, rc, q->d));
  *out = q.release();
  return NB200_OK;
}
nb200_status nb200_deep_plan(const nb200_sample_batch* sample_batches, size_t n_sample_batches, const nb200_sample_entry* entries, size_t n_entries,
                             const uint32_t random_coeff[4], uint32_t* lines_out, uint32_t* alphas_out) {
  if ((!sample_batches && n_sample_batches) || (!entries && n_entries) || !random_coeff || (!lines_out && n_sample_batches) || (!alphas_out && n_entries))
    return NB200_ERR_ARG;
  std::vector<SampleBatch> hb(n_sample_batches);
  size_t total = 0;
  for (size_t b = 0; b < n_sample_batches; ++b) {
    const nb200_sample_batch& sb = sample_batches[b];
    if (sb.first_entry != total || sb.n_entries > n_entries - total) return NB200_ERR_ARG;
    memcpy(hb[b].p.x.c, sb.point, 16); memcpy(hb[b].p.y.c, sb.point + 4, 16);
    for (size_t e = sb.first_entry; e < sb.first_entry + sb.n_entries; ++e) {
      qm31 v; memcpy(v.c, entries[e].value, 16);
      hb[b].cols.push_back({nullptr, v});
    }
    total += sb.n_entries;
  }
  if (total != n_entries) return NB200_ERR_ARG;
  qm31 rc; memcpy(rc.c, random_coeff, 16);
  std::vector<QLineDev> lines; std::vector<QEntryDev> qe; std::vector<uint2> ranges;
  deep_plan(hb, rc, lines, qe, ranges);
  static_assert(sizeof(QLineDev) == 24 * 4, "QLineDev: 24 words");
  if (n_sample_batches) memcpy(lines_out, lines.data(), lines.size() * sizeof(QLineDev));
  for (size_t e = 0; e < qe.size(); ++e) memcpy(alphas_out + 4 * e, qe[e].c, 16);
  return NB200_OK;
}
nb200_status nb200_constraint_quotients(nb200_scheme* s, const nb200_air* air, uint32_t component, const uint32_t* params, size_t n_params,
                                        const uint32_t* coeffs, size_t n_coeffs, nb200_cols* accum) {
  if (!s || !air || !accum || (!coeffs && n_coeffs)) return NB200_ERR_ARG;
  nb200_ctx* ctx = s->ctx;
  NB_ARG(ctx, component < air->prog.comps.size(), "constraint quotients: component index");
  NB_ARG(ctx, !component_is_sharded(s, air->prog.comps[component]),
         "constraint quotients: the component reads sharded columns, which only the half-domain entry (nb200_constraint_quotients_half) evaluates");
  NB_ARG(ctx, n_params == air->prog.n_params, "constraint quotients: parameter table size");
  std::vector<qm31> cf(n_coeffs);
  if (n_coeffs) memcpy(cf.data(), coeffs, n_coeffs * 16);
  DevBuf d_params;
  NB_TRY(upload_params(ctx, params, n_params, d_params));
  NB_TRY(component_quotients(s, const_cast<nb200_air*>(air), component, d_params.p, cf, Q_FULL, accum, nullptr, nullptr));
  // params is caller memory: make sure the copy has been consumed before returning
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return NB200_OK;
}
nb200_status nb200_constraint_quotients_half(nb200_scheme* s, const nb200_air* air, uint32_t component, const uint32_t* params, size_t n_params,
                                             const uint32_t* coeffs, size_t n_coeffs, nb200_cols* q_d1, nb200_cols* q_high_d2, nb200_cols* q_high_d1) {
  if (!s || !air || !q_d1 || !q_high_d2 || !q_high_d1 || (!coeffs && n_coeffs)) return NB200_ERR_ARG;
  nb200_ctx* ctx = s->ctx;
  NB_ARG(ctx, component < air->prog.comps.size(), "constraint quotients: component index");
  NB_ARG(ctx, quotient_mode(s, air->prog.comps[component]) == Q_HALF, "constraint quotients (half domains): nb200_prove evaluates this component with Q_FULL");
  NB_ARG(ctx, n_params == air->prog.n_params, "constraint quotients: parameter table size");
  std::vector<qm31> cf(n_coeffs);
  if (n_coeffs) memcpy(cf.data(), coeffs, n_coeffs * 16);
  DevBuf d_params;
  NB_TRY(upload_params(ctx, params, n_params, d_params));
  // the same dispatch as commit_composition: a component that reads sharded columns takes the sharded route
  nb200_air* air_h = const_cast<nb200_air*>(air);
  if (component_is_sharded(s, air->prog.comps[component])) NB_TRY(component_quotients_sharded(s, air_h, component, d_params.p, cf, q_d1, q_high_d2, q_high_d1));
  else NB_TRY(component_quotients(s, air_h, component, d_params.p, cf, Q_HALF, q_d1, q_high_d2, q_high_d1));
  NB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return NB200_OK;
}

}  // extern "C"
