// ORACLE — TEST INFRASTRUCTURE ONLY (see fields.h header).  C entry points for ctypes, used solely by
// tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
#include "vcs.h"
#include "prove.h"
#include <memory>
#include <mutex>
#ifdef _OPENMP
#include <omp.h>
#endif

using namespace orc;

static std::map<uint32_t, std::shared_ptr<TwiddleTree>>& tw_cache() { static std::map<uint32_t, std::shared_ptr<TwiddleTree>> m; return m; }
static std::mutex tw_mu;
static const TwiddleTree& orc_get_twiddles(uint32_t domain_log);
namespace orc { const TwiddleTree& get_twiddles(uint32_t domain_log) { return orc_get_twiddles(domain_log); } }
// twiddle tree whose root is the half coset of the canonic circle domain of `domain_log`
static const TwiddleTree& orc_get_twiddles(uint32_t domain_log) {
  std::lock_guard<std::mutex> g(tw_mu);
  auto& m = tw_cache();
  // any cached bigger tree works (suffix property) but keep it simple/explicit: exact size
  auto it = m.find(domain_log);
  if (it == m.end()) {
    auto t = std::make_shared<TwiddleTree>(precompute_twiddles(CanonicCoset(domain_log).circle_domain().half_coset));
    it = m.emplace(domain_log, t).first;
  }
  return *it->second;
}

extern "C" {

int orc_num_threads() {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}
void orc_set_num_threads(int n) {
#ifdef _OPENMP
  omp_set_num_threads(n);
#else
  (void)n;
#endif
}
void orc_set_flavor(int merkle_hash, int draw_domain_sep, int pow_variant) {
  flavor().merkle_hash = merkle_hash; flavor().draw_domain_sep = draw_domain_sep; flavor().pow_variant = pow_variant;
}

// ---- fields (for the field-axiom tests) ----
uint32_t orc_m31_mul(uint32_t a, uint32_t b) { return (M31::raw(a) * M31::raw(b)).v; }
uint32_t orc_m31_inv(uint32_t a) { return inv(M31::raw(a)).v; }
void orc_qm31_mul(const uint32_t a[4], const uint32_t b[4], uint32_t out[4]) {
  QM31 r = QM31::from_u32(a[0], a[1], a[2], a[3]) * QM31::from_u32(b[0], b[1], b[2], b[3]);
  for (int k = 0; k < 4; ++k) out[k] = r.coord(k);
}
void orc_qm31_inv(const uint32_t a[4], uint32_t out[4]) {
  QM31 r = inv(QM31::from_u32(a[0], a[1], a[2], a[3]));
  for (int k = 0; k < 4; ++k) out[k] = r.coord(k);
}

// ---- circle ----
void orc_circle_domain_at(uint32_t log_size, uint64_t i, uint32_t out_xy[2]) {
  CirclePoint<M31> p = CanonicCoset(log_size).circle_domain().at(i);
  out_xy[0] = p.x.v; out_xy[1] = p.y.v;
}
uint64_t orc_bit_reverse_index(uint64_t i, uint32_t log_size) { return bit_reverse_index(i, log_size); }
uint64_t orc_coset_index_to_circle_domain_index(uint64_t i, uint32_t log_size) { return coset_index_to_circle_domain_index(i, log_size); }
// reference finalize_columns: coset order -> circle-domain order -> bit reverse
void orc_finalize_column(const uint32_t* in, uint32_t log_size, uint32_t* out) {
  size_t n = (size_t)1 << log_size;
  std::vector<uint32_t> v(in, in + n);
  std::vector<uint32_t> r = coset_order_to_circle_domain_order(v);
  bit_reverse(r);
  memcpy(out, r.data(), n * 4);
}

// ---- poly ----
void orc_twiddles(uint32_t domain_log, uint32_t* tw, uint32_t* itw) {
  const TwiddleTree& t = orc_get_twiddles(domain_log);
  for (size_t i = 0; i < t.twiddles.size(); ++i) { tw[i] = t.twiddles[i].v; itw[i] = t.itwiddles[i].v; }
}
void orc_interpolate(uint32_t log_size, const uint32_t* evals, uint32_t* coeffs) {
  const TwiddleTree& t = orc_get_twiddles(log_size);
  size_t n = (size_t)1 << log_size;
  Col v(n); for (size_t i = 0; i < n; ++i) v[i] = M31::raw(evals[i]);
  Col c = interpolate(CanonicCoset(log_size).circle_domain(), std::move(v), t);
  for (size_t i = 0; i < n; ++i) coeffs[i] = c[i].v;
}
void orc_evaluate(uint32_t coeff_log, uint32_t domain_log, const uint32_t* coeffs, uint32_t* evals) {
  const TwiddleTree& t = orc_get_twiddles(domain_log);
  size_t n = (size_t)1 << coeff_log;
  Col c(n); for (size_t i = 0; i < n; ++i) c[i] = M31::raw(coeffs[i]);
  Col v = evaluate(CanonicCoset(domain_log).circle_domain(), c, t);
  for (size_t i = 0; i < v.size(); ++i) evals[i] = v[i].v;
}
// batched, OpenMP over columns (cpu_baseline): evals (n_cols x 2^log) -> lde (n_cols x 2^(log+blowup)); column-major contiguous
void orc_interpolate_evaluate_batch(uint32_t log_size, uint32_t log_blowup, size_t n_cols, const uint32_t* evals, uint32_t* coeffs_out, uint32_t* lde_out) {
  const TwiddleTree& t1 = orc_get_twiddles(log_size);
  const TwiddleTree& t2 = orc_get_twiddles(log_size + log_blowup);
  size_t n = (size_t)1 << log_size, m = (size_t)1 << (log_size + log_blowup);
  CircleDomain d1 = CanonicCoset(log_size).circle_domain(), d2 = CanonicCoset(log_size + log_blowup).circle_domain();
#pragma omp parallel for schedule(dynamic)
  for (size_t c = 0; c < n_cols; ++c) {
    Col v(n); for (size_t i = 0; i < n; ++i) v[i] = M31::raw(evals[c * n + i]);
    Col co = interpolate(d1, std::move(v), t1);
    if (coeffs_out) for (size_t i = 0; i < n; ++i) coeffs_out[c * n + i] = co[i].v;
    Col e = evaluate(d2, co, t2);
    for (size_t i = 0; i < m; ++i) lde_out[c * m + i] = e[i].v;
  }
}
void orc_eval_at_point(uint32_t log_size, const uint32_t* coeffs, const uint32_t px[4], const uint32_t py[4], uint32_t out[4]) {
  size_t n = (size_t)1 << log_size;
  Col c(n); for (size_t i = 0; i < n; ++i) c[i] = M31::raw(coeffs[i]);
  QM31 r = eval_at_point(c, CirclePoint<QM31>(QM31::from_u32(px[0], px[1], px[2], px[3]), QM31::from_u32(py[0], py[1], py[2], py[3])));
  for (int k = 0; k < 4; ++k) out[k] = r.coord(k);
}

// ---- hash / merkle ----
void orc_blake2s(const uint8_t* data, size_t len, uint8_t out[32]) { Hash32 h = blake2s_hash(data, len); memcpy(out, h.data(), 32); }
void orc_blake2s_compress(uint32_t h[8], const uint32_t m[16], uint32_t t0, uint32_t t1, uint32_t f0, uint32_t f1) { b2s_compress(h, m, t0, t1, f0, f1); }

// columns: n_cols pointers, log sizes. layers_out (optional): concatenated layers from root (1 hash) to leaves.
void orc_merkle_commit(size_t n_cols, const uint32_t* const* cols, const uint32_t* log_sizes, uint8_t root[32], uint8_t* layers_out) {
  std::vector<Col> store(n_cols);
  std::vector<const Col*> ptrs(n_cols);
  for (size_t c = 0; c < n_cols; ++c) {
    size_t n = (size_t)1 << log_sizes[c];
    store[c].resize(n);
    for (size_t i = 0; i < n; ++i) store[c][i] = M31::raw(cols[c][i]);
    ptrs[c] = &store[c];
  }
  MerkleProver mp = MerkleProver::commit(ptrs);
  memcpy(root, mp.root().data(), 32);
  if (layers_out) {
    size_t off = 0;
    for (auto& L : mp.layers) { memcpy(layers_out + off, L.data(), L.size() * 32); off += L.size() * 32; }
  }
}

// Decommit: queries given per log size as (log_sizes_q[k], positions concatenated with counts).
// Outputs are written to caller buffers with lengths returned through *n_*.
void orc_merkle_decommit(size_t n_cols, const uint32_t* const* cols, const uint32_t* log_sizes,
                         size_t n_q_sizes, const uint32_t* q_log_sizes, const uint64_t* q_counts, const uint64_t* q_positions,
                         uint32_t* queried_values, size_t* n_queried, uint8_t* hash_witness, size_t* n_hash, uint32_t* column_witness, size_t* n_colw) {
  std::vector<Col> store(n_cols);
  std::vector<const Col*> ptrs(n_cols);
  for (size_t c = 0; c < n_cols; ++c) {
    size_t n = (size_t)1 << log_sizes[c];
    store[c].resize(n);
    for (size_t i = 0; i < n; ++i) store[c][i] = M31::raw(cols[c][i]);
    ptrs[c] = &store[c];
  }
  MerkleProver mp = MerkleProver::commit(ptrs);
  std::map<uint32_t, std::vector<size_t>> q;
  size_t off = 0;
  for (size_t k = 0; k < n_q_sizes; ++k) {
    std::vector<size_t> v(q_positions + off, q_positions + off + q_counts[k]);
    off += q_counts[k];
    q[q_log_sizes[k]] = v;
  }
  auto res = mp.decommit(q, ptrs);
  *n_queried = res.first.size(); *n_hash = res.second.hash_witness.size(); *n_colw = res.second.column_witness.size();
  for (size_t i = 0; i < res.first.size(); ++i) queried_values[i] = res.first[i].v;
  for (size_t i = 0; i < res.second.hash_witness.size(); ++i) memcpy(hash_witness + 32 * i, res.second.hash_witness[i].data(), 32);
  for (size_t i = 0; i < res.second.column_witness.size(); ++i) column_witness[i] = res.second.column_witness[i].v;
}

// ---- channel (opaque handle) ----
void* orc_channel_new() { return new Channel(); }
void orc_channel_free(void* c) { delete (Channel*)c; }
void orc_channel_digest(void* c, uint8_t out[32]) { memcpy(out, ((Channel*)c)->digest.data(), 32); }
void orc_channel_mix_u64(void* c, uint64_t v) { ((Channel*)c)->mix_u64(v); }
void orc_channel_mix_u32s(void* c, const uint32_t* w, size_t n) { ((Channel*)c)->mix_u32s(w, n); }
void orc_channel_mix_felts(void* c, const uint32_t* felts, size_t n) {
  std::vector<QM31> f(n);
  for (size_t i = 0; i < n; ++i) f[i] = QM31::from_u32(felts[4 * i], felts[4 * i + 1], felts[4 * i + 2], felts[4 * i + 3]);
  ((Channel*)c)->mix_felts(f);
}
void orc_channel_mix_root(void* c, const uint8_t root[32]) { Hash32 h; memcpy(h.data(), root, 32); ((Channel*)c)->mix_root(h); }
void orc_channel_draw_felt(void* c, uint32_t out[4]) { QM31 q = ((Channel*)c)->draw_felt(); for (int k = 0; k < 4; ++k) out[k] = q.coord(k); }
void orc_channel_draw_felts(void* c, size_t n, uint32_t* out) {
  auto v = ((Channel*)c)->draw_felts(n);
  for (size_t i = 0; i < n; ++i) for (int k = 0; k < 4; ++k) out[4 * i + k] = v[i].coord(k);
}
void orc_channel_draw_random_bytes(void* c, uint8_t out[32]) { Hash32 h = ((Channel*)c)->draw_random_bytes(); memcpy(out, h.data(), 32); }

}  // extern "C"

// ---- prove / verify -------------------------------------------------------------------------------
#include "verify.h"

namespace {
struct OrcProver {
  Air air;
  std::vector<Tree> trees;
  std::vector<std::vector<Col>> trace_evals;  // [tree][col]: the committed evaluations (for logup generation)
};
std::string g_err;

struct PostcardReader {
  const uint8_t* p; size_t n, i = 0;
  uint64_t varint() { uint64_t v = 0; int s = 0; while (true) { if (i >= n) throw std::runtime_error("postcard: truncated"); uint8_t b = p[i++]; v |= (uint64_t)(b & 0x7f) << s; if (!(b & 0x80)) return v; s += 7; if (s > 63) throw std::runtime_error("postcard: varint too long"); } }
  M31 m31() { uint64_t v = varint(); if (v >= P) throw std::runtime_error("postcard: M31 out of range"); return M31::raw((uint32_t)v); }
  QM31 qm31() { M31 a = m31(), b = m31(), c = m31(), d = m31(); return QM31(CM31(a, b), CM31(c, d)); }
  Hash32 hash() { if (i + 32 > n) throw std::runtime_error("postcard: truncated hash"); Hash32 h; memcpy(h.data(), p + i, 32); i += 32; return h; }
  MerkleDecommitment decommitment() {
    MerkleDecommitment d; size_t nh = varint(); for (size_t k = 0; k < nh; ++k) d.hash_witness.push_back(hash());
    size_t nc = varint(); for (size_t k = 0; k < nc; ++k) d.column_witness.push_back(m31());
    return d;
  }
  FriLayerProof fri_layer() { FriLayerProof l; size_t nw = varint(); for (size_t k = 0; k < nw; ++k) l.fri_witness.push_back(qm31()); l.decommitment = decommitment(); l.commitment = hash(); return l; }
  Proof proof() {
    Proof pr;
    pr.config.pow_bits = (uint32_t)varint(); pr.config.fri.log_blowup_factor = (uint32_t)varint();
    pr.config.fri.log_last_layer_degree_bound = (uint32_t)varint(); pr.config.fri.n_queries = (uint32_t)varint();
    size_t nc = varint(); for (size_t k = 0; k < nc; ++k) pr.commitments.push_back(hash());
    size_t nt = varint(); pr.sampled_values.resize(nt);
    for (auto& t : pr.sampled_values) { t.resize(varint()); for (auto& c : t) { c.resize(varint()); for (auto& q : c) q = qm31(); } }
    size_t nd = varint(); for (size_t k = 0; k < nd; ++k) pr.decommitments.push_back(decommitment());
    size_t nq = varint(); pr.queried_values.resize(nq);
    for (auto& t : pr.queried_values) { t.resize(varint()); for (auto& v : t) v = m31(); }
    pr.proof_of_work = varint();
    pr.fri_proof.first_layer = fri_layer();
    size_t ni = varint(); for (size_t k = 0; k < ni; ++k) pr.fri_proof.inner_layers.push_back(fri_layer());
    size_t nl = varint(); for (size_t k = 0; k < nl; ++k) pr.fri_proof.last_layer_poly.push_back(qm31());
    pr.fri_proof.last_layer_log_size = (uint32_t)varint();
    if (i != n) throw std::runtime_error("postcard: trailing bytes");
    return pr;
  }
};
std::vector<QM31> read_params(const uint32_t* p, size_t n) { std::vector<QM31> v(n); for (size_t i = 0; i < n; ++i) v[i] = QM31::from_u32(p[4 * i], p[4 * i + 1], p[4 * i + 2], p[4 * i + 3]); return v; }
}  // namespace

extern "C" {

const char* orc_last_error() { return g_err.c_str(); }

void* orc_prover_new(const uint32_t* air_words, size_t n) {
  try { OrcProver* p = new OrcProver(); p->air = Air::parse(air_words, n); return p; }
  catch (std::exception& e) { g_err = e.what(); return nullptr; }
}
void orc_prover_free(void* p) { delete (OrcProver*)p; }

// TreeBuilder::extend_evals + commit (machine.rs:208-263): interpolate, LDE, Merkle, mix_root
int orc_prover_commit(void* pp, void* ch, size_t n_cols, const uint32_t* const* cols, const uint32_t* logs, uint32_t log_blowup, uint8_t root[32]) {
  try {
    OrcProver* p = (OrcProver*)pp;
    std::vector<Col> ev(n_cols);
    for (size_t c = 0; c < n_cols; ++c) { size_t n = (size_t)1 << logs[c]; ev[c].resize(n); for (size_t i = 0; i < n; ++i) ev[c][i] = M31::raw(cols[c][i]); }
    p->trees.push_back(commit_evals(ev, log_blowup, *(Channel*)ch));
    p->trace_evals.push_back(std::move(ev));
    memcpy(root, p->trees.back().merkle.root().data(), 32);
    return 0;
  } catch (std::exception& e) { g_err = e.what(); return 1; }
}

// generate_interaction_trace for one component (traits.rs:124-145 semantics via LogupTraceGenerator)
int orc_prover_gen_interaction(void* pp, uint32_t comp, const uint32_t* params, size_t n_params, uint32_t* out_cols, uint32_t claimed[4]) {
  try {
    OrcProver* p = (OrcProver*)pp;
    const Component& c = p->air.comps.at(comp);
    std::vector<std::vector<Col>> te = p->trace_evals;
    te.resize(3);
    auto r = gen_interaction_trace(c, te, read_params(params, n_params));
    size_t n = (size_t)1 << c.log_size;
    for (size_t k = 0; k < r.first.size(); ++k) for (size_t i = 0; i < n; ++i) out_cols[k * n + i] = r.first[k][i].v;
    for (int k = 0; k < 4; ++k) claimed[k] = r.second.coord(k);
    return 0;
  } catch (std::exception& e) { g_err = e.what(); return 1; }
}

// stwo::prover::prove (machine.rs:286-290) -> postcard bytes of StarkProof
int orc_prover_prove(void* pp, void* ch, const uint32_t* params, size_t n_params, uint32_t pow_bits, uint32_t log_blowup, uint32_t log_last, uint32_t n_queries,
                     uint8_t* out, size_t cap, size_t* len) {
  try {
    OrcProver* p = (OrcProver*)pp;
    PcsConfig cfg; cfg.pow_bits = pow_bits; cfg.fri.log_blowup_factor = log_blowup; cfg.fri.log_last_layer_degree_bound = log_last; cfg.fri.n_queries = n_queries;
    Proof pr = prove(p->air, read_params(params, n_params), p->trees, *(Channel*)ch, cfg);
    Postcard pc; pc.proof(pr);
    *len = pc.out.size();
    if (pc.out.size() > cap) { g_err = "proof buffer too small"; return 2; }
    memcpy(out, pc.out.data(), pc.out.size());
    return 0;
  } catch (ProveError& e) { g_err = e.what(); return 5; }
  catch (std::exception& e) { g_err = e.what(); return 1; }
}

// verify postcard proof bytes; `ch` must be in the state the prover's channel had when prove() started
int orc_verify(const uint32_t* air_words, size_t n_air, const uint32_t* params, size_t n_params, const uint8_t* proof, size_t proof_len,
               void* ch, const uint32_t* n_cols_per_tree /*3*/, const uint32_t* col_logs_flat) {
  try {
    Air air = Air::parse(air_words, n_air);
    PostcardReader rd{proof, proof_len};
    Proof pr = rd.proof();
    // re-encoding must reproduce the bytes (canonical encoding)
    Postcard pc; pc.proof(pr);
    if (pc.out.size() != proof_len || memcmp(pc.out.data(), proof, proof_len) != 0) throw VerifyError("postcard: non-canonical encoding");
    std::vector<std::vector<uint32_t>> logs(3);
    size_t off = 0;
    for (int t = 0; t < 3; ++t) { logs[t].assign(col_logs_flat + off, col_logs_flat + off + n_cols_per_tree[t]); off += n_cols_per_tree[t]; }
    verify(air, read_params(params, n_params), pr, *(Channel*)ch, logs);
    return 0;
  } catch (std::exception& e) { g_err = e.what(); return 1; }
}

void* orc_channel_clone(void* c) { return new Channel(*(Channel*)c); }

// ---- backend-trait level operations (FriOps / QuotientOps / AccumulationOps / GrindOps / ComponentProver), used by the
// op-level parity tests of the C ABI.  Secure columns travel as 4 coordinate columns: buf[k * n + i].
namespace {
SecureCol read_secure(const uint32_t* buf, size_t n) { SecureCol s; s.resize(n); for (int k = 0; k < 4; ++k) for (size_t i = 0; i < n; ++i) s.c[k][i] = M31::raw(buf[k * n + i]); return s; }
void write_secure(const SecureCol& s, uint32_t* buf) { size_t n = s.size(); for (int k = 0; k < 4; ++k) for (size_t i = 0; i < n; ++i) buf[k * n + i] = s.c[k][i].v; }
QM31 read_q(const uint32_t* p) { return QM31::from_u32(p[0], p[1], p[2], p[3]); }
}

// FriOps::fold_line on LineDomain(Coset::half_odds(log_size)) (the domain FriProver::commit walks)
void orc_fold_line(uint32_t log_size, const uint32_t* src, const uint32_t alpha[4], uint32_t* dst) {
  size_t n = (size_t)1 << log_size;
  SecureCol s = read_secure(src, n);
  LineEval e; e.domain = LineDomain(Coset::half_odds(log_size)); e.values.resize(n);
  for (size_t i = 0; i < n; ++i) e.values[i] = s.at(i);
  LineEval o = fold_line(e, read_q(alpha));
  write_secure(to_secure_col(o.values), dst);
}

// FriOps::fold_circle_into_line: dst (2^(src_log-1) values, in/out) = dst * alpha^2 + fold(src)
void orc_fold_circle_into_line(uint32_t src_log, uint32_t* dst, const uint32_t* src, const uint32_t alpha[4]) {
  size_t n = (size_t)1 << src_log;
  SecureCol s = read_secure(src, n), d = read_secure(dst, n / 2);
  LineEval e; e.domain = LineDomain(Coset::half_odds(src_log - 1)); e.values.resize(n / 2);
  for (size_t i = 0; i < n / 2; ++i) e.values[i] = d.at(i);
  fold_circle_into_line(e, s, src_log, read_q(alpha));
  write_secure(to_secure_col(e.values), dst);
}

// QuotientOps::accumulate_quotients; batch b covers entries [first[b], first[b] + count[b]); entry = (column index, sampled value)
void orc_accumulate_quotients(uint32_t log_size, size_t n_cols, const uint32_t* const* cols, const uint32_t random_coeff[4],
                              size_t n_batches, const uint32_t* points /*8 per batch: x[4], y[4]*/, const uint64_t* first, const uint64_t* count,
                              const uint32_t* entry_cols, const uint32_t* entry_values /*4 per entry*/, uint32_t* out) {
  size_t n = (size_t)1 << log_size;
  std::vector<Col> c(n_cols);
  for (size_t k = 0; k < n_cols; ++k) { c[k].resize(n); for (size_t i = 0; i < n; ++i) c[k][i] = M31::raw(cols[k][i]); }
  std::vector<const Col*> cp; for (auto& x : c) cp.push_back(&x);
  std::vector<ColumnSampleBatch> batches(n_batches);
  for (size_t b = 0; b < n_batches; ++b) {
    batches[b].point = CirclePoint<QM31>{read_q(points + 8 * b), read_q(points + 8 * b + 4)};
    for (uint64_t e = first[b]; e < first[b] + count[b]; ++e) batches[b].cols.push_back({(size_t)entry_cols[e], read_q(entry_values + 4 * e)});
  }
  write_secure(accumulate_quotients(log_size, cp, read_q(random_coeff), batches), out);
}

// GrindOps::grind on a channel whose digest is `digest`
uint64_t orc_grind(const uint8_t digest[32], uint32_t pow_bits) {
  Channel ch; memcpy(ch.digest.data(), digest, 32);
  return grind(ch, pow_bits);
}

// ComponentProver::evaluate_constraint_quotients_on_domain for component `comp` over the prover's committed trees, on
// CanonicCoset(eval_log).circle_domain() (eval_log = 0: the component's own, log_size + log_expand; any eval_log > log_size):
// accum (4 coordinate columns of 2^eval_log, in/out) += quotients
int orc_prover_constraint_quotients(void* pp, uint32_t comp, uint32_t eval_log, const uint32_t* params, size_t n_params, const uint32_t* coeffs /*4 per constraint*/,
                                    uint32_t* accum) {
  try {
    OrcProver* p = (OrcProver*)pp;
    const Component& c = p->air.comps.at(comp);
    if (eval_log == 0) eval_log = c.eval_log();
    size_t en = (size_t)1 << eval_log;
    SecureCol acc = read_secure(accum, en);
    std::vector<QM31> coeff(c.n_constraints);
    for (uint32_t k = 0; k < c.n_constraints; ++k) coeff[k] = read_q(coeffs + 4 * k);
    component_quotients(c, p->trees, read_params(params, n_params), coeff, acc, eval_log);
    write_secure(acc, accum);
    return 0;
  } catch (std::exception& e) { g_err = e.what(); return 1; }
}

// ColumnOps::bit_reverse_column
void orc_bit_reverse_column(uint32_t* col, uint32_t log_size) {
  size_t n = (size_t)1 << log_size;
  for (size_t i = 0; i < n; ++i) { size_t j = bit_reverse_index(i, log_size); if (i < j) std::swap(col[i], col[j]); }
}

}  // extern "C"
