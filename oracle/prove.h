// ORACLE — TEST INFRASTRUCTURE ONLY (see fields.h header).  PARITY UNPINNED: the reference pins no proof
// bytes (SURVEY.md §0 F4); every [risk] item of SURVEY Appendix A is called out where it is decided.
// Restates the rest of stwo @0790eba's prover as driven by nexus-zkvm prover/src/machine.rs:130-297:
//   constraint-framework FrameworkComponent (domain + point evaluation, logup constraints)  — here over a
//     bytecode AIR, because the reference's AIR is Rust generic code that cannot be executed in this image;
//   prover/air/accumulation.rs (DomainEvaluationAccumulator), prover/mod.rs (prove), prover/pcs (prove_values),
//   core/pcs/quotients.rs + backend/cpu/quotients.rs, prover/fri.rs + core/fri.rs, core/queries.rs,
//   core/proof_of_work / GrindOps, core/proof.rs (+ postcard encoding), constraint-framework logup.rs
//   (LogupTraceGenerator) and a verifier (core/verifier.rs, core/pcs/verifier.rs, core/fri.rs verifier half).
#pragma once
#include "vcs.h"
#include <stdexcept>
#include <memory>
#include <functional>
#include <set>
#include <string>

namespace orc {

// ---------------------------------------------------------------------------------------------------
// config  (stwo core/pcs/mod.rs PcsConfig::default(), core/fri.rs FriConfig)            [risk A.4]
struct FriConfig {
  uint32_t log_blowup_factor = 1, log_last_layer_degree_bound = 0;
  uint32_t n_queries = 3;
  size_t last_layer_domain_size() const { return (size_t)1 << (log_last_layer_degree_bound + log_blowup_factor); }
};
struct PcsConfig { uint32_t pow_bits = 5; FriConfig fri; };

struct SecureCol {  // SecureColumnByCoords
  Col c[4];
  size_t size() const { return c[0].size(); }
  void resize(size_t n) { for (auto& x : c) x.assign(n, M31()); }
  QM31 at(size_t i) const { return QM31(CM31(c[0][i], c[1][i]), CM31(c[2][i], c[3][i])); }
  void set(size_t i, QM31 v) { c[0][i] = v.a.a; c[1][i] = v.a.b; c[2][i] = v.b.a; c[3][i] = v.b.b; }
};
inline QM31 from_partial_evals(const QM31 v[4]) {
  // v0 + v1*i + v2*u + v3*i*u
  QM31 I = QM31::from_u32(0, 1, 0, 0), U = QM31::from_u32(0, 0, 1, 0), IU = QM31::from_u32(0, 0, 0, 1);
  return v[0] + v[1] * I + v[2] * U + v[3] * IU;
}

// ---------------------------------------------------------------------------------------------------
// AIR bytecode (format documented in DESIGN.md §AIR bytecode; emitted by nexus_zkvm_b200/air.py, the stand-in
// for a recording `EvalAtRow` on the Rust side — SURVEY.md §7.3-4)
enum Op : uint32_t {
  OP_LOADM = 0, OP_CONSTB = 1, OP_ADDB = 2, OP_SUBB = 3, OP_MULB = 4, OP_NEGB = 5,
  OP_PARAME = 6, OP_ADDE = 8, OP_SUBE = 9, OP_MULE = 10, OP_NEGE = 11,
  OP_ADDEB = 12, OP_SUBEB = 13, OP_MULEB = 14, OP_BTOE = 15, OP_LOADME = 16,
  OP_CONSTRB = 17, OP_CONSTRE = 18, OP_FRAC = 19
};
struct Instr { uint32_t op, dst, a, b; };
struct MaskRef { uint32_t tree, col; int32_t off; };
struct Component {
  uint32_t log_size = 0, log_expand = 0, n_constraints = 0;
  std::vector<MaskRef> masks;
  uint32_t n_base_regs = 0, n_ext_regs = 0;
  std::vector<Instr> prog;
  // logup trace generation (host/"next" row f2): program emitting OP_FRAC(num_ext_reg, den_ext_reg) per fraction
  uint32_t n_fracs = 0, lg_base_regs = 0, lg_ext_regs = 0;
  std::vector<Instr> logup_prog;
  std::vector<uint32_t> batching;     // fraction -> batch (column) id
  uint32_t cumsum_shift_param = 0xFFFFFFFFu;
  uint32_t interaction_col0 = 0;      // first tree-2 column of this component
  uint32_t eval_log() const { return log_size + log_expand; }
  uint32_t n_logup_cols() const { uint32_t m = 0; for (auto b : batching) m = std::max(m, b + 1); return m; }
};
struct Air {
  uint32_t n_params = 0;
  std::vector<Component> comps;
  static Air parse(const uint32_t* w, size_t n) {
    size_t p = 0;
    auto rd = [&]() -> uint32_t { if (p >= n) throw std::runtime_error("air: truncated"); return w[p++]; };
    if (rd() != 0x5241424Eu) throw std::runtime_error("air: bad magic");
    if (rd() != 1) throw std::runtime_error("air: bad version");
    Air a; a.n_params = rd();
    uint32_t nc = rd();
    for (uint32_t k = 0; k < nc; ++k) {
      Component c;
      c.log_size = rd(); c.log_expand = rd(); c.n_constraints = rd();
      uint32_t nm = rd();
      for (uint32_t i = 0; i < nm; ++i) { MaskRef m; m.tree = rd(); m.col = rd(); m.off = (int32_t)rd(); c.masks.push_back(m); }
      c.n_base_regs = rd(); c.n_ext_regs = rd();
      uint32_t ni = rd();
      for (uint32_t i = 0; i < ni; ++i) { Instr in; in.op = rd(); in.dst = rd(); in.a = rd(); in.b = rd(); c.prog.push_back(in); }
      c.n_fracs = rd(); c.lg_base_regs = rd(); c.lg_ext_regs = rd();
      uint32_t nl = rd();
      for (uint32_t i = 0; i < nl; ++i) { Instr in; in.op = rd(); in.dst = rd(); in.a = rd(); in.b = rd(); c.logup_prog.push_back(in); }
      for (uint32_t i = 0; i < c.n_fracs; ++i) c.batching.push_back(rd());
      c.cumsum_shift_param = rd(); c.interaction_col0 = rd();
      a.comps.push_back(std::move(c));
    }
    return a;
  }
};

// Generic interpreter.  B = type of "base" registers (M31 on a domain, QM31 at an out-of-domain point).
template <class B> struct LiftB;
template <> struct LiftB<M31> {
  static QM31 to_e(M31 x) { return QM31::from_m31(x); }
  static QM31 mul_eb(QM31 e, M31 b) { return e * b; }
  static M31 cst(uint32_t v) { return M31::raw(v); }
  static QM31 combine(const M31 m[4]) { return QM31(CM31(m[0], m[1]), CM31(m[2], m[3])); }
};
template <> struct LiftB<QM31> {
  static QM31 to_e(QM31 x) { return x; }
  static QM31 mul_eb(QM31 e, QM31 b) { return e * b; }
  static QM31 cst(uint32_t v) { return QM31::from_m31(M31::raw(v)); }
  static QM31 combine(const QM31 m[4]) { return from_partial_evals(m); }
};
template <class B, class OnConstraint, class OnFrac>
inline void run_program(const std::vector<Instr>& prog, const B* mask, const std::vector<QM31>& params,
                        std::vector<B>& br, std::vector<QM31>& er, OnConstraint on_c, OnFrac on_f) {
  for (const Instr& in : prog) {
    switch (in.op) {
      case OP_LOADM: br[in.dst] = mask[in.a]; break;
      case OP_CONSTB: br[in.dst] = LiftB<B>::cst(in.a); break;
      case OP_ADDB: br[in.dst] = br[in.a] + br[in.b]; break;
      case OP_SUBB: br[in.dst] = br[in.a] - br[in.b]; break;
      case OP_MULB: br[in.dst] = br[in.a] * br[in.b]; break;
      case OP_NEGB: br[in.dst] = -br[in.a]; break;
      case OP_PARAME: er[in.dst] = params.at(in.a); break;
      case OP_ADDE: er[in.dst] = er[in.a] + er[in.b]; break;
      case OP_SUBE: er[in.dst] = er[in.a] - er[in.b]; break;
      case OP_MULE: er[in.dst] = er[in.a] * er[in.b]; break;
      case OP_NEGE: er[in.dst] = -er[in.a]; break;
      case OP_ADDEB: er[in.dst] = er[in.a] + LiftB<B>::to_e(br[in.b]); break;
      case OP_SUBEB: er[in.dst] = er[in.a] - LiftB<B>::to_e(br[in.b]); break;
      case OP_MULEB: er[in.dst] = LiftB<B>::mul_eb(er[in.a], br[in.b]); break;
      case OP_BTOE: er[in.dst] = LiftB<B>::to_e(br[in.a]); break;
      case OP_LOADME: er[in.dst] = LiftB<B>::combine(mask + in.a); break;
      case OP_CONSTRB: on_c(LiftB<B>::to_e(br[in.a])); break;
      case OP_CONSTRE: on_c(er[in.a]); break;
      case OP_FRAC: on_f(er[in.a], er[in.b]); break;
      default: throw std::runtime_error("air: bad opcode");
    }
  }
}

// constraint-framework/src/lib.rs (utils): offset_bit_reversed_circle_domain_index
inline size_t offset_bit_reversed_circle_domain_index(size_t i, uint32_t domain_log_size, uint32_t eval_log_size, int64_t offset) {
  int64_t prev = (int64_t)bit_reverse_index(i, eval_log_size);
  int64_t half = (int64_t)1 << (eval_log_size - 1);
  int64_t step = offset * ((int64_t)1 << (eval_log_size - domain_log_size - 1));
  auto rem = [](int64_t a, int64_t m) { int64_t r = a % m; return r < 0 ? r + m : r; };
  if (prev < half) prev = rem(prev + step, half);
  else prev = rem(prev - step, half) + half;
  return bit_reverse_index((size_t)prev, eval_log_size);
}

// ---------------------------------------------------------------------------------------------------
// commitment scheme state
struct Tree {
  std::vector<Col> polys;   // coefficients
  std::vector<Col> evals;   // LDE on CanonicCoset(log + blowup).circle_domain(), bit-reversed
  MerkleProver merkle;
  std::vector<const Col*> eval_ptrs() const { std::vector<const Col*> p; for (auto& e : evals) p.push_back(&e); return p; }
};
inline uint32_t log2_of(size_t n) { uint32_t l = 0; while (((size_t)1 << l) < n) ++l; return l; }

const TwiddleTree& get_twiddles(uint32_t domain_log);  // cache (defined in capi.cc)

inline Col interpolate_col(const Col& evals) {
  uint32_t lg = log2_of(evals.size());
  if (lg == 0) return evals;
  return interpolate(CanonicCoset(lg).circle_domain(), evals, get_twiddles(lg));
}
inline Col evaluate_col(const Col& coeffs, uint32_t domain_log) {
  if (domain_log == 0) return coeffs;
  return evaluate(CanonicCoset(domain_log).circle_domain(), coeffs, get_twiddles(domain_log));
}
// TreeBuilder::extend_evals + commit
inline Tree commit_evals(const std::vector<Col>& evals, uint32_t log_blowup, Channel& ch) {
  Tree t;
  t.polys.resize(evals.size()); t.evals.resize(evals.size());
#pragma omp parallel for schedule(dynamic)
  for (size_t i = 0; i < evals.size(); ++i) {
    t.polys[i] = interpolate_col(evals[i]);
    t.evals[i] = evaluate_col(t.polys[i], log2_of(evals[i].size()) + log_blowup);
  }
  t.merkle = MerkleProver::commit(t.eval_ptrs());
  ch.mix_root(t.merkle.root());
  return t;
}
inline Tree commit_polys(const std::vector<Col>& polys, uint32_t log_blowup, Channel& ch) {
  Tree t;
  t.polys = polys; t.evals.resize(polys.size());
  for (size_t i = 0; i < polys.size(); ++i) t.evals[i] = evaluate_col(polys[i], log2_of(polys[i].size()) + log_blowup);
  t.merkle = MerkleProver::commit(t.eval_ptrs());
  ch.mix_root(t.merkle.root());
  return t;
}

// ---------------------------------------------------------------------------------------------------
// LogupTraceGenerator semantics (constraint-framework logup.rs) driven by the component's logup program.
// Input: the component's own trace columns per tree (values on the trace domain, bit-reversed circle-domain order).
// Output: 4 base columns per logup column (appended to tree 2) and the claimed sum.                [risk A.8c]
inline void inclusive_prefix_sum_coset_order(Col& col) {
  // data is in bit-reversed circle-domain order; the running sum follows coset (trace) order
  uint32_t lg = log2_of(col.size());
  size_t n = col.size();
  M31 acc;
  for (size_t i = 0; i < n; ++i) {
    size_t pos = bit_reverse_index(coset_index_to_circle_domain_index(i, lg), lg);
    acc = acc + col[pos];
    col[pos] = acc;
  }
}
inline std::pair<std::vector<Col>, QM31> gen_interaction_trace(const Component& c, const std::vector<std::vector<Col>>& tree_evals /* [tree][global col] */,
                                                                const std::vector<QM31>& params) {
  size_t n = (size_t)1 << c.log_size;
  uint32_t ncols = c.n_logup_cols();
  std::vector<SecureCol> out(ncols);
  for (auto& s : out) s.resize(n);
  if (ncols == 0) return {{}, QM31::zero()};
#pragma omp parallel
  {
    std::vector<M31> mask(c.masks.size());
    std::vector<M31> br(c.lg_base_regs); std::vector<QM31> er(c.lg_ext_regs);
    std::vector<QM31> num(c.n_fracs), den(c.n_fracs);
#pragma omp for schedule(static)
    for (size_t row = 0; row < n; ++row) {
      for (size_t m = 0; m < c.masks.size(); ++m) {
        const MaskRef& mr = c.masks[m];
        if (mr.tree == 2 || mr.off != 0) { mask[m] = M31(); continue; }  // the logup program only reads offset-0 trace cells
        mask[m] = tree_evals[mr.tree][mr.col][row];
      }
      size_t f = 0;
      run_program<M31>(c.logup_prog, mask.data(), params, br, er, [](QM31) {}, [&](QM31 nu, QM31 de) { num[f] = nu; den[f] = de; ++f; });
      // batches: sum of fractions of a batch, cumulatively over batches (finalize_col adds the previous column)
      QM31 running = QM31::zero();
      for (uint32_t b = 0; b < ncols; ++b) {
        QM31 fn = QM31::zero(), fd = QM31::one();
        for (uint32_t k = 0; k < c.n_fracs; ++k) if (c.batching[k] == b) { fn = fn * den[k] + num[k] * fd; fd = fd * den[k]; }
        running = running + fn * inv(fd);
        out[b].set(row, running);
      }
    }
  }
  // finalize_last: claimed sum, shift, prefix sum of the last column in coset order
  SecureCol& last = out[ncols - 1];
  M31 sums[4];
  for (int k = 0; k < 4; ++k) for (size_t i = 0; i < n; ++i) sums[k] = sums[k] + last.c[k][i];
  QM31 claimed(CM31(sums[0], sums[1]), CM31(sums[2], sums[3]));
  QM31 shift = claimed * inv(M31::raw((uint32_t)(n % P)));
  for (int k = 0; k < 4; ++k) {
    M31 s = M31::raw(shift.coord(k));
    for (size_t i = 0; i < n; ++i) last.c[k][i] = last.c[k][i] - s;
    inclusive_prefix_sum_coset_order(last.c[k]);
  }
  std::vector<Col> cols;
  for (auto& s : out) for (int k = 0; k < 4; ++k) cols.push_back(std::move(s.c[k]));
  return {cols, claimed};
}

// ---------------------------------------------------------------------------------------------------
// composition polynomial (prover/air/{component_prover,accumulation}.rs + constraint-framework component.rs)
inline std::vector<QM31> secure_powers(QM31 x, size_t n) { std::vector<QM31> p(n); QM31 a = QM31::one(); for (size_t i = 0; i < n; ++i) { p[i] = a; a = a * x; } return p; }

// ComponentProver::evaluate_constraint_quotients_on_domain for one component: acc[row] += (sum_k coeff[k] * constraint_k(row)) / vanishing(row)
// on CanonicCoset(elog).circle_domain() (bit-reversed); `coeff` are the random-coefficient powers assigned to this component.  elog = 0 means the
// component's own eval_log (the prover's domain); any elog > log_size gives the same quotient polynomial on another domain.
inline void component_quotients(const Component& c, const std::vector<Tree>& trees, const std::vector<QM31>& params, const std::vector<QM31>& coeff, SecureCol& acc,
                                uint32_t elog = 0) {
  if (elog == 0) elog = c.eval_log();
  if (elog <= c.log_size) throw std::runtime_error("constraint quotients: the evaluation domain must be larger than the trace domain");
  size_t en = (size_t)1 << elog;
  CircleDomain eval_domain = CanonicCoset(elog).circle_domain();
  // evaluate every referenced column on the eval domain
  std::map<std::pair<uint32_t, uint32_t>, Col> ext;
  for (auto& m : c.masks) {
    auto key = std::make_pair(m.tree, m.col);
    if (!ext.count(key)) ext[key] = evaluate_col(trees.at(m.tree).polys.at(m.col), elog);
  }
  std::vector<const Col*> mcol(c.masks.size());
  for (size_t m = 0; m < c.masks.size(); ++m) mcol[m] = &ext[{c.masks[m].tree, c.masks[m].col}];
  // denominators: coset_vanishing(trace coset, eval_domain.at(i)) for i < 2^log_expand, bit reversed, inverted
  Coset trace_coset = CanonicCoset(c.log_size).coset;
  std::vector<M31> dinv((size_t)1 << (elog - c.log_size));
  for (size_t i = 0; i < dinv.size(); ++i) dinv[i] = inv(coset_vanishing<M31>(trace_coset, eval_domain.at(i)));
  bit_reverse(dinv);
#pragma omp parallel
  {
    std::vector<M31> mask(c.masks.size());
    std::vector<M31> br(c.n_base_regs); std::vector<QM31> er(c.n_ext_regs);
#pragma omp for schedule(static)
    for (size_t row = 0; row < en; ++row) {
      for (size_t m = 0; m < c.masks.size(); ++m) {
        size_t r = c.masks[m].off == 0 ? row : offset_bit_reversed_circle_domain_index(row, c.log_size, elog, c.masks[m].off);
        mask[m] = (*mcol[m])[r];
      }
      QM31 row_res = QM31::zero(); size_t k = 0;
      run_program<M31>(c.prog, mask.data(), params, br, er, [&](QM31 v) { row_res = row_res + coeff[k] * v; ++k; }, [](QM31, QM31) {});
      M31 di = dinv[row >> c.log_size];
      acc.set(row, acc.at(row) + row_res * di);
    }
  }
}

inline std::array<Col, 4> compute_composition(const Air& air, const std::vector<Tree>& trees, const std::vector<QM31>& params, QM31 random_coeff) {
  size_t n_total = 0; uint32_t max_log = 0;
  for (auto& c : air.comps) { n_total += c.n_constraints; max_log = std::max(max_log, c.eval_log()); }
  std::vector<QM31> powers = secure_powers(random_coeff, n_total);
  std::vector<std::unique_ptr<SecureCol>> sub(max_log + 1);
  size_t g0 = 0;
  for (const Component& c : air.comps) {
    uint32_t elog = c.eval_log();
    // this component's coefficients: the last n_constraints of the remaining powers, reversed
    std::vector<QM31> coeff(c.n_constraints);
    for (uint32_t k = 0; k < c.n_constraints; ++k) coeff[k] = powers[n_total - 1 - (g0 + k)];
    g0 += c.n_constraints;
    if (!sub[elog]) { sub[elog] = std::make_unique<SecureCol>(); sub[elog]->resize((size_t)1 << elog); }
    component_quotients(c, trees, params, coeff, *sub[elog]);
  }
  // DomainEvaluationAccumulator::finalize
  std::array<Col, 4> cur; bool have = false;
  for (uint32_t lg = 1; lg <= max_log; ++lg) {
    if (!sub[lg]) continue;
    SecureCol& v = *sub[lg];
    if (have) for (int k = 0; k < 4; ++k) { Col e = evaluate_col(cur[k], lg); for (size_t i = 0; i < e.size(); ++i) v.c[k][i] = v.c[k][i] + e[i]; }
    for (int k = 0; k < 4; ++k) cur[k] = interpolate_col(v.c[k]);
    have = true;
  }
  if (!have) for (int k = 0; k < 4; ++k) cur[k].assign((size_t)1 << max_log, M31());
  return cur;
}

// ---------------------------------------------------------------------------------------------------
// OODS sampling
inline CirclePoint<QM31> get_random_point(Channel& ch) {  // core/circle.rs CirclePoint::<SecureField>::get_random_point
  QM31 t = ch.draw_felt();
  QM31 t2 = t * t;
  QM31 ip = inv(t2 + QM31::one());
  QM31 x = (QM31::one() - t2) * ip;
  QM31 y = (t + t) * ip;
  return CirclePoint<QM31>(x, y);
}
inline CirclePoint<QM31> mul_signed_ef(CirclePoint<M31> step, int64_t off) {
  CirclePoint<M31> p = step.mul((uint64_t)(off < 0 ? -off : off));
  if (off < 0) p = p.conjugate();
  return to_ef(p);
}
typedef std::vector<std::vector<std::vector<CirclePoint<QM31>>>> MaskPoints;   // [tree][col][k]
typedef std::vector<std::vector<std::vector<QM31>>> SampledValues;            // [tree][col][k]

// Components::mask_points: per tree/column the list of sample points (declaration order of offsets), preprocessed
// columns sampled at the point itself when used, composition columns at the point.
inline MaskPoints mask_points(const Air& air, const std::vector<size_t>& n_cols_per_tree, CirclePoint<QM31> point,
                              std::vector<std::vector<std::vector<int32_t>>>* offsets_out = nullptr) {
  MaskPoints mp(4);
  std::vector<std::vector<std::vector<int32_t>>> offs(4);
  for (int t = 0; t < 3; ++t) { mp[t].resize(n_cols_per_tree[t]); offs[t].resize(n_cols_per_tree[t]); }
  for (const Component& c : air.comps) {
    CirclePoint<M31> step = CanonicCoset(c.log_size).step();
    for (const MaskRef& m : c.masks) {
      auto& o = offs[m.tree].at(m.col);
      if (std::find(o.begin(), o.end(), m.off) != o.end()) continue;
      o.push_back(m.off);
      mp[m.tree][m.col].push_back(point + mul_signed_ef(step, m.off));
    }
  }
  mp[3].assign(4, std::vector<CirclePoint<QM31>>{point});
  offs[3].assign(4, std::vector<int32_t>{0});
  if (offsets_out) *offsets_out = offs;
  return mp;
}

// eval_composition_polynomial_at_point (PointEvaluator / PointEvaluationAccumulator)
inline QM31 eval_composition_at_point(const Air& air, CirclePoint<QM31> point, const SampledValues& sv,
                                      const std::vector<std::vector<std::vector<int32_t>>>& offs, const std::vector<QM31>& params, QM31 random_coeff) {
  QM31 accumulation = QM31::zero();
  for (const Component& c : air.comps) {
    std::vector<QM31> mask(c.masks.size());
    for (size_t m = 0; m < c.masks.size(); ++m) {
      const MaskRef& mr = c.masks[m];
      const auto& o = offs[mr.tree][mr.col];
      size_t k = std::find(o.begin(), o.end(), mr.off) - o.begin();
      mask[m] = sv[mr.tree][mr.col].at(k);
    }
    QM31 dinv = inv(coset_vanishing<QM31>(CanonicCoset(c.log_size).coset, point));
    std::vector<QM31> br(c.n_base_regs), er(c.n_ext_regs);
    run_program<QM31>(c.prog, mask.data(), params, br, er, [&](QM31 v) { accumulation = accumulation * random_coeff + dinv * v; }, [](QM31, QM31) {});
  }
  return accumulation;
}

// ---------------------------------------------------------------------------------------------------
// DEEP quotients (core/pcs/quotients.rs + prover/backend/cpu/quotients.rs)
struct PointSample { CirclePoint<QM31> point; QM31 value; };
struct ColumnSampleBatch { CirclePoint<QM31> point; std::vector<std::pair<size_t, QM31>> cols; };
inline std::vector<ColumnSampleBatch> sample_batches_new_vec(const std::vector<const std::vector<PointSample>*>& samples) {
  // group by point, keeping first-seen order                                                [risk: IndexMap vs BTreeMap]
  std::vector<ColumnSampleBatch> out;
  for (size_t ci = 0; ci < samples.size(); ++ci)
    for (const PointSample& s : *samples[ci]) {
      size_t k = 0;
      for (; k < out.size(); ++k) if (out[k].point == s.point) break;
      if (k == out.size()) out.push_back(ColumnSampleBatch{s.point, {}});
      out[k].cols.push_back({ci, s.value});
    }
  return out;
}
struct LineCoeffs { QM31 a, b, c; };
inline LineCoeffs complex_conjugate_line_coeffs(const PointSample& s, QM31 alpha) {
  QM31 a = s.value.complex_conjugate() - s.value;
  QM31 c = s.point.y.complex_conjugate() - s.point.y;
  QM31 b = s.value * c - a * s.point.y;
  return LineCoeffs{alpha * a, alpha * b, alpha * c};
}
inline SecureCol accumulate_quotients(uint32_t log_size, const std::vector<const Col*>& columns, QM31 random_coeff, const std::vector<ColumnSampleBatch>& batches) {
  CircleDomain domain = CanonicCoset(log_size).circle_domain();
  size_t n = domain.size();
  std::vector<std::vector<LineCoeffs>> line(batches.size());
  std::vector<QM31> batch_coeff(batches.size());
  for (size_t b = 0; b < batches.size(); ++b) {
    QM31 alpha = QM31::one();
    for (auto& cv : batches[b].cols) { alpha = alpha * random_coeff; line[b].push_back(complex_conjugate_line_coeffs(PointSample{batches[b].point, cv.second}, alpha)); }
    batch_coeff[b] = pow(random_coeff, batches[b].cols.size());
  }
  SecureCol out; out.resize(n);
  // domain points in bit-reversed order
  std::vector<CirclePoint<M31>> pts(n);
  {
    std::vector<CirclePoint<M31>> nat(n);
    CirclePoint<M31> cur = domain.half_coset.initial(), st = domain.half_coset.step();
    for (size_t i = 0; i < n / 2; ++i) { nat[i] = cur; nat[n / 2 + i] = cur.conjugate(); cur = cur + st; }
    for (size_t i = 0; i < n; ++i) pts[i] = nat[bit_reverse_index(i, log_size)];
  }
#pragma omp parallel for schedule(static)
  for (size_t row = 0; row < n; ++row) {
    CirclePoint<M31> dp = pts[row];
    QM31 acc = QM31::zero();
    for (size_t b = 0; b < batches.size(); ++b) {
      const ColumnSampleBatch& sb = batches[b];
      CM31 prx = sb.point.x.a, pry = sb.point.y.a, pix = sb.point.x.b, piy = sb.point.y.b;
      CM31 den = (prx - CM31(dp.x, M31())) * piy - (pry - CM31(dp.y, M31())) * pix;
      CM31 dinv = inv(den);
      QM31 numer = QM31::zero();
      for (size_t k = 0; k < sb.cols.size(); ++k) {
        const LineCoeffs& lc = line[b][k];
        QM31 value = lc.c * (*columns[sb.cols[k].first])[row];
        QM31 linear = lc.a * dp.y + lc.b;
        numer = numer + (value - linear);
      }
      acc = acc * batch_coeff[b] + mul_cm31(numer, dinv);
    }
    out.set(row, acc);
  }
  return out;
}

// ---------------------------------------------------------------------------------------------------
// proof structures (core/proof.rs, core/pcs/mod.rs CommitmentSchemeProof, core/fri.rs FriProof)   [risk A.12]
struct FriLayerProof { std::vector<QM31> fri_witness; MerkleDecommitment decommitment; Hash32 commitment; };
struct FriProof { FriLayerProof first_layer; std::vector<FriLayerProof> inner_layers; std::vector<QM31> last_layer_poly; uint32_t last_layer_log_size = 0; };
struct Proof {
  PcsConfig config;
  std::vector<Hash32> commitments;
  SampledValues sampled_values;
  std::vector<MerkleDecommitment> decommitments;
  std::vector<std::vector<M31>> queried_values;
  uint64_t proof_of_work = 0;
  FriProof fri_proof;
};
// postcard (serde) encoding: LEB128 varints for integers and lengths, arrays of u8 raw
struct Postcard {
  std::vector<uint8_t> out;
  void varint(uint64_t v) { while (v >= 0x80) { out.push_back((uint8_t)(v | 0x80)); v >>= 7; } out.push_back((uint8_t)v); }
  void m31(M31 v) { varint(v.v); }
  void qm31(QM31 v) { for (int k = 0; k < 4; ++k) varint(v.coord(k)); }
  void hash(const Hash32& h) { out.insert(out.end(), h.begin(), h.end()); }
  void decommitment(const MerkleDecommitment& d) {
    varint(d.hash_witness.size()); for (auto& h : d.hash_witness) hash(h);
    varint(d.column_witness.size()); for (auto v : d.column_witness) m31(v);
  }
  void fri_layer(const FriLayerProof& l) { varint(l.fri_witness.size()); for (auto& q : l.fri_witness) qm31(q); decommitment(l.decommitment); hash(l.commitment); }
  void proof(const Proof& p) {
    varint(p.config.pow_bits); varint(p.config.fri.log_blowup_factor); varint(p.config.fri.log_last_layer_degree_bound); varint(p.config.fri.n_queries);
    varint(p.commitments.size()); for (auto& h : p.commitments) hash(h);
    varint(p.sampled_values.size());
    for (auto& t : p.sampled_values) { varint(t.size()); for (auto& c : t) { varint(c.size()); for (auto& q : c) qm31(q); } }
    varint(p.decommitments.size()); for (auto& d : p.decommitments) decommitment(d);
    varint(p.queried_values.size()); for (auto& t : p.queried_values) { varint(t.size()); for (auto v : t) m31(v); }
    varint(p.proof_of_work);
    fri_layer(p.fri_proof.first_layer);
    varint(p.fri_proof.inner_layers.size()); for (auto& l : p.fri_proof.inner_layers) fri_layer(l);
    varint(p.fri_proof.last_layer_poly.size()); for (auto& q : p.fri_proof.last_layer_poly) qm31(q);
    varint(p.fri_proof.last_layer_log_size);
  }
};

// ---------------------------------------------------------------------------------------------------
// FRI (prover/fri.rs, core/fri.rs, backend/cpu/fri.rs)
struct Queries {
  std::vector<size_t> positions; uint32_t log_domain_size;
  static Queries generate(Channel& ch, uint32_t log_domain_size, size_t n_queries) {  // core/queries.rs
    std::set<size_t> q; size_t cnt = 0; size_t mask = ((size_t)1 << log_domain_size) - 1;
    while (true) {
      Hash32 r = ch.draw_random_bytes();
      for (int k = 0; k < 8; ++k) {
        uint32_t w; memcpy(&w, r.data() + 4 * k, 4);
        q.insert((size_t)w & mask);
        if (++cnt == n_queries) { Queries o; o.positions.assign(q.begin(), q.end()); o.log_domain_size = log_domain_size; return o; }
      }
    }
  }
  Queries fold(uint32_t n_folds) const {
    Queries o; o.log_domain_size = log_domain_size - n_folds;
    for (size_t p : positions) { size_t f = p >> n_folds; if (o.positions.empty() || o.positions.back() != f) o.positions.push_back(f); }
    return o;
  }
};
struct LineEval { LineDomain domain; std::vector<QM31> values; };  // bit-reversed order
inline LineEval fold_line(const LineEval& e, QM31 alpha) {
  size_t n = e.values.size();
  LineEval out; out.domain = e.domain.dbl(); out.values.resize(n / 2);
  uint32_t lg = e.domain.log_size();
  for (size_t i = 0; i < n / 2; ++i) {
    M31 x = e.domain.at(bit_reverse_index(i << 1, lg));
    QM31 f0 = e.values[2 * i], f1 = e.values[2 * i + 1];
    ibutterfly(f0, f1, inv(x));
    out.values[i] = f0 + alpha * f1;
  }
  return out;
}
inline void fold_circle_into_line(LineEval& dst, const SecureCol& src, uint32_t src_log, QM31 alpha) {
  CircleDomain domain = CanonicCoset(src_log).circle_domain();
  QM31 alpha_sq = alpha * alpha;
  size_t n = src.size();
  for (size_t i = 0; i < n / 2; ++i) {
    CirclePoint<M31> p = domain.at(bit_reverse_index(i << 1, src_log));
    QM31 f0 = src.at(2 * i), f1 = src.at(2 * i + 1);
    ibutterfly(f0, f1, inv(p.y));
    QM31 f_prime = alpha * f1 + f0;
    dst.values[i] = dst.values[i] * alpha_sq + f_prime;
  }
}
inline std::vector<const Col*> coord_ptrs(const std::vector<SecureCol>& cols) { std::vector<const Col*> p; for (auto& s : cols) for (int k = 0; k < 4; ++k) p.push_back(&s.c[k]); return p; }
inline SecureCol to_secure_col(const std::vector<QM31>& v) { SecureCol s; s.resize(v.size()); for (size_t i = 0; i < v.size(); ++i) s.set(i, v[i]); return s; }

// line interpolation for the last layer (core/poly/line.rs LineEvaluation::interpolate); returns ordered coefficients
inline std::vector<QM31> line_interpolate_ordered(const LineEval& e) {
  std::vector<QM31> v = e.values; bit_reverse(v);  // natural order
  LineDomain d = e.domain;
  size_t n = v.size();
  while (d.size() > 1) {
    size_t ds = d.size();
    for (size_t c0 = 0; c0 < n; c0 += ds)
      for (size_t i = 0; i < ds / 2; ++i) { M31 x = d.at(i); ibutterfly(v[c0 + i], v[c0 + ds / 2 + i], inv(x)); }
    d = d.dbl();
  }
  M31 sc = inv(M31::raw((uint32_t)n));
  for (auto& q : v) q = q * sc;
  bit_reverse(v);  // LinePoly stores bit-reversed; into_ordered_coefficients undoes it — net: the fft output order reversed once
  return v;
}

struct FriProver {
  FriConfig config;
  std::vector<SecureCol> first_cols; std::vector<uint32_t> first_logs; MerkleProver first_tree;
  struct Inner { LineEval eval; SecureCol cols; MerkleProver tree; };
  std::vector<Inner> inner;
  std::vector<QM31> last_layer_poly;

  static FriProver commit(Channel& ch, FriConfig cfg, std::vector<SecureCol> columns, std::vector<uint32_t> logs) {
    FriProver fp; fp.config = cfg;
    fp.first_cols = std::move(columns); fp.first_logs = logs;
    fp.first_tree = MerkleProver::commit(coord_ptrs(fp.first_cols));
    ch.mix_root(fp.first_tree.root());
    QM31 circle_alpha = ch.draw_felt();
    uint32_t first_inner_log = fp.first_logs[0] - 1;
    LineEval layer; layer.domain = LineDomain(Coset::half_odds(first_inner_log)); layer.values.assign((size_t)1 << first_inner_log, QM31::zero());
    size_t ci = 0;
    while (layer.values.size() > cfg.last_layer_domain_size()) {
      while (ci < fp.first_cols.size() && (fp.first_cols[ci].size() >> 1) == layer.values.size()) {
        fold_circle_into_line(layer, fp.first_cols[ci], fp.first_logs[ci], circle_alpha); ++ci;
      }
      Inner in; in.eval = layer; in.cols = to_secure_col(layer.values);
      std::vector<const Col*> p; for (int k = 0; k < 4; ++k) p.push_back(&in.cols.c[k]);
      in.tree = MerkleProver::commit(p);
      ch.mix_root(in.tree.root());
      QM31 alpha = ch.draw_felt();
      layer = fold_line(in.eval, alpha);
      fp.inner.push_back(std::move(in));
    }
    if (ci != fp.first_cols.size()) throw std::runtime_error("fri: not all columns consumed");
    if (layer.values.size() != cfg.last_layer_domain_size()) throw std::runtime_error("fri: last layer size");
    std::vector<QM31> coeffs = line_interpolate_ordered(layer);
    size_t bound = (size_t)1 << cfg.log_last_layer_degree_bound;
    for (size_t i = bound; i < coeffs.size(); ++i) if (!coeffs[i].is_zero()) throw std::runtime_error("fri: invalid degree");
    coeffs.resize(bound);
    std::vector<QM31> stored = coeffs; bit_reverse(stored);  // LinePoly::from_ordered_coefficients
    fp.last_layer_poly = stored;
    ch.mix_felts(fp.last_layer_poly);
    return fp;
  }

  static void positions_and_witness(const SecureCol& col, const std::vector<size_t>& queries, uint32_t fold_step,
                                    std::vector<size_t>& positions, std::vector<QM31>& witness) {
    size_t i = 0;
    while (i < queries.size()) {
      size_t j = i; size_t key = queries[i] >> fold_step;
      while (j < queries.size() && (queries[j] >> fold_step) == key) ++j;
      size_t start = key << fold_step;
      size_t q = i;
      for (size_t pos = start; pos < start + ((size_t)1 << fold_step); ++pos) {
        positions.push_back(pos);
        if (q < j && queries[q] == pos) { ++q; continue; }
        witness.push_back(col.at(pos));
      }
      i = j;
    }
  }

  std::pair<FriProof, std::map<uint32_t, std::vector<size_t>>> decommit(Channel& ch) {
    uint32_t max_log = first_logs[0];
    Queries queries = Queries::generate(ch, max_log, config.n_queries);
    std::map<uint32_t, std::vector<size_t>> by_log;
    for (uint32_t lg : first_logs) by_log[lg] = queries.fold(max_log - lg).positions;
    FriProof proof;
    {  // first layer
      std::map<uint32_t, std::vector<size_t>> dpos;
      for (size_t c = 0; c < first_cols.size(); ++c) {
        Queries cq = queries.fold(max_log - first_logs[c]);
        std::vector<size_t> pos;
        positions_and_witness(first_cols[c], cq.positions, 1, pos, proof.first_layer.fri_witness);
        dpos[first_logs[c]] = pos;
      }
      proof.first_layer.decommitment = first_tree.decommit(dpos, coord_ptrs(first_cols)).second;
      proof.first_layer.commitment = first_tree.root();
    }
    Queries lq = queries.fold(1);
    for (auto& in : inner) {
      FriLayerProof lp;
      std::vector<size_t> pos;
      positions_and_witness(in.cols, lq.positions, 1, pos, lp.fri_witness);
      std::map<uint32_t, std::vector<size_t>> dpos; dpos[in.eval.domain.log_size()] = pos;
      std::vector<const Col*> p; for (int k = 0; k < 4; ++k) p.push_back(&in.cols.c[k]);
      lp.decommitment = in.tree.decommit(dpos, p).second;
      lp.commitment = in.tree.root();
      proof.inner_layers.push_back(std::move(lp));
      lq = lq.fold(1);
    }
    proof.last_layer_poly = last_layer_poly;
    proof.last_layer_log_size = config.log_last_layer_degree_bound;
    return {proof, by_log};
  }
};

// GrindOps::grind: smallest nonce whose mixed digest has >= pow_bits trailing zero bits       [risk A.11]
inline bool pow_ok(const Channel& ch, uint64_t nonce, uint32_t pow_bits) { Channel c = ch; c.mix_u64(nonce); return c.trailing_zeros() >= pow_bits; }
inline uint64_t grind(const Channel& ch, uint32_t pow_bits) { for (uint64_t n = 0;; ++n) if (pow_ok(ch, n, pow_bits)) return n; }

// ---------------------------------------------------------------------------------------------------
// stwo::prover::prove + CommitmentSchemeProver::prove_values
struct ProveError : std::runtime_error { using std::runtime_error::runtime_error; };

inline Proof prove(const Air& air, const std::vector<QM31>& params, std::vector<Tree>& trees /* 3 committed trees */, Channel& ch, PcsConfig config) {
  if (trees.size() != 3) throw std::runtime_error("prove: expects the 3 trace trees to be committed");
  QM31 random_coeff = ch.draw_felt();
  std::array<Col, 4> comp = compute_composition(air, trees, params, random_coeff);
  trees.push_back(commit_polys(std::vector<Col>(comp.begin(), comp.end()), config.fri.log_blowup_factor, ch));
  CirclePoint<QM31> oods = get_random_point(ch);
  std::vector<size_t> ncols{trees[0].polys.size(), trees[1].polys.size(), trees[2].polys.size()};
  std::vector<std::vector<std::vector<int32_t>>> offs;
  MaskPoints mp = mask_points(air, ncols, oods, &offs);
  // prove_values
  std::vector<std::vector<std::vector<PointSample>>> samples(4);
  Proof proof; proof.config = config;
  proof.sampled_values.resize(4);
  for (int t = 0; t < 4; ++t) {
    samples[t].resize(trees[t].polys.size()); proof.sampled_values[t].resize(trees[t].polys.size());
    for (size_t c = 0; c < trees[t].polys.size(); ++c)
      for (auto& pt : mp[t][c]) { QM31 v = eval_at_point(trees[t].polys[c], pt); samples[t][c].push_back(PointSample{pt, v}); proof.sampled_values[t][c].push_back(v); }
  }
  std::vector<QM31> flat;
  for (auto& t : proof.sampled_values) for (auto& c : t) for (auto& v : c) flat.push_back(v);
  ch.mix_felts(flat);
  QM31 q_coeff = ch.draw_felt();
  // compute_fri_quotients: all columns of all trees, sorted by LDE size (desc, stable), grouped by size
  struct CS { const Col* col; const std::vector<PointSample>* s; uint32_t log; };
  std::vector<CS> all;
  for (int t = 0; t < 4; ++t) for (size_t c = 0; c < trees[t].evals.size(); ++c) all.push_back(CS{&trees[t].evals[c], &samples[t][c], log2_of(trees[t].evals[c].size())});
  std::stable_sort(all.begin(), all.end(), [](const CS& a, const CS& b) { return a.log > b.log; });
  std::vector<SecureCol> quotients; std::vector<uint32_t> qlogs;
  for (size_t i = 0; i < all.size();) {
    size_t j = i; while (j < all.size() && all[j].log == all[i].log) ++j;
    std::vector<const Col*> cols; std::vector<const std::vector<PointSample>*> ss;
    for (size_t k = i; k < j; ++k) { cols.push_back(all[k].col); ss.push_back(all[k].s); }
    quotients.push_back(accumulate_quotients(all[i].log, cols, q_coeff, sample_batches_new_vec(ss)));
    qlogs.push_back(all[i].log);
    i = j;
  }
  FriProver fri = FriProver::commit(ch, config.fri, std::move(quotients), qlogs);
  proof.proof_of_work = grind(ch, config.pow_bits);
  ch.mix_u64(proof.proof_of_work);
  auto dec = fri.decommit(ch);
  proof.fri_proof = dec.first;
  for (int t = 0; t < 4; ++t) {
    proof.commitments.push_back(trees[t].merkle.root());
    auto r = trees[t].merkle.decommit(dec.second, trees[t].eval_ptrs());
    proof.queried_values.push_back(r.first);
    proof.decommitments.push_back(r.second);
  }
  // sanity check (ProvingError::ConstraintsNotSatisfied)
  QM31 cv[4] = {proof.sampled_values[3][0][0], proof.sampled_values[3][1][0], proof.sampled_values[3][2][0], proof.sampled_values[3][3][0]};
  if (from_partial_evals(cv) != eval_composition_at_point(air, oods, proof.sampled_values, offs, params, random_coeff))
    throw ProveError("ConstraintsNotSatisfied");
  return proof;
}

}  // namespace orc
