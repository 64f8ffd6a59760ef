// ORACLE — TEST INFRASTRUCTURE ONLY (see fields.h header).  PARITY UNPINNED.
// An independent verifier for proofs produced by prove.h / by the CUDA path: restates the checks of
// stwo @0790eba core/verifier.rs (verify), core/pcs/verifier.rs (verify_values), core/fri.rs (FriVerifier),
// core/vcs/verifier.rs (MerkleVerifier), as reached from nexus-zkvm prover/src/machine.rs:318-485.
// It is written from the protocol, not by inverting the prover code, so it catches prover-side slips.
#pragma once
#include "prove.h"

namespace orc {

struct VerifyError : std::runtime_error { using std::runtime_error::runtime_error; };

// MerkleVerifier::verify. col_logs: log sizes of the tree's columns in commitment order.
inline void merkle_verify(const Hash32& root, const std::vector<uint32_t>& col_logs_in, const std::map<uint32_t, std::vector<size_t>>& queries,
                          const std::vector<M31>& queried_values, const MerkleDecommitment& d) {
  std::vector<uint32_t> logs = col_logs_in;
  std::stable_sort(logs.begin(), logs.end(), [](uint32_t a, uint32_t b) { return a > b; });
  uint32_t max_log = logs.empty() ? 0 : logs[0];
  size_t qv = 0, hw = 0, cw = 0, ci = 0;
  std::vector<std::pair<size_t, Hash32>> last;
  for (int l = (int)max_log; l >= 0; --l) {
    size_t n_here = 0;
    while (ci < logs.size() && logs[ci] == (uint32_t)l) { ++ci; ++n_here; }
    static const std::vector<size_t> empty;
    auto it = queries.find((uint32_t)l);
    const std::vector<size_t>& lq = it == queries.end() ? empty : it->second;
    size_t pq = 0, cq = 0;
    std::vector<std::pair<size_t, Hash32>> cur;
    while (true) {
      bool has_p = pq < last.size(), has_c = cq < lq.size();
      if (!has_p && !has_c) break;
      size_t node;
      if (has_p && has_c) node = std::min(last[pq].first / 2, lq[cq]);
      else if (has_p) node = last[pq].first / 2;
      else node = lq[cq];
      Hash32 left, right; bool has_children = (uint32_t)l < max_log;
      if (has_children) {
        if (pq < last.size() && last[pq].first == 2 * node) left = last[pq++].second;
        else { if (hw >= d.hash_witness.size()) throw VerifyError("merkle: witness too short"); left = d.hash_witness[hw++]; }
        if (pq < last.size() && last[pq].first == 2 * node + 1) right = last[pq++].second;
        else { if (hw >= d.hash_witness.size()) throw VerifyError("merkle: witness too short"); right = d.hash_witness[hw++]; }
      }
      std::vector<M31> vals(n_here);
      bool queried = cq < lq.size() && lq[cq] == node;
      if (queried) { ++cq; if (qv + n_here > queried_values.size()) throw VerifyError("merkle: too few queried values"); for (size_t k = 0; k < n_here; ++k) vals[k] = queried_values[qv++]; }
      else { if (cw + n_here > d.column_witness.size()) throw VerifyError("merkle: column witness too short"); for (size_t k = 0; k < n_here; ++k) vals[k] = d.column_witness[cw++]; }
      cur.push_back({node, hash_node(has_children ? &left : nullptr, has_children ? &right : nullptr, vals.data(), vals.size())});
    }
    last.swap(cur);
  }
  if (qv != queried_values.size() || hw != d.hash_witness.size() || cw != d.column_witness.size()) throw VerifyError("merkle: witness too long");
  if (last.size() != 1 || last[0].first != 0 || last[0].second != root) throw VerifyError("merkle: root mismatch");
}

inline QM31 line_poly_eval(const std::vector<QM31>& coeffs_bitrev, uint32_t log_size, QM31 x) {
  // LinePoly::eval_at_point: fold(coeffs, [x, pi(x), ...]) with the first factor applied to the top split.  Unlike CirclePoly::eval_at_point
  // there is no reversal: the coefficients are stored bit-reversed, so the top split of the stored order is bit 0 of the ordered one (x).
  // A reversal here is invisible while the last layer has at most two coefficients (log_last_layer_degree_bound <= 1).
  std::vector<QM31> d; for (uint32_t i = 0; i < log_size; ++i) { d.push_back(x); x = double_x(x); }
  std::function<QM31(const QM31*, size_t, const QM31*)> rec = [&](const QM31* v, size_t n, const QM31* f) -> QM31 {
    if (n == 1) return v[0];
    return rec(v, n / 2, f + 1) + rec(v + n / 2, n / 2, f + 1) * f[0];
  };
  return rec(coeffs_bitrev.data(), coeffs_bitrev.size(), d.data());
}

// col_logs[t] = trace log size of every column of tree t (t < 3), in commitment order.
inline void verify(const Air& air, const std::vector<QM31>& params, const Proof& proof, Channel ch, const std::vector<std::vector<uint32_t>>& col_logs) {
  const PcsConfig& cfg = proof.config;
  if (proof.commitments.size() != 4 || proof.sampled_values.size() != 4 || proof.queried_values.size() != 4 || proof.decommitments.size() != 4)
    throw VerifyError("shape: expected 4 trees");
  QM31 random_coeff = ch.draw_felt();
  uint32_t comp_log = 0; for (auto& c : air.comps) comp_log = std::max(comp_log, c.eval_log());
  ch.mix_root(proof.commitments[3]);
  CirclePoint<QM31> oods = get_random_point(ch);
  std::vector<size_t> ncols{col_logs[0].size(), col_logs[1].size(), col_logs[2].size()};
  std::vector<std::vector<std::vector<int32_t>>> offs;
  MaskPoints mp = mask_points(air, ncols, oods, &offs);
  std::vector<std::vector<uint32_t>> logs = col_logs;
  logs.resize(4); logs[3].assign(4, comp_log);
  for (int t = 0; t < 4; ++t) {
    if (proof.sampled_values[t].size() != logs[t].size()) throw VerifyError("shape: sampled_values columns");
    for (size_t c = 0; c < logs[t].size(); ++c) if (proof.sampled_values[t][c].size() != mp[t][c].size()) throw VerifyError("shape: sampled_values points");
  }
  QM31 cv[4] = {proof.sampled_values[3][0][0], proof.sampled_values[3][1][0], proof.sampled_values[3][2][0], proof.sampled_values[3][3][0]};
  if (from_partial_evals(cv) != eval_composition_at_point(air, oods, proof.sampled_values, offs, params, random_coeff)) throw VerifyError("OodsNotMatching");
  std::vector<QM31> flat;
  for (auto& t : proof.sampled_values) for (auto& c : t) for (auto& v : c) flat.push_back(v);
  ch.mix_felts(flat);
  QM31 q_coeff = ch.draw_felt();

  // quotient column sizes
  struct CRef { int t; size_t c; uint32_t log; };
  std::vector<CRef> all;
  for (int t = 0; t < 4; ++t) for (size_t c = 0; c < logs[t].size(); ++c) all.push_back(CRef{t, c, logs[t][c] + cfg.fri.log_blowup_factor});
  std::stable_sort(all.begin(), all.end(), [](const CRef& a, const CRef& b) { return a.log > b.log; });
  std::vector<uint32_t> qlogs; std::vector<std::vector<CRef>> groups;
  for (size_t i = 0; i < all.size();) { size_t j = i; while (j < all.size() && all[j].log == all[i].log) ++j; qlogs.push_back(all[i].log); groups.emplace_back(all.begin() + i, all.begin() + j); i = j; }
  uint32_t max_log = qlogs.at(0);

  // FRI commit-phase replay
  const FriProof& fp = proof.fri_proof;
  ch.mix_root(fp.first_layer.commitment);
  QM31 circle_alpha = ch.draw_felt();
  std::vector<QM31> alphas;
  uint32_t inner_log = max_log - 1;
  size_t expected_inner = 0;
  for (size_t sz = (size_t)1 << inner_log; sz > cfg.fri.last_layer_domain_size(); sz >>= 1) ++expected_inner;
  if (fp.inner_layers.size() != expected_inner) throw VerifyError("fri: wrong number of layers");
  for (auto& l : fp.inner_layers) { ch.mix_root(l.commitment); alphas.push_back(ch.draw_felt()); }
  if (fp.last_layer_poly.size() > ((size_t)1 << cfg.fri.log_last_layer_degree_bound)) throw VerifyError("fri: last layer degree");
  ch.mix_felts(fp.last_layer_poly);
  if (!pow_ok(ch, proof.proof_of_work, cfg.pow_bits)) throw VerifyError("ProofOfWork");
  ch.mix_u64(proof.proof_of_work);
  Queries queries = Queries::generate(ch, max_log, cfg.fri.n_queries);
  std::map<uint32_t, std::vector<size_t>> by_log;
  for (uint32_t lg : qlogs) by_log[lg] = queries.fold(max_log - lg).positions;

  // trace / composition Merkle decommitments
  for (int t = 0; t < 4; ++t) {
    std::vector<uint32_t> lde_logs; for (uint32_t l : logs[t]) lde_logs.push_back(l + cfg.fri.log_blowup_factor);
    merkle_verify(proof.commitments[t], lde_logs, by_log, proof.queried_values[t], proof.decommitments[t]);
  }
  // queried value lookup: value(t, c, k-th query of its size)
  std::vector<std::map<uint32_t, std::pair<size_t, std::vector<size_t>>>> layout(4);  // per tree: log -> (offset, cols in layer order)
  for (int t = 0; t < 4; ++t) {
    std::vector<size_t> order(logs[t].size()); for (size_t i = 0; i < order.size(); ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return logs[t][a] > logs[t][b]; });
    size_t off = 0;
    for (size_t i = 0; i < order.size();) {
      uint32_t lg = logs[t][order[i]] + cfg.fri.log_blowup_factor;
      size_t j = i; std::vector<size_t> cols; while (j < order.size() && logs[t][order[j]] + cfg.fri.log_blowup_factor == lg) cols.push_back(order[j++]);
      layout[t][lg] = {off, cols};
      off += cols.size() * by_log[lg].size();
      i = j;
    }
  }
  auto queried = [&](int t, size_t c, uint32_t lg, size_t k) -> M31 {
    auto& L = layout[t].at(lg);
    size_t idx = std::find(L.second.begin(), L.second.end(), c) - L.second.begin();
    return proof.queried_values[t].at(L.first + k * L.second.size() + idx);
  };

  // quotient evaluations at the query positions, per size group
  std::vector<std::map<size_t, QM31>> qvals(qlogs.size());
  for (size_t g = 0; g < groups.size(); ++g) {
    uint32_t lg = qlogs[g];
    std::vector<std::vector<PointSample>> samples(groups[g].size());
    std::vector<const std::vector<PointSample>*> sp;
    for (size_t k = 0; k < groups[g].size(); ++k) {
      const CRef& r = groups[g][k];
      for (size_t p = 0; p < mp[r.t][r.c].size(); ++p) samples[k].push_back(PointSample{mp[r.t][r.c][p], proof.sampled_values[r.t][r.c][p]});
    }
    for (auto& s : samples) sp.push_back(&s);
    std::vector<ColumnSampleBatch> batches = sample_batches_new_vec(sp);
    CircleDomain domain = CanonicCoset(lg).circle_domain();
    const std::vector<size_t>& pos = by_log[lg];
    for (size_t qi = 0; qi < pos.size(); ++qi) {
      CirclePoint<M31> dp = domain.at(bit_reverse_index(pos[qi], lg));
      QM31 acc = QM31::zero();
      for (auto& sb : batches) {
        CM31 den = (sb.point.x.a - CM31(dp.x, M31())) * sb.point.y.b - (sb.point.y.a - CM31(dp.y, M31())) * sb.point.x.b;
        QM31 numer = QM31::zero(); QM31 alpha = QM31::one();
        for (auto& cv2 : sb.cols) {
          alpha = alpha * q_coeff;
          LineCoeffs lc = complex_conjugate_line_coeffs(PointSample{sb.point, cv2.second}, alpha);
          const CRef& r = groups[g][cv2.first];
          numer = numer + (lc.c * queried(r.t, r.c, lg, qi) - (lc.a * dp.y + lc.b));
        }
        acc = acc * pow(q_coeff, sb.cols.size()) + mul_cm31(numer, inv(den));
      }
      qvals[g][pos[qi]] = acc;
    }
  }

  // FRI first layer: rebuild the folding pairs from computed values + witnesses, check the Merkle decommitment
  size_t wi = 0;
  std::vector<M31> first_flat_values;
  std::map<uint32_t, std::vector<size_t>> first_dpos;
  std::vector<std::map<size_t, QM31>> pair_vals(qlogs.size());
  for (size_t g = 0; g < groups.size(); ++g) {
    uint32_t lg = qlogs[g];
    const std::vector<size_t>& pos = by_log[lg];
    std::vector<size_t> dpos;
    for (size_t i = 0; i < pos.size();) {
      size_t j = i; while (j < pos.size() && (pos[j] >> 1) == (pos[i] >> 1)) ++j;
      for (size_t p = (pos[i] >> 1) << 1; p < ((pos[i] >> 1) << 1) + 2; ++p) {
        dpos.push_back(p);
        if (qvals[g].count(p)) pair_vals[g][p] = qvals[g][p];
        else { if (wi >= fp.first_layer.fri_witness.size()) throw VerifyError("fri: first layer witness too short"); pair_vals[g][p] = fp.first_layer.fri_witness[wi++]; }
      }
      i = j;
    }
    first_dpos[lg] = dpos;
  }
  if (wi != fp.first_layer.fri_witness.size()) throw VerifyError("fri: first layer witness too long");
  {
    std::vector<uint32_t> clogs; for (uint32_t lg : qlogs) for (int k = 0; k < 4; ++k) clogs.push_back(lg);
    for (size_t g = 0; g < groups.size(); ++g)  // flat values: layer desc, node asc, 4 coordinate columns
      for (size_t p : first_dpos[qlogs[g]]) for (int k = 0; k < 4; ++k) first_flat_values.push_back(M31::raw(pair_vals[g][p].coord(k)));
    merkle_verify(fp.first_layer.commitment, clogs, first_dpos, first_flat_values, fp.first_layer.decommitment);
  }
  // inner layers
  std::map<size_t, QM31> cur;  // folded values at the current line layer's query positions
  Queries lq = queries.fold(1);
  uint32_t llog = inner_log;
  for (size_t k = 0; k <= fp.inner_layers.size(); ++k) {
    // fold in circle columns whose folded size equals this layer
    std::map<size_t, QM31> vals;
    for (size_t p : lq.positions) vals[p] = cur.count(p) ? cur[p] : QM31::zero();
    for (size_t g = 0; g < groups.size(); ++g) {
      if (qlogs[g] - 1 != llog) continue;
      CircleDomain dom = CanonicCoset(qlogs[g]).circle_domain();
      for (size_t p : lq.positions) {
        QM31 f0 = pair_vals[g].at(2 * p), f1 = pair_vals[g].at(2 * p + 1);
        CirclePoint<M31> pt = dom.at(bit_reverse_index(2 * p, qlogs[g]));
        ibutterfly(f0, f1, inv(pt.y));
        vals[p] = vals[p] * (circle_alpha * circle_alpha) + (circle_alpha * f1 + f0);
      }
    }
    if (k == fp.inner_layers.size()) { cur = vals; break; }
    const FriLayerProof& lp = fp.inner_layers[k];
    std::map<size_t, QM31> pv; std::vector<size_t> dpos; size_t w = 0;
    for (size_t i = 0; i < lq.positions.size();) {
      size_t j = i; while (j < lq.positions.size() && (lq.positions[j] >> 1) == (lq.positions[i] >> 1)) ++j;
      for (size_t p = (lq.positions[i] >> 1) << 1; p < ((lq.positions[i] >> 1) << 1) + 2; ++p) {
        dpos.push_back(p);
        if (vals.count(p)) pv[p] = vals[p];
        else { if (w >= lp.fri_witness.size()) throw VerifyError("fri: layer witness too short"); pv[p] = lp.fri_witness[w++]; }
      }
      i = j;
    }
    if (w != lp.fri_witness.size()) throw VerifyError("fri: layer witness too long");
    std::vector<M31> flatv; for (size_t p : dpos) for (int c = 0; c < 4; ++c) flatv.push_back(M31::raw(pv[p].coord(c)));
    std::map<uint32_t, std::vector<size_t>> dq; dq[llog] = dpos;
    merkle_verify(lp.commitment, std::vector<uint32_t>(4, llog), dq, flatv, lp.decommitment);
    LineDomain ld(Coset::half_odds(llog));
    Queries nq = lq.fold(1);
    std::map<size_t, QM31> nxt;
    for (size_t p : nq.positions) {
      QM31 f0 = pv.at(2 * p), f1 = pv.at(2 * p + 1);
      M31 x = ld.at(bit_reverse_index(2 * p, llog));
      ibutterfly(f0, f1, inv(x));
      nxt[p] = f0 + alphas[k] * f1;
    }
    cur = nxt; lq = nq; llog -= 1;
  }
  // last layer
  LineDomain last_dom(Coset::half_odds(llog));
  for (size_t p : lq.positions) {
    M31 x = last_dom.at(bit_reverse_index(p, llog));
    if (line_poly_eval(fp.last_layer_poly, fp.last_layer_log_size, QM31::from_m31(x)) != cur.at(p)) throw VerifyError("fri: last layer evaluation mismatch");
  }
}

}  // namespace orc
