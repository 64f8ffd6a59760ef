// AIR bytecode: host representation + parser (format: nexus_zkvm_b200/air.py docstring, DESIGN.md §AIR bytecode).
// The bytecode is what a recording `EvalAtRow` produces from the reference's chips
// (nexus-zkvm prover/src/traits.rs:45-50, prover/src/components/mod.rs:39-57); the constraint kernels interpret it.
#pragma once
#include "m31.cuh"
#include <string>
#include <utility>
#include <vector>
#include <stdexcept>

namespace nb {

enum AirOp : u32 {
  OP_LOADM = 0, OP_CONSTB = 1, OP_ADDB = 2, OP_SUBB = 3, OP_MULB = 4, OP_NEGB = 5,
  OP_PARAME = 6, OP_ADDE = 8, OP_SUBE = 9, OP_MULE = 10, OP_NEGE = 11,
  OP_ADDEB = 12, OP_SUBEB = 13, OP_MULEB = 14, OP_BTOE = 15, OP_LOADME = 16,
  OP_CONSTRB = 17, OP_CONSTRE = 18, OP_FRAC = 19
};
struct AirInstr { u32 op, dst, a, b; };
struct AirMask { u32 tree, col; int32_t off; };
struct AirComponent {
  u32 log_size = 0, log_expand = 0, n_constraints = 0;
  std::vector<AirMask> masks;
  u32 n_base_regs = 0, n_ext_regs = 0;
  std::vector<AirInstr> prog;
  u32 n_fracs = 0, lg_base_regs = 0, lg_ext_regs = 0;
  std::vector<AirInstr> logup_prog;
  std::vector<u32> batching;
  u32 cumsum_shift_param = 0xFFFFFFFFu, interaction_col0 = 0;
  u32 eval_log() const { return log_size + log_expand; }
  u32 n_logup_cols() const { u32 m = 0; for (u32 b : batching) m = b + 1 > m ? b + 1 : m; return m; }
};
struct AirProgram {
  u32 n_params = 0;
  std::vector<AirComponent> comps;
};

inline void air_check_prog(const std::vector<AirInstr>& prog, u32 nb_regs, u32 ne_regs, size_t n_masks, u32 n_params) {
  auto B = [&](u32 r) { if (r >= nb_regs) throw std::runtime_error("air: base register out of range"); };
  auto E = [&](u32 r) { if (r >= ne_regs) throw std::runtime_error("air: ext register out of range"); };
  for (const AirInstr& in : prog) {
    switch (in.op) {
      case OP_LOADM: B(in.dst); if (in.a >= n_masks) throw std::runtime_error("air: mask out of range"); break;
      case OP_CONSTB: B(in.dst); if (in.a >= P31) throw std::runtime_error("air: constant out of range"); break;
      case OP_ADDB: case OP_SUBB: case OP_MULB: B(in.dst); B(in.a); B(in.b); break;
      case OP_NEGB: B(in.dst); B(in.a); break;
      case OP_PARAME: E(in.dst); if (in.a >= n_params) throw std::runtime_error("air: param out of range"); break;
      case OP_ADDE: case OP_SUBE: case OP_MULE: E(in.dst); E(in.a); E(in.b); break;
      case OP_NEGE: E(in.dst); E(in.a); break;
      case OP_ADDEB: case OP_SUBEB: case OP_MULEB: E(in.dst); E(in.a); B(in.b); break;
      case OP_BTOE: E(in.dst); B(in.a); break;
      case OP_LOADME: E(in.dst); if ((size_t)in.a + 4 > n_masks) throw std::runtime_error("air: ext mask out of range"); break;
      case OP_CONSTRB: B(in.a); break;
      case OP_CONSTRE: E(in.a); break;
      case OP_FRAC: E(in.a); E(in.b); break;
      default: throw std::runtime_error("air: bad opcode");
    }
  }
}

inline AirProgram air_parse(const u32* w, size_t n) {
  size_t p = 0;
  auto rd = [&]() -> u32 { if (p >= n) throw std::runtime_error("air: truncated"); return w[p++]; };
  auto rd_prog = [&](std::vector<AirInstr>& out, u32 cnt) {
    for (u32 i = 0; i < cnt; ++i) { AirInstr in; in.op = rd(); in.dst = rd(); in.a = rd(); in.b = rd(); out.push_back(in); }
  };
  if (rd() != 0x5241424Eu) throw std::runtime_error("air: bad magic");
  if (rd() != 1) throw std::runtime_error("air: unsupported version");
  AirProgram a; a.n_params = rd();
  u32 nc = rd();
  for (u32 k = 0; k < nc; ++k) {
    AirComponent c;
    c.log_size = rd(); c.log_expand = rd(); c.n_constraints = rd();
    if (c.log_size < 1 || c.log_size + c.log_expand > 28) throw std::runtime_error("air: component size out of range");
    u32 nm = rd();
    for (u32 i = 0; i < nm; ++i) { AirMask m; m.tree = rd(); m.col = rd(); m.off = (int32_t)rd(); if (m.tree > 2) throw std::runtime_error("air: bad tree"); c.masks.push_back(m); }
    c.n_base_regs = rd(); c.n_ext_regs = rd();
    rd_prog(c.prog, rd());
    c.n_fracs = rd(); c.lg_base_regs = rd(); c.lg_ext_regs = rd();
    rd_prog(c.logup_prog, rd());
    for (u32 i = 0; i < c.n_fracs; ++i) c.batching.push_back(rd());
    c.cumsum_shift_param = rd(); c.interaction_col0 = rd();
    air_check_prog(c.prog, c.n_base_regs, c.n_ext_regs, c.masks.size(), a.n_params);
    air_check_prog(c.logup_prog, c.lg_base_regs, c.lg_ext_regs, c.masks.size(), a.n_params);
    // the interaction-trace generator reads the trace domain row by row: a lookup fraction built from a next-row value or from an interaction
    // column has no upstream counterpart (LogupTraceGenerator sees only the current row of the original / preprocessed traces) and would silently
    // read zeros in logup_generate — reject it here instead of failing the proof at the very end
    for (auto& in : c.logup_prog) {
      if (in.op == OP_LOADM && (c.masks[in.a].off != 0 || c.masks[in.a].tree == 2)) throw std::runtime_error("air: a logup fraction reads a mask with a row offset or an interaction column");
      if (in.op == OP_LOADME) throw std::runtime_error("air: a logup fraction reads an extension (interaction) mask");
    }
    u32 nconstr = 0, nfr = 0;
    for (auto& in : c.prog) if (in.op == OP_CONSTRB || in.op == OP_CONSTRE) ++nconstr;
    for (auto& in : c.logup_prog) if (in.op == OP_FRAC) ++nfr;
    if (nconstr != c.n_constraints || nfr != c.n_fracs) throw std::runtime_error("air: constraint/fraction count mismatch");
    for (size_t i = 1; i < c.batching.size(); ++i) if (c.batching[i] < c.batching[i - 1] || c.batching[i] > c.batching[i - 1] + 1) throw std::runtime_error("air: logup batching must be non-decreasing");
    if (!c.batching.empty() && c.batching[0] != 0) throw std::runtime_error("air: logup batching must start at 0");
    a.comps.push_back(std::move(c));
  }
  if (p != n) throw std::runtime_error("air: trailing words");
  return a;
}

// Degree of each constraint (declaration order) in the trace polynomials, walked over the constraint program: a mask has degree 1,
// a constant or a parameter 0, a product the sum of its operands' degrees and a sum or difference their maximum.
inline std::vector<u32> constraint_degrees(const AirComponent& c) {
  std::vector<u32> db(c.n_base_regs + 1, 0), de(c.n_ext_regs + 1, 0), out;
  auto mx = [](u32 x, u32 y) { return x > y ? x : y; };
  for (const AirInstr& in : c.prog) {
    switch (in.op) {
      case OP_LOADM: db[in.dst] = 1; break;
      case OP_CONSTB: db[in.dst] = 0; break;
      case OP_ADDB: case OP_SUBB: db[in.dst] = mx(db[in.a], db[in.b]); break;
      case OP_MULB: db[in.dst] = db[in.a] + db[in.b]; break;
      case OP_NEGB: db[in.dst] = db[in.a]; break;
      case OP_PARAME: de[in.dst] = 0; break;
      case OP_LOADME: de[in.dst] = 1; break;
      case OP_ADDE: case OP_SUBE: de[in.dst] = mx(de[in.a], de[in.b]); break;
      case OP_MULE: de[in.dst] = de[in.a] + de[in.b]; break;
      case OP_NEGE: de[in.dst] = de[in.a]; break;
      case OP_ADDEB: case OP_SUBEB: de[in.dst] = mx(de[in.a], db[in.b]); break;
      case OP_MULEB: de[in.dst] = de[in.a] + db[in.b]; break;
      case OP_BTOE: de[in.dst] = db[in.a]; break;
      case OP_CONSTRB: out.push_back(db[in.a]); break;
      case OP_CONSTRE: out.push_back(de[in.a]); break;
      default: break;
    }
  }
  return out;
}

// A constraint of degree d has a quotient C / Z of circle degree (d - 1) 2^log_size: for d <= 2 it lies in the span of the first
// 2^(log_size + 2) circle-FFT basis vectors, the part of the composition a Q_HALF component interpolates from the committed LDE domain
// alone (prove.cu, component_quotients).  Only the constraints above that bound contribute to the upper half.
static const u32 AIR_LOW_DEGREE = 2;
inline std::vector<char> high_constraints(const AirComponent& c) {
  std::vector<char> h;
  for (u32 d : constraint_degrees(c)) h.push_back(d > AIR_LOW_DEGREE ? 1 : 0);
  return h;
}
inline size_t count_high(const std::vector<char>& high) { size_t n = 0; for (char x : high) n += x ? 1 : 0; return n; }

// The masks the constraints flagged in `keep` read (directly or through shared subexpressions, at any row offset): a backward walk over
// the program from those constraints' sinks.
inline std::vector<char> masks_read_by(const AirComponent& c, const std::vector<char>& keep) {
  std::vector<char> nb(c.n_base_regs + 1, 0), ne(c.n_ext_regs + 1, 0), used(c.masks.size(), 0);
  u32 k = c.n_constraints;
  for (size_t pc = c.prog.size(); pc-- > 0;) {
    const AirInstr& in = c.prog[pc];
    switch (in.op) {
      case OP_CONSTRB: if (keep[--k]) nb[in.a] = 1; break;
      case OP_CONSTRE: if (keep[--k]) ne[in.a] = 1; break;
      case OP_LOADM: if (nb[in.dst]) used[in.a] = 1; nb[in.dst] = 0; break;
      case OP_CONSTB: nb[in.dst] = 0; break;
      case OP_ADDB: case OP_SUBB: case OP_MULB: if (nb[in.dst]) { nb[in.dst] = 0; nb[in.a] = nb[in.b] = 1; } break;
      case OP_NEGB: if (nb[in.dst]) { nb[in.dst] = 0; nb[in.a] = 1; } break;
      case OP_PARAME: ne[in.dst] = 0; break;
      case OP_LOADME: if (ne[in.dst]) for (u32 i = 0; i < 4; ++i) used[in.a + i] = 1; ne[in.dst] = 0; break;
      case OP_ADDE: case OP_SUBE: case OP_MULE: if (ne[in.dst]) { ne[in.dst] = 0; ne[in.a] = ne[in.b] = 1; } break;
      case OP_NEGE: if (ne[in.dst]) { ne[in.dst] = 0; ne[in.a] = 1; } break;
      case OP_ADDEB: case OP_SUBEB: case OP_MULEB: if (ne[in.dst]) { ne[in.dst] = 0; ne[in.a] = 1; nb[in.b] = 1; } break;
      case OP_BTOE: if (ne[in.dst]) { ne[in.dst] = 0; nb[in.a] = 1; } break;
      default: break;
    }
  }
  return used;
}

// register kind ('b' base, 'e' secure, 0 none) of operands a and b and of the destination
inline void operand_kinds(u32 op, char& ka, char& kb, char& kd) {
  ka = kb = kd = 0;
  switch (op) {
    case OP_LOADM: case OP_CONSTB: kd = 'b'; break;
    case OP_ADDB: case OP_SUBB: case OP_MULB: ka = kb = kd = 'b'; break;
    case OP_NEGB: ka = kd = 'b'; break;
    case OP_PARAME: case OP_LOADME: kd = 'e'; break;
    case OP_ADDE: case OP_SUBE: case OP_MULE: ka = kb = kd = 'e'; break;
    case OP_NEGE: ka = kd = 'e'; break;
    case OP_ADDEB: case OP_SUBEB: case OP_MULEB: ka = kd = 'e'; kb = 'b'; break;
    case OP_BTOE: ka = 'b'; kd = 'e'; break;
    case OP_CONSTRB: ka = 'b'; break;
    case OP_CONSTRE: ka = 'e'; break;
    case OP_FRAC: ka = kb = 'e'; break;
    default: break;
  }
}

// Reaching definitions: def_a / def_b[pc] = position of the instruction whose result operand a / b of prog[pc] reads (-1: none).  Registers
// are reused, so a register number alone names nothing; a position does.
inline void prog_defs(const std::vector<AirInstr>& prog, u32 nb, u32 ne, std::vector<int>& def_a, std::vector<int>& def_b) {
  const int n = (int)prog.size();
  def_a.assign(n, -1); def_b.assign(n, -1);
  std::vector<int> cur_b(nb + 1, -1), cur_e(ne + 1, -1);
  for (int pc = 0; pc < n; ++pc) {
    const AirInstr& in = prog[pc];
    char ka, kb, kd;
    operand_kinds(in.op, ka, kb, kd);
    if (ka) def_a[pc] = (ka == 'b' ? cur_b : cur_e)[in.a];
    if (kb) def_b[pc] = (kb == 'b' ? cur_b : cur_e)[in.b];
    if (kd) (kd == 'b' ? cur_b : cur_e)[in.dst] = pc;
  }
}

// ---- lookup tables and their lookups, read off the logup programs (nb200_table_multiplicities)
// Every fraction's denominator is Relation::combine (air.py ComponentBuilder.combine): sum_i alpha_i v_i - z, i.e.
//   SUBE(ADDE(..ADDE(MULEB(PARAME alpha_0, v_0), MULEB(PARAME alpha_1, v_1)).., MULEB(PARAME alpha_n-1, v_n-1)), PARAME z).
// The relation is named by its z parameter, the tuple is (v_0 .. v_n-1).  A table fraction has the numerator -m for one tree-1 mask m (its
// multiplicity column) and a tuple that reads tree-0 masks and constants only; every other fraction into a relation that has a table
// fraction is a lookup of that table, and must have a base-field numerator.  Relations without a table fraction are not counted.
enum FracKind : u32 { FRAC_IGNORED = 0, FRAC_TABLE = 1, FRAC_LOOKUP = 2, FRAC_BAD = 3 };
struct AirFrac {
  u32 kind = FRAC_IGNORED;
  u32 rel = 0xFFFFFFFFu;     // z parameter of the relation (0xFFFFFFFF: the denominator does not parse)
  u32 mult_mask = 0;         // FRAC_TABLE: the mask of the multiplicity column
  int num = -1;              // position of the base value whose BTOE is the numerator (-1: not a base value)
  std::vector<int> tuple;    // positions of the instructions that compute v_0 .. v_n-1
  std::string why;           // FRAC_BAD: what does not parse
};
inline std::vector<std::vector<AirFrac>> air_lookup_tables(const AirProgram& a) {
  std::vector<std::vector<AirFrac>> out(a.comps.size());
  std::vector<char> has_table(a.n_params, 0);
  std::vector<std::vector<u32>> alphas(a.n_params);   // per z: the alpha parameter of each tuple position seen so far
  for (size_t k = 0; k < a.comps.size(); ++k) {
    const AirComponent& c = a.comps[k];
    const std::vector<AirInstr>& prog = c.logup_prog;
    std::vector<int> da, db;
    prog_defs(prog, c.lg_base_regs, c.lg_ext_regs, da, db);
    std::vector<signed char> t0(prog.size(), -1);     // memo: the base value reads tree-0 masks and constants only
    auto only_tree0 = [&](int q, auto& self) -> bool {
      if (q < 0) return false;
      if (t0[q] >= 0) return t0[q] != 0;
      const AirInstr& in = prog[q];
      bool r = false;
      switch (in.op) {
        case OP_LOADM: r = c.masks[in.a].tree == 0; break;
        case OP_CONSTB: r = true; break;
        case OP_ADDB: case OP_SUBB: case OP_MULB: r = self(da[q], self) && self(db[q], self); break;
        case OP_NEGB: r = self(da[q], self); break;
        default: break;
      }
      t0[q] = r ? 1 : 0;
      return r;
    };
    auto param = [&](int q) { return q >= 0 && prog[q].op == OP_PARAME; };
    for (size_t pc = 0; pc < prog.size(); ++pc) {
      if (prog[pc].op != OP_FRAC) continue;
      AirFrac f;
      const int d = db[pc];
      if (d >= 0 && prog[d].op == OP_SUBE && param(db[d])) {
        f.rel = prog[db[d]].a;
        std::vector<std::pair<u32, int>> terms;   // (alpha parameter, value), last term first
        auto term = [&](int t) {
          if (t < 0 || prog[t].op != OP_MULEB || !param(da[t]) || db[t] < 0) return false;
          terms.push_back({prog[da[t]].a, db[t]});
          return true;
        };
        bool ok = true;
        int x = da[d];
        while (ok && x >= 0 && prog[x].op == OP_ADDE) { ok = term(db[x]); x = da[x]; }
        ok = ok && term(x);
        if (ok) {
          std::vector<u32>& al = alphas[f.rel];
          for (size_t i = 0; i < terms.size() && ok; ++i) {
            const u32 alpha = terms[terms.size() - 1 - i].first;
            if (i < al.size()) ok = al[i] == alpha;
            else al.push_back(alpha);
            f.tuple.push_back(terms[terms.size() - 1 - i].second);
          }
          if (!ok) f.why = "the tuple's alpha parameters differ from another fraction's of the same relation";
        } else {
          f.why = "the denominator is not sum_i alpha_i v_i - z with base-field v_i";
        }
        if (!ok) { f.kind = FRAC_BAD; f.tuple.clear(); }
      } else {
        f.kind = FRAC_BAD;
        f.why = "the denominator is not a combination minus the relation's z parameter";
      }
      const int nq = da[pc];
      if (nq >= 0 && prog[nq].op == OP_BTOE) f.num = da[nq];
      if (f.kind != FRAC_BAD && f.num >= 0 && prog[f.num].op == OP_NEGB) {
        const int m = da[f.num];
        bool table = m >= 0 && prog[m].op == OP_LOADM && c.masks[prog[m].a].tree == 1 && c.masks[prog[m].a].off == 0;
        for (int v : f.tuple) table = table && only_tree0(v, only_tree0);
        if (table) { f.kind = FRAC_TABLE; f.mult_mask = prog[m].a; has_table[f.rel] = 1; }
      }
      out[k].push_back(std::move(f));
    }
  }
  for (auto& comp : out)
    for (AirFrac& f : comp) {
      if (f.kind == FRAC_TABLE) continue;
      const bool into_table = f.rel < a.n_params && has_table[f.rel];
      if (f.kind == FRAC_BAD) { if (f.rel < a.n_params && !into_table) f.kind = FRAC_IGNORED; continue; }   // not needed
      if (!into_table) continue;
      if (f.num < 0) { f.kind = FRAC_BAD; f.why = "a lookup into a table has a numerator outside the base field"; continue; }
      f.kind = FRAC_LOOKUP;
    }
  return out;
}

}  // namespace nb
