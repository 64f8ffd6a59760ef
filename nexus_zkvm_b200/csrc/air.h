// AIR bytecode: host representation + parser (format: nexus_zkvm_b200/air.py docstring, DESIGN.md §AIR bytecode).
// The bytecode is what a recording `EvalAtRow` produces from the reference's chips
// (nexus-zkvm prover/src/traits.rs:45-50, prover/src/components/mod.rs:39-57); the constraint kernels interpret it.
#pragma once
#include "m31.cuh"
#include <string>
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

}  // namespace nb
