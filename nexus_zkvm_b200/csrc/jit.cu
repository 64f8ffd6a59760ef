// Runtime specialisation of an AIR component's constraint program: the SSA bytecode (air.h) is translated to CUDA C,
// compiled once per loaded AIR with NVRTC for sm_90a and launched instead of the bytecode interpreter
// (interp.cu).  Same arithmetic, same accumulation order => bit-identical results; the point is that the virtual
// registers become machine registers and the decode loop disappears (SURVEY.md §7.3-4 "NVRTC-specialised kernel").
// Replaces, like the interpreter, FrameworkComponent::evaluate_constraint_quotients_on_domain reached from
// stwo::prover::prove at nexus-zkvm prover/src/machine.rs:286-290.
//
// libnvrtc is opened with dlopen at first use; if it is missing (or NB200_JIT=0) the interpreter kernels — also CUDA —
// are used.  The generated function is cut into __noinline__ chunks of a few hundred statements: NVVM's optimiser is
// super-linear in function size (27 s for one 4400-statement function vs 7 s chunked, measured).
#include "pcs.h"
#include "jit.h"
#include <dlfcn.h>
#include <unistd.h>
#include <cstring>
#include <cstdio>
#include <nvrtc.h>
#include <sstream>
#include <algorithm>
#include <functional>
#include <map>
#include <cstdlib>

namespace nb {

namespace {
struct Nvrtc {
  void* h = nullptr;
  nvrtcResult (*CreateProgram)(nvrtcProgram*, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
  nvrtcResult (*CompileProgram)(nvrtcProgram, int, const char* const*) = nullptr;
  nvrtcResult (*GetCUBINSize)(nvrtcProgram, size_t*) = nullptr;
  nvrtcResult (*GetCUBIN)(nvrtcProgram, char*) = nullptr;
  nvrtcResult (*GetProgramLogSize)(nvrtcProgram, size_t*) = nullptr;
  nvrtcResult (*GetProgramLog)(nvrtcProgram, char*) = nullptr;
  nvrtcResult (*DestroyProgram)(nvrtcProgram*) = nullptr;
  bool ok = false;
};
Nvrtc& nvrtc() {
  static Nvrtc n;
  static bool tried = false;
  if (tried) return n;
  tried = true;
  const char* names[] = {"libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so.12"};
  for (const char* nm : names) { n.h = dlopen(nm, RTLD_NOW | RTLD_LOCAL); if (n.h) break; }
  if (!n.h) return n;
#define NB_SYM(f) n.f = (decltype(n.f))dlsym(n.h, "nvrtc" #f); if (!n.f) return n;
  NB_SYM(CreateProgram) NB_SYM(CompileProgram) NB_SYM(GetCUBINSize) NB_SYM(GetCUBIN) NB_SYM(GetProgramLogSize) NB_SYM(GetProgramLog) NB_SYM(DestroyProgram)
#undef NB_SYM
  n.ok = true;
  return n;
}

const char* kPrelude = R"SRC(
typedef unsigned int u32; typedef unsigned long long u64;
#define P31 0x7fffffffu
struct Q { u32 c0, c1, c2, c3; };
__device__ __forceinline__ u32 mn(u32 a, u32 b) { return a < b ? a : b; }
__device__ __forceinline__ u32 add(u32 a, u32 b) { u32 s = a + b; return mn(s, s - P31); }
__device__ __forceinline__ u32 sub(u32 a, u32 b) { u32 d = a - b; return mn(d, d + P31); }
__device__ __forceinline__ u32 neg(u32 a) { return a ? P31 - a : 0u; }
// one product: a * 2b = hi * 2^32 + lo  =>  a * b = hi * 2^31 + lo / 2 == hi + lo / 2 (mod P), below 2P
__device__ __forceinline__ u32 mul2(u32 a, u32 b2) { u64 p = (u64)a * (u64)b2; u32 s = (u32)(p >> 32) + ((u32)p >> 1); return mn(s, s - P31); }
__device__ __forceinline__ u32 mul(u32 a, u32 b) { return mul2(a, b + b); }
// canonical residue of any 64-bit value: 2^32 == 2 and 2^31 == 1 (mod P)
__device__ __forceinline__ u32 red64(u64 x) {
  u64 y;                                                // y = 2 * hi + lo < 3 * 2^32 (mad.wide keeps NVVM from expanding it into a carry chain)
  asm("mad.wide.u32 %0, %1, 2, %2;" : "=l"(y) : "r"((u32)(x >> 32)), "l"((u64)(u32)x));
  u32 yl = (u32)y, yh = (u32)(y >> 32);
  u32 s = (yl & P31) + __funnelshift_r(yl, yh, 31);     // <= P + 5
  return mn(s, s - P31);
}
__device__ __forceinline__ Q qadd(Q x, Q y) { return Q{add(x.c0, y.c0), add(x.c1, y.c1), add(x.c2, y.c2), add(x.c3, y.c3)}; }
__device__ __forceinline__ Q qsub(Q x, Q y) { return Q{sub(x.c0, y.c0), sub(x.c1, y.c1), sub(x.c2, y.c2), sub(x.c3, y.c3)}; }
__device__ __forceinline__ Q qneg(Q x) { return Q{neg(x.c0), neg(x.c1), neg(x.c2), neg(x.c3)}; }
__device__ __forceinline__ Q qmulb(Q x, u32 b) { u32 b2 = b + b; return Q{mul2(x.c0, b2), mul2(x.c1, b2), mul2(x.c2, b2), mul2(x.c3, b2)}; }
__device__ __forceinline__ Q qaddb(Q x, u32 b) { x.c0 = add(x.c0, b); return x; }
__device__ __forceinline__ Q qsubb(Q x, u32 b) { x.c0 = sub(x.c0, b); return x; }
// acc + x * y in QM31 with every coordinate accumulated in 64 bits and reduced once.  (a + bu)(c + du) = (ac + R bd) + (ad + bc)u,
// R = 2 + i (the formula of m31.cuh qm31_mul), regrouped per coordinate of x so that each output is four products:
//   r0 = x0 y0 - x1 y1 + x2 (2 y2 - y3) - x3 (y2 + 2 y3)      r1 = x0 y1 + x1 y0 + x2 (y2 + 2 y3) + x3 (2 y2 - y3)
//   r2 = x0 y2 - x1 y3 + x2 y0 - x3 y1                        r3 = x0 y3 + x1 y2 + x2 y1 + x3 y0
// ny1 = P - y1, ny3 = P - y3, g = 2 y2 - y3, gp = y2 + 2 y3, h = P - gp: all <= P, so 4 products + acc < 2^64.
__device__ __forceinline__ Q qmac(Q acc, Q x, u32 y0, u32 y1, u32 y2, u32 y3, u32 ny1, u32 ny3, u32 g, u32 gp, u32 h) {
  u64 r0 = (u64)acc.c0 + (u64)x.c0 * y0 + (u64)x.c1 * ny1 + (u64)x.c2 * g + (u64)x.c3 * h;
  u64 r1 = (u64)acc.c1 + (u64)x.c0 * y1 + (u64)x.c1 * y0 + (u64)x.c2 * gp + (u64)x.c3 * g;
  u64 r2 = (u64)acc.c2 + (u64)x.c0 * y2 + (u64)x.c1 * ny3 + (u64)x.c2 * y0 + (u64)x.c3 * ny1;
  u64 r3 = (u64)acc.c3 + (u64)x.c0 * y3 + (u64)x.c1 * y2 + (u64)x.c2 * y1 + (u64)x.c3 * y0;
  return Q{red64(r0), red64(r1), red64(r2), red64(r3)};
}
__device__ __forceinline__ Q qmul(Q x, Q y) {
  u32 gp = add(add(y.c3, y.c3), y.c2), g = sub(add(y.c2, y.c2), y.c3);
  return qmac(Q{0u, 0u, 0u, 0u}, x, y.c0, y.c1, y.c2, y.c3, P31 - y.c1, P31 - y.c3, g, gp, P31 - gp);
}
// x^(P-2): 30 squarings + 8 products
__device__ __forceinline__ u32 sqn(u32 x, int n) { for (int i = 0; i < n; ++i) x = mul(x, x); return x; }
__device__ __forceinline__ u32 minv(u32 x) {
  u32 a2 = mul(sqn(x, 1), x), a4 = mul(sqn(a2, 2), a2), a8 = mul(sqn(a4, 4), a4), a16 = mul(sqn(a8, 8), a8);
  u32 a24 = mul(sqn(a16, 8), a8), a28 = mul(sqn(a24, 4), a4), a29 = mul(sqn(a28, 1), x);
  return mul(sqn(a29, 2), x);
}
// (a + bu)^-1 = (a - bu) / (a^2 - (2 + i) b^2), a, b in CM31 (the formula of m31.cuh qm31_inv); the CM31 inverse is conj / norm
__device__ __noinline__ Q qinv(Q q) {
  u32 b2r = sub(mul(q.c2, q.c2), mul(q.c3, q.c3)), b2i = mul(add(q.c2, q.c2), q.c3);           // b^2
  u32 a2r = sub(mul(q.c0, q.c0), mul(q.c1, q.c1)), a2i = mul(add(q.c0, q.c0), q.c1);           // a^2
  u32 dr = sub(a2r, sub(add(b2r, b2r), b2i)), di = sub(a2i, add(add(b2i, b2i), b2r));          // a^2 - (2 b^2 + i b^2)
  u32 ni = minv(add(mul(dr, dr), mul(di, di)));
  u32 ir = mul(dr, ni), ii = neg(mul(di, ni));                                                 // 1 / denom
  return Q{sub(mul(q.c0, ir), mul(q.c1, ii)), add(mul(q.c0, ii), mul(q.c1, ir)),
           neg(sub(mul(q.c2, ir), mul(q.c3, ii))), neg(add(mul(q.c2, ii), mul(q.c3, ir)))};
}
__device__ __forceinline__ Q ldq(const u32* p) { uint4 v = __ldg(reinterpret_cast<const uint4*>(p)); return Q{v.x, v.y, v.z, v.w}; }
// rr + coeff * x with the coefficient's derived multipliers precomputed by the host (12 words per constraint, see jit_coeff_table)
__device__ __forceinline__ Q qmac_tab(Q acc, Q x, const u32* t) {
  uint4 a = __ldg(reinterpret_cast<const uint4*>(t)), b = __ldg(reinterpret_cast<const uint4*>(t) + 1), c = __ldg(reinterpret_cast<const uint4*>(t) + 2);
  return qmac(acc, x, a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x);
}
)SRC";

// the arithmetic / load opcodes shared by the constraint and the logup programs
template <class Ld>
void emit_op(std::ostringstream& o, const AirInstr& in, Ld ld) {
  switch (in.op) {
    case OP_LOADM: o << "b[" << in.dst << "] = " << ld(in.a) << ";"; break;
    case OP_CONSTB: o << "b[" << in.dst << "] = " << in.a << "u;"; break;
    case OP_ADDB: o << "b[" << in.dst << "] = add(b[" << in.a << "], b[" << in.b << "]);"; break;
    case OP_SUBB: o << "b[" << in.dst << "] = sub(b[" << in.a << "], b[" << in.b << "]);"; break;
    case OP_MULB: o << "b[" << in.dst << "] = mul(b[" << in.a << "], b[" << in.b << "]);"; break;
    case OP_NEGB: o << "b[" << in.dst << "] = neg(b[" << in.a << "]);"; break;
    case OP_PARAME: o << "e[" << in.dst << "] = ldq(params + " << 4 * in.a << ");"; break;
    case OP_ADDE: o << "e[" << in.dst << "] = qadd(e[" << in.a << "], e[" << in.b << "]);"; break;
    case OP_SUBE: o << "e[" << in.dst << "] = qsub(e[" << in.a << "], e[" << in.b << "]);"; break;
    case OP_MULE: o << "e[" << in.dst << "] = qmul(e[" << in.a << "], e[" << in.b << "]);"; break;
    case OP_NEGE: o << "e[" << in.dst << "] = qneg(e[" << in.a << "]);"; break;
    case OP_ADDEB: o << "e[" << in.dst << "] = qaddb(e[" << in.a << "], b[" << in.b << "]);"; break;
    case OP_SUBEB: o << "e[" << in.dst << "] = qsubb(e[" << in.a << "], b[" << in.b << "]);"; break;
    case OP_MULEB: o << "e[" << in.dst << "] = qmulb(e[" << in.a << "], b[" << in.b << "]);"; break;
    case OP_BTOE: o << "e[" << in.dst << "] = Q{b[" << in.a << "], 0u, 0u, 0u};"; break;
    case OP_LOADME: o << "e[" << in.dst << "] = Q{" << ld(in.a) << ", " << ld(in.a + 1) << ", " << ld(in.a + 2) << ", " << ld(in.a + 3) << "};"; break;
    default: break;
  }
}

struct Regs { std::vector<u32> rb, re; int wb = -1, we = -1; };   // registers a statement reads and writes (base / secure)
static Regs instr_regs(const AirInstr& in) {
  Regs r;
  char ka, kb, kd;
  operand_kinds(in.op, ka, kb, kd);
  if (ka) (ka == 'b' ? r.rb : r.re).push_back(in.a);
  if (kb) (kb == 'b' ? r.rb : r.re).push_back(in.b);
  if (kd) (kd == 'b' ? r.wb : r.we) = (int)in.dst;
  return r;
}
struct Stmt { std::string code; Regs r; bool effect = false; int constr = -1; };   // effect: adds constraint `constr` to rr (never removed as dead)
template <class Ld>
static Stmt op_stmt(const AirInstr& in, Ld ld) {
  std::ostringstream o;
  emit_op(o, in, ld);
  return Stmt{o.str(), instr_regs(in)};
}

// Which virtual registers cross a chunk boundary?  in[ci] = registers read in chunk ci or later before they are rewritten.  A chunk loads only
// those from the state struct and stores only the ones it wrote that a later chunk still reads: the real v1 AIR keeps 26 base + 15 secure
// registers alive somewhere (shared selectors such as IsTypeR), and copying all 90 words in and out of local memory at each of its 19 chunk
// boundaries cost more than the arithmetic (the synthetic ADD machine has 4 + 4 and never showed it).
struct ChunkLive { std::vector<std::vector<u32>> in_b, in_e, out_b, out_e; };
// chunk ci is the statements of program positions [ci * ch, (ci + 1) * ch)
static ChunkLive chunk_liveness(const std::vector<std::vector<Stmt>>& at, size_t ch, u32 nb, u32 ne) {
  const size_t n_chunks = (at.size() + ch - 1) / ch;
  auto end = [&](size_t ci) { return std::min(at.size(), (ci + 1) * ch); };
  ChunkLive L; L.in_b.resize(n_chunks); L.in_e.resize(n_chunks); L.out_b.resize(n_chunks); L.out_e.resize(n_chunks);
  std::vector<char> lb(nb + 1, 0), le(ne + 1, 0);
  std::vector<std::vector<char>> after_b(n_chunks), after_e(n_chunks);   // live sets at the END of each chunk
  for (size_t ci = n_chunks; ci-- > 0;) {
    after_b[ci] = lb; after_e[ci] = le;
    for (size_t pc = end(ci); pc-- > ci * ch;)
      for (size_t i = at[pc].size(); i-- > 0;) {
        const Regs& r = at[pc][i].r;
        if (r.wb >= 0) lb[r.wb] = 0;
        if (r.we >= 0) le[r.we] = 0;
        for (u32 x : r.rb) lb[x] = 1;
        for (u32 x : r.re) le[x] = 1;
      }
    for (u32 r = 0; r < nb; ++r) if (lb[r]) L.in_b[ci].push_back(r);
    for (u32 r = 0; r < ne; ++r) if (le[r]) L.in_e[ci].push_back(r);
  }
  for (size_t ci = 0; ci < n_chunks; ++ci) {
    std::vector<char> wrb(nb + 1, 0), wre(ne + 1, 0);
    for (size_t pc = ci * ch; pc < end(ci); ++pc)
      for (const Stmt& st : at[pc]) {
        if (st.r.wb >= 0) wrb[st.r.wb] = 1;
        if (st.r.we >= 0) wre[st.r.we] = 1;
      }
    for (u32 r = 0; r < nb; ++r) if (wrb[r] && after_b[ci][r]) L.out_b[ci].push_back(r);
    for (u32 r = 0; r < ne; ++r) if (wre[r] && after_e[ci][r]) L.out_e[ci].push_back(r);
  }
  return L;
}

// column base pointers live in constant memory (filled before every launch, jit_launch): an access costs no pointer load from global memory
// (the real AIR reads 2765 mask values per row: one dependent global load less per value)
static std::string ccols_decl(const AirComponent& c) {
  return "#define NB_NMASKS " + std::to_string(c.masks.size()) + "\n__constant__ const u32* ccols[NB_NMASKS > 0 ? NB_NMASKS : 1];\n";
}

// The kernel the constraint (D1 and D2), LogUp and check programs are generated as.  at[pc] holds the statements of program position pc; the
// positions are cut into __noinline__ chunks of `ch`, each of which loads the registers it reads from the state struct St and stores the ones
// a later chunk reads (chunk_liveness).  A chunk without code is left out.  The strings are the parts that differ between the programs.
struct ChunkedKernel {
  size_t ch = 0;
  u32 nb = 0, ne = 0;      // base / secure registers
  std::string state;       // St's fields after the registers
  std::string decls;       // between the column table and the first chunk
  std::string params;      // a chunk's parameters after St& s
  std::string enter;       // the end of a chunk's first line: its state fields loaded from s
  std::string leave;       // a chunk's last lines: its state fields stored back
  std::string last;        // lines at the end of the last chunk, before its stores
  std::string sig;         // nbjit's parameters
  std::string prologue;    // nbjit's lines before St s
  std::string init;        // nbjit's lines after the registers are zeroed
  std::string args;        // a chunk call's arguments after s
  std::string epilogue;    // nbjit's lines after the last chunk
};
static void emit_chunked(std::ostringstream& o, const AirComponent& c, const std::vector<std::vector<Stmt>>& at, const ChunkedKernel& k) {
  const size_t n_chunks = (at.size() + k.ch - 1) / k.ch;
  const ChunkLive live = chunk_liveness(at, k.ch, k.nb, k.ne);
  o << "struct St { u32 b[" << k.nb << "]; Q e[" << k.ne << "];" << k.state << " };\n" << ccols_decl(c) << k.decls;
  std::vector<char> has_code(n_chunks, 0);   // the D2 kernel leaves out most statements
  for (size_t pc = 0; pc < at.size(); ++pc)
    for (const Stmt& st : at[pc]) if (!st.code.empty()) has_code[pc / k.ch] = 1;
  for (size_t ci = 0; ci < n_chunks; ++ci) {
    if (!has_code[ci]) continue;
    o << "__device__ __noinline__ void chunk" << ci << "(St& s, " << k.params << ") {\n";
    o << "  u32 b[" << k.nb << "]; Q e[" << k.ne << "];" << k.enter << "\n";
    for (u32 r : live.in_b[ci]) o << "  b[" << r << "] = s.b[" << r << "];";
    for (u32 r : live.in_e[ci]) o << "  e[" << r << "] = s.e[" << r << "];";
    o << "\n";
    for (size_t pc = ci * k.ch; pc < std::min(at.size(), (ci + 1) * k.ch); ++pc) {
      o << "  ";
      for (size_t i = 0; i < at[pc].size(); ++i) o << (i ? " " : "") << at[pc][i].code;
      o << "\n";
    }
    if (ci + 1 == n_chunks) o << k.last;
    for (u32 r : live.out_b[ci]) o << "  s.b[" << r << "] = b[" << r << "];";
    for (u32 r : live.out_e[ci]) o << "  s.e[" << r << "] = e[" << r << "];";
    o << "\n" << k.leave << "}\n";
  }
  // The CTAs re-converge (__syncthreads) after every chunk: the warps of a CTA then execute the same few tens of KB of straight-line
  // code at a time and the instruction cache serves them from one fetch.  Without the barriers the warps drift apart over the ~0.7 MB
  // program and the kernel becomes instruction-fetch bound.
  o << "extern \"C\" __global__ void __launch_bounds__(" << JIT_BLOCK << ", 1) nbjit(" << k.sig << ") {\n" << k.prologue << "  St s;\n"
    << "  for (int i = 0; i < " << k.nb << "; ++i) s.b[i] = 0u;\n  for (int i = 0; i < " << k.ne << "; ++i) s.e[i] = Q{0u, 0u, 0u, 0u};\n" << k.init;
  for (size_t ci = 0; ci < n_chunks; ++ci)
    if (has_code[ci]) o << "  chunk" << ci << "(s, " << k.args << ");\n  __syncthreads();\n";
  o << k.epilogue << "}\n";
}

// ---- folding the random coefficient into LogUp denominators
// finalize_logup_batched (air.py) emits every LogUp constraint of a single fraction as coeff * (diff * den - num), where
// den = sum_i alpha^i v_i - z is linear in the parameters with base-field v_i, and num is a base value.  In the field
//   coeff * (diff * den - num) = diff * (coeff * den) - coeff * num,   coeff * den = sum_i (coeff alpha^i) v_i - coeff z,
// so once the products coeff * alpha^i and coeff * z are known, coeff * den costs the 4 products per term that den costs and the
// constraint's full QM31 product by its coefficient disappears (16 products and 4 reductions per row).  The kernel computes those
// products once per CTA into shared memory (nbfold); field arithmetic is exact, so every accumulator word stays the same.
// A constraint folds when, by reaching definitions (registers are reused, so a register number alone names nothing):
//   CONSTRE(SUBE(MULE(diff, den) or MULE(den, diff), BTOE(base))), den an ADDE / SUBE tree over MULEB(PARAME, base) and PARAME,
// and the SUBE and MULE results have no other reader.  Fractions batched in pairs (den a product of two denominators) do not.
// The den's own terms and partial sums may be shared with other constraints (air.py merges equal nodes), so they are not scaled in
// place: coeff * den is summed afresh at the MULE from the base values the den read, and a base value whose register is rewritten
// before that point is first copied to a register of its own.  Whatever only the folded dens read is then dropped as dead code.
struct ConstraintPlan {
  std::vector<std::vector<Stmt>> at;               // the statements emitted at each program position
  u32 nb = 0;                                      // base registers, the copies of folded base values included
  std::vector<std::pair<u32, u32>> slots;          // nbfold[i] = coeff[slots[i].first] * params[slots[i].second]
};

// `keep[k] == 0`: constraint k is left out (with everything only it reads)
template <class Ld>
static ConstraintPlan plan_constraints(const AirComponent& c, Ld ld, u32 nb, u32 ne, const std::vector<char>& keep) {
  const std::vector<AirInstr>& prog = c.prog;
  const int n = (int)prog.size();
  // def_a / def_b[pc]: position of the instruction whose result operand a / b of prog[pc] reads (-1: none);
  // uses[d]: readers of the result of d; next_def[d]: position of the next write to d's destination register
  std::vector<int> def_a(n, -1), def_b(n, -1), uses(n, 0), next_def(n, n);
  {
    std::vector<int> cur_b(nb, -1), cur_e(ne, -1);
    for (int pc = 0; pc < n; ++pc) {
      const AirInstr& in = prog[pc];
      char ka, kb, kd;
      operand_kinds(in.op, ka, kb, kd);
      if (ka) { def_a[pc] = (ka == 'b' ? cur_b : cur_e)[in.a]; if (def_a[pc] >= 0) ++uses[def_a[pc]]; }
      if (kb) { def_b[pc] = (kb == 'b' ? cur_b : cur_e)[in.b]; if (def_b[pc] >= 0) ++uses[def_b[pc]]; }
      if (kd) {
        int& cur = (kd == 'b' ? cur_b : cur_e)[in.dst];
        if (cur >= 0) next_def[cur] = pc;
        cur = pc;
      }
    }
  }
  ConstraintPlan pl;
  pl.nb = nb;
  pl.at.resize(n);
  u32 k = 0;
  std::vector<u32> coeff_of(n, 0);   // constraint index of each CONSTRB / CONSTRE
  for (int pc = 0; pc < n; ++pc) {
    const AirInstr& in = prog[pc];
    std::ostringstream o;
    int constr = -1;
    switch (in.op) {
      case OP_CONSTRB: o << "rr = qadd(rr, qmulb(ldq(coeff + " << JIT_COEFF_WORDS * k << "), b[" << in.a << "]));"; coeff_of[pc] = k; constr = (int)k++; break;
      case OP_CONSTRE: o << "rr = qmac_tab(rr, e[" << in.a << "], coeff + " << JIT_COEFF_WORDS * k << ");"; coeff_of[pc] = k; constr = (int)k++; break;
      default: emit_op(o, in, ld); break;
    }
    if (constr >= 0 && !keep[constr]) continue;
    pl.at[pc].push_back(Stmt{o.str(), instr_regs(in), constr >= 0, constr});
  }

  struct Term { bool neg; u32 param; int bdef; };   // -/+ params[param] * (bdef < 0 ? 1 : the base value prog[bdef] wrote)
  std::function<bool(int, bool, std::vector<Term>&)> linear = [&](int q, bool neg, std::vector<Term>& t) {
    if (q < 0) return false;
    switch (prog[q].op) {
      case OP_PARAME: t.push_back(Term{neg, prog[q].a, -1}); return true;
      case OP_MULEB:
        if (def_a[q] < 0 || prog[def_a[q]].op != OP_PARAME || def_b[q] < 0) return false;
        t.push_back(Term{neg, prog[def_a[q]].a, def_b[q]});
        return true;
      case OP_ADDE: return linear(def_a[q], neg, t) && linear(def_b[q], neg, t);
      case OP_SUBE: return linear(def_a[q], neg, t) && linear(def_b[q], !neg, t);
      default: return false;
    }
  };
  std::map<std::pair<u32, u32>, u32> slot_of;
  std::map<int, u32> copy_of;   // base value (defining position) -> the register that keeps it for a later fold
  for (int pc = 0; pc < n; ++pc) {
    if (prog[pc].op != OP_CONSTRE || !keep[coeff_of[pc]]) continue;
    const int s = def_a[pc];
    if (s < 0 || prog[s].op != OP_SUBE || uses[s] != 1) continue;
    const int m = def_a[s], nu = def_b[s];
    if (m < 0 || prog[m].op != OP_MULE || uses[m] != 1 || nu < 0 || prog[nu].op != OP_BTOE || def_a[nu] < 0) continue;
    std::vector<Term> t;
    u32 diff = prog[m].a;
    if (!linear(def_b[m], false, t)) {
      t.clear();
      diff = prog[m].b;
      if (!linear(def_a[m], false, t)) continue;
    }
    const u32 kc = coeff_of[pc];
    // at the MULE: rr += diff * (coeff * den), coeff * den summed from the folded products and the base values the den read
    std::ostringstream o;
    Regs r;
    r.re.push_back(diff);
    o << "{ Q cd;";
    for (size_t i = 0; i < t.size(); ++i) {
      auto key = std::make_pair(kc, t[i].param);
      auto it = slot_of.find(key);
      if (it == slot_of.end()) { it = slot_of.emplace(key, (u32)pl.slots.size()).first; pl.slots.push_back(key); }
      std::string v = "ldf(" + std::to_string(it->second) + ")";
      if (t[i].bdef >= 0) {
        const int d = t[i].bdef;
        u32 reg = prog[d].dst;
        if (next_def[d] < m) {   // the register is rewritten before the MULE: keep the value in a register of its own
          auto ci = copy_of.find(d);
          if (ci == copy_of.end()) {
            ci = copy_of.emplace(d, pl.nb++).first;
            Regs cr; cr.rb.push_back(reg); cr.wb = (int)ci->second;
            pl.at[d].push_back(Stmt{"b[" + std::to_string(ci->second) + "] = b[" + std::to_string(reg) + "];", cr, false});
          }
          reg = ci->second;
        }
        v = "qmulb(" + v + ", b[" + std::to_string(reg) + "])";
        r.rb.push_back(reg);
      }
      if (i == 0) o << " cd = " << (t[i].neg ? "qneg(" + v + ")" : v) << ";";
      else o << " cd = " << (t[i].neg ? "qsub" : "qadd") << "(cd, " << v << ");";
    }
    o << " rr = qmacq(rr, e[" << diff << "], cd); }";
    pl.at[m] = {Stmt{o.str(), r, true, (int)kc}};
    // at the SUBE: rr -= coeff * num (a constant 0 or 1 needs no product)
    const AirInstr& bv = prog[def_a[nu]];
    pl.at[s].clear();
    std::ostringstream q;
    Regs qr;
    const std::string cf = "ldq(coeff + " + std::to_string(JIT_COEFF_WORDS * kc) + ")";
    if (bv.op == OP_CONSTB && bv.a == 1) q << "rr = qsub(rr, " << cf << ");";
    else if (bv.op == OP_CONSTB) q << "rr = qsub(rr, qmulb(" << cf << ", " << bv.a << "u));";
    else { q << "rr = qsub(rr, qmulb(" << cf << ", e[" << prog[s].b << "].c0));"; qr.re.push_back(prog[s].b); }
    if (!(bv.op == OP_CONSTB && bv.a == 0)) pl.at[s].push_back(Stmt{q.str(), qr, true, (int)kc});
    pl.at[pc].clear();
  }
  // dead code: a statement stays if it adds to rr or a later statement reads what it writes
  std::vector<char> need_b(pl.nb + 1, 0), need_e(ne + 1, 0);
  for (int pc = n; pc-- > 0;) {
    for (size_t i = pl.at[pc].size(); i-- > 0;) {
      Stmt& st = pl.at[pc][i];
      if (!st.effect && !(st.r.wb >= 0 && need_b[st.r.wb]) && !(st.r.we >= 0 && need_e[st.r.we])) { st = Stmt(); continue; }
      if (st.r.wb >= 0) need_b[st.r.wb] = 0;
      if (st.r.we >= 0) need_e[st.r.we] = 0;
      for (u32 x : st.r.rb) need_b[x] = 1;
      for (u32 x : st.r.re) need_e[x] = 1;
    }
  }
  return pl;
}

// d2 = false: every constraint, summed into a0..a3; when h0..h3 are given, the constraints of degree above AIR_LOW_DEGREE are also
//             summed on their own into h0..h3 (for the committed LDE domain D1 of a Q_HALF component: prove.cu, component_quotients).
// d2 = true:  the constraints of degree above AIR_LOW_DEGREE only, into a0..a3 (for the half coset D2); the masks no such constraint
//             reads are never loaded and may be null.
std::string gen_source(const AirComponent& c, bool d2) {
  std::ostringstream o;
  if (d2) o << "// constraint quotients on D2: the constraints of degree > " << AIR_LOW_DEGREE << " only\n";
  o << kPrelude;
  const u32 DL = c.log_size;  // EL (the canonic domain the rows belong to) is a kernel argument: whole domains and half domains share the kernel
  // offset_bit_reversed_circle_domain_index with the domain sizes baked in
  o << "__device__ __forceinline__ u32 offrow(u32 i, int off, u32 EL) { const u32 DL = " << DL << ";\n"
    << "  u32 prev = __brev(i) >> (32 - EL); u32 half = 1u << (EL - 1); long long step = (long long)off * (1ll << (EL - DL - 1)); long long v;\n"
    << "  if (prev < half) { v = ((long long)prev + step) % (long long)half; if (v < 0) v += half; }\n"
    << "  else { v = ((long long)prev - step) % (long long)half; if (v < 0) v += half; v += half; }\n"
    << "  return __brev((u32)v) >> (32 - EL); }\n";
  const u32 ne = c.n_ext_regs ? c.n_ext_regs : 1;
  auto ld = [&](u32 m) {
    std::ostringstream s;
    if (c.masks[m].off == 0) s << "__ldg(ccols[" << m << "] + row)";
    else s << "__ldg(ccols[" << m << "] + offrow(row, " << c.masks[m].off << ", EL))";
    return s.str();
  };
  const std::vector<char> high = high_constraints(c);
  ConstraintPlan pl = plan_constraints(c, ld, c.n_base_regs ? c.n_base_regs : 1, ne, d2 ? high : std::vector<char>(c.n_constraints, 1));
  // rh: the high constraints' part of rr, taken as the change of rr across their statements (no products of its own)
  const bool track_high = !d2 && count_high(high) > 0;
  if (track_high)
    for (auto& at : pl.at)
      for (Stmt& st : at)
        if (st.effect && high[st.constr]) st.code = "{ const Q r0 = rr; " + st.code + " rh = qadd(rh, qsub(rr, r0)); }";
  ChunkedKernel kk;
  kk.ch = 250; kk.nb = pl.nb; kk.ne = ne;
  kk.state = track_high ? " Q rr; Q rh;" : " Q rr;";
  if (!pl.slots.empty()) {
    // the folded products coeff_k * params[p]: (k, p) per slot, and their values, computed by each CTA before the first chunk
    std::ostringstream d;
    d << "#ifndef __CUDACC__\n#define __shared__\n#endif\n#define NB_NFOLD " << pl.slots.size() << "\n__constant__ const uint2 nbfold_src[NB_NFOLD] = {";
    for (size_t i = 0; i < pl.slots.size(); ++i) d << (i ? ", " : "") << "{" << pl.slots[i].first << "u, " << pl.slots[i].second << "u}";
    d << "};\n__shared__ uint4 nbfold[NB_NFOLD];\n"
      << "__device__ __forceinline__ Q ldf(u32 i) { const uint4 v = nbfold[i]; return Q{v.x, v.y, v.z, v.w}; }\n"
      << "__device__ __forceinline__ Q qmacq(Q acc, Q x, Q y) {\n"
      << "  u32 gp = add(add(y.c3, y.c3), y.c2), g = sub(add(y.c2, y.c2), y.c3);\n"
      << "  return qmac(acc, x, y.c0, y.c1, y.c2, y.c3, P31 - y.c1, P31 - y.c3, g, gp, P31 - gp);\n}\n";
    kk.decls = d.str();
  }
  kk.params = "const u32* const* __restrict__ cols, const u32* __restrict__ params, const u32* __restrict__ coeff, u32 row, u32 EL";
  kk.enter = track_high ? " Q rr = s.rr; Q rh = s.rh;" : " Q rr = s.rr;";
  kk.leave = track_high ? "  s.rr = rr; s.rh = rh;\n" : "  s.rr = rr;\n";
  kk.sig = "const u32* const* __restrict__ cols, const u32* __restrict__ params, const u32* __restrict__ coeff,\n"
          "    const u32* __restrict__ dinv, u32* __restrict__ a0, u32* __restrict__ a1, u32* __restrict__ a2, u32* __restrict__ a3, u32 EL, u32 row0,\n"
          "    u32* __restrict__ h0 = nullptr, u32* __restrict__ h1 = nullptr, u32* __restrict__ h2 = nullptr, u32* __restrict__ h3 = nullptr";
  kk.prologue = "  const u32 row = row0 + blockIdx.x * blockDim.x + threadIdx.x;   // row0: a rank of a multi-GPU proof evaluates its slice of the domain's rows\n";
  kk.init = track_high ? "  s.rr = Q{0u, 0u, 0u, 0u};\n  s.rh = Q{0u, 0u, 0u, 0u};\n" : "  s.rr = Q{0u, 0u, 0u, 0u};\n";
  if (!pl.slots.empty())
    kk.init += "  for (u32 i = threadIdx.x; i < NB_NFOLD; i += blockDim.x) {\n"
              "    const Q f = qmac_tab(Q{0u, 0u, 0u, 0u}, ldq(params + 4 * nbfold_src[i].y), coeff + " + std::to_string(JIT_COEFF_WORDS) + " * nbfold_src[i].x);\n"
              "    nbfold[i] = uint4{f.c0, f.c1, f.c2, f.c3};\n  }\n  __syncthreads();\n";
  kk.args = "cols, params, coeff, row, EL";
  std::ostringstream e;
  e << "  const u32 di = __ldg(dinv + (row >> " << DL << "));\n"
    << "  a0[row] = add(a0[row], mul(s.rr.c0, di)); a1[row] = add(a1[row], mul(s.rr.c1, di));\n"
    << "  a2[row] = add(a2[row], mul(s.rr.c2, di)); a3[row] = add(a3[row], mul(s.rr.c3, di));\n";
  if (track_high)
    e << "  if (h0) {\n"
      << "    h0[row] = add(h0[row], mul(s.rh.c0, di)); h1[row] = add(h1[row], mul(s.rh.c1, di));\n"
      << "    h2[row] = add(h2[row], mul(s.rh.c2, di)); h3[row] = add(h3[row], mul(s.rh.c3, di));\n  }\n";
  kk.epilogue = e.str();
  emit_chunked(o, c, pl.at, kk);
  return o.str();
}

// LogupTraceGenerator for one component (interp.cu interp_kernel<.., LOGUP> is the bytecode version): run the logup program, combine the
// fractions of each batch (write_frac), add to the running row sum and store the 4 coordinate columns of the batch (finalize_col).
// The prefix sum over rows of the last column stays in logup_generate.
std::string gen_logup_source(const AirComponent& c) {
  std::ostringstream o;
  o << kPrelude;
  auto ld = [&](u32 m) {
    std::ostringstream s;
    // next-row masks and interaction-trace masks are not inputs of the logup program (they read as zero, as in the interpreter)
    if (m < c.masks.size() && c.masks[m].off == 0 && c.masks[m].tree != 2) s << "__ldg(ccols[" << m << "] + row)";
    else s << "0u";
    return s.str();
  };
  // The QM31 inverse (one per batch of fractions; 38 M31 products for x^(P-2) alone) is batched over G consecutive batches of the same
  // row: prefix products, ONE inverse, back-substitution (3 products per extra batch).  The inverse is unique, so the values are the
  // interpreter's.  `pending` batches wait in pfn/pfd until the group is full; the running row sum is then advanced batch by batch.
  const int G = 4;
  u32 k = 0; bool have = false; u32 cur_batch = 0;
  std::vector<u32> pending;   // batch ids waiting in slots 0..pending.size()-1 (tracked at code-generation time)
  auto flush = [&](std::ostringstream& o2) {
    const int n = (int)pending.size();
    if (n == 0) return;
    o2 << "  {\n";
    for (int g = 1; g < n; ++g) o2 << "    Q pp" << g << " = qmul(" << (g == 1 ? std::string("pfd0") : "pp" + std::to_string(g - 1)) << ", pfd" << g << ");\n";
    o2 << "    Q iv = qinv(" << (n == 1 ? std::string("pfd0") : "pp" + std::to_string(n - 1)) << ");\n";
    for (int g = n - 1; g >= 1; --g)
      o2 << "    { Q t = qmul(iv, " << (g == 1 ? std::string("pfd0") : "pp" + std::to_string(g - 1)) << "); iv = qmul(iv, pfd" << g << "); pfd" << g << " = t; }\n";
    o2 << "    pfd0 = iv;\n";
    for (int g = 0; g < n; ++g) {
      o2 << "    run = qadd(run, qmul(pfn" << g << ", pfd" << g << "));\n";
      for (int cc = 0; cc < 4; ++cc) o2 << "    out[(" << (4 * (size_t)pending[g] + cc) << "ull << LS) + row] = run.c" << cc << ";\n";
    }
    o2 << "  }\n";
    pending.clear();
  };
  auto finalize = [&](std::ostringstream& o2) {   // the current batch's combined fraction fn / fd is complete
    o2 << "  pfn" << pending.size() << " = fn; pfd" << pending.size() << " = fd;\n";
    pending.push_back(cur_batch);
    if ((int)pending.size() == G) flush(o2);
  };
  std::vector<std::vector<Stmt>> at(c.logup_prog.size());
  for (size_t pc = 0; pc < c.logup_prog.size(); ++pc) {
    const AirInstr& in = c.logup_prog[pc];
    if (in.op != OP_FRAC) { at[pc].push_back(op_stmt(in, ld)); continue; }
    std::ostringstream s;   // whole lines, the previous batch's completion first (the emitter writes the first indent and the last newline)
    u32 bt = c.batching[k];
    if (have && bt != cur_batch) { finalize(s); have = false; }
    if (!have) s << "  fn = e[" << in.a << "]; fd = e[" << in.b << "];";                      // first fraction of the batch: 0/1 + n/d
    else s << "  fn = qadd(qmul(fn, e[" << in.b << "]), qmul(e[" << in.a << "], fd)); fd = qmul(fd, e[" << in.b << "]);";
    cur_batch = bt; have = true; ++k;
    at[pc].push_back(Stmt{s.str().substr(2), instr_regs(in)});
  }
  std::ostringstream last;
  if (have) finalize(last);
  flush(last);
  ChunkedKernel kk;
  kk.ch = 150; kk.nb = c.lg_base_regs ? c.lg_base_regs : 1; kk.ne = c.lg_ext_regs ? c.lg_ext_regs : 1;
  kk.state = " Q fn, fd, run;";
  kk.decls = "struct Pend { Q n[" + std::to_string(G) + "], d[" + std::to_string(G) + "]; };\n";
  kk.params = "Pend& pe, const u32* const* __restrict__ cols, const u32* __restrict__ params, u32* __restrict__ out, u32 row, u32 LS";
  std::ostringstream enter, leave;
  enter << " Q fn = s.fn, fd = s.fd, run = s.run;";
  leave << "  s.fn = fn; s.fd = fd; s.run = run;\n";
  for (int g = 0; g < G; ++g) {
    enter << "\n  Q pfn" << g << " = pe.n[" << g << "], pfd" << g << " = pe.d[" << g << "];";
    leave << "  pe.n[" << g << "] = pfn" << g << "; pe.d[" << g << "] = pfd" << g << ";\n";
  }
  kk.enter = enter.str();
  kk.leave = leave.str();
  kk.last = last.str();
  kk.sig = "const u32* const* __restrict__ cols, const u32* __restrict__ params, u32* __restrict__ out, u32 LS";
  kk.prologue = "  const u32 row = blockIdx.x * blockDim.x + threadIdx.x;\n";
  kk.init = "  s.fn = Q{0u, 0u, 0u, 0u}; s.fd = Q{1u, 0u, 0u, 0u}; s.run = Q{0u, 0u, 0u, 0u};\n"
            "  Pend pe; for (int i = 0; i < 4; ++i) { pe.n[i] = Q{0u, 0u, 0u, 0u}; pe.d[i] = Q{1u, 0u, 0u, 0u}; }\n";
  kk.args = "pe, cols, params, out, row, LS";
  emit_chunked(o, c, at, kk);
  return o.str();
}

// Columns are in bit-reversed circle-domain order.  Position i holds circle-domain index brev(i), which is coset (trace) row 2j for circle
// index j < N/2 and 2N - 2j - 1 above (the inverse of coset_index_to_circle_domain_index).
static std::string coset_rows(const AirComponent& c) {
  return "#define NB_DL " + std::to_string(c.log_size) + "u\n#define NB_N (1u << NB_DL)\n"
         "__device__ __forceinline__ u32 pos_to_row(u32 i) { const u32 j = __brev(i) >> (32 - NB_DL); return j < NB_N / 2 ? 2 * j : 2 * NB_N - 2 * j - 1; }\n";
}

// The constraint check (the GPU counterpart of stwo's assert_constraints_on_polys): the plain constraint program on the trace domain
// CanonicCoset(log_size) itself, one thread per row, with no random coefficients and no vanishing division — every CONSTRB / CONSTRE sink
// tests its own value for zero.  A warp counts its failing rows with one ballot and finds the first one (in coset order) with one
// min-reduction, so a constraint costs one atomicAdd and one atomicMin per warp that sees a failure, none per row.
std::string gen_check_source(const AirComponent& c) {
  std::ostringstream o;
  o << "// constraint check on the trace domain: each constraint tested for zero on every row\n";
  o << kPrelude;
  // a mask at offset `off` reads coset row (r + off) mod N, wrapping at both ends as assert_constraints_on_polys does
  o << coset_rows(c)
    << "__device__ __forceinline__ u32 row_to_pos(u32 r) { const u32 j = (r & 1) ? NB_N - (r + 1) / 2 : r / 2; return __brev(j) >> (32 - NB_DL); }\n"
    << "__device__ __forceinline__ u32 offrow(u32 r, int off) { return row_to_pos((r + (u32)off) & (NB_N - 1)); }   // N divides 2^32\n"
    // every prelude operation returns a canonical residue; P is also taken as zero for a constraint that is a raw (unreduced) cell
    << "__device__ __forceinline__ bool nzb(u32 v) { return v != 0u && v != P31; }\n"
    << "__device__ __forceinline__ bool nze(Q v) { return nzb(v.c0) || nzb(v.c1) || nzb(v.c2) || nzb(v.c3); }\n"
    // one warp: count the failing rows, the first of them in coset order; rows past the domain (live = false) never fail
    << "__device__ __forceinline__ void check(u32 k, bool bad, u32 r, u32* __restrict__ nfail, u32* __restrict__ first) {\n"
    << "  const unsigned am = __activemask();\n"
    << "  const unsigned m = __ballot_sync(am, bad);\n"
    << "  if (m) {\n"
    << "    const u32 lo = __reduce_min_sync(am, bad ? r : 0xffffffffu);\n"
    << "    if ((threadIdx.x & 31u) == (u32)(__ffs(am) - 1)) { atomicAdd(nfail + k, (u32)__popc(m)); atomicMin(first + k, lo); }\n"
    << "  }\n}\n";
  auto ld = [&](u32 m) {
    std::ostringstream s;
    if (c.masks[m].off == 0) s << "__ldg(ccols[" << m << "] + pos)";
    else s << "__ldg(ccols[" << m << "] + offrow(r, " << c.masks[m].off << "))";
    return s.str();
  };
  std::vector<std::vector<Stmt>> at(c.prog.size());
  u32 k = 0;
  for (size_t pc = 0; pc < c.prog.size(); ++pc) {
    const AirInstr& in = c.prog[pc];
    Stmt st = op_stmt(in, ld);
    if (in.op == OP_CONSTRB) st.code = "check(" + std::to_string(k++) + "u, live && nzb(b[" + std::to_string(in.a) + "]), r, nfail, first);";
    if (in.op == OP_CONSTRE) st.code = "check(" + std::to_string(k++) + "u, live && nze(e[" + std::to_string(in.a) + "]), r, nfail, first);";
    at[pc].push_back(st);
  }
  ChunkedKernel kk;
  kk.ch = 250; kk.nb = c.n_base_regs ? c.n_base_regs : 1; kk.ne = c.n_ext_regs ? c.n_ext_regs : 1;
  kk.params = "const u32* __restrict__ params, u32* __restrict__ nfail, u32* __restrict__ first, u32 pos, u32 r, bool live";
  // nfail[k] / first[k]: rows on which constraint k is non-zero and the first of them in coset order (0xffffffff: none)
  kk.sig = "const u32* __restrict__ params, u32* __restrict__ nfail, u32* __restrict__ first";
  kk.prologue = "  const u32 gid = blockIdx.x * blockDim.x + threadIdx.x;\n"
                "  const bool live = gid < NB_N;\n"
                "  const u32 pos = live ? gid : 0u;   // a thread past the domain runs row 0 with its results masked: every thread reaches the barriers\n"
                "  const u32 r = pos_to_row(pos);\n";
  kk.args = "params, nfail, first, pos, r, live";
  emit_chunked(o, c, at, kk);
  return o.str();
}

// The table-multiplicity count (nb200_table_multiplicities) of one component, from its logup program as air_lookup_tables reads it.
// mode 0 (build): every table fraction's tuple on every row goes into an open-addressing hash keyed by (relation, length, values), the
//                 value being the row's bin: tbase[t] + the row's position (finalized order).  A tuple that is already there sets *err.
// mode 1 (probe): every lookup with a nonzero numerator finds its tuple's bin and adds the numerator to its u64 counter (in shared memory
//                 when the caller privatises the bins, nsh > 0).  A tuple without a bin is unmatched: um[0] counts them, um[1] keeps the
//                 smallest (component << 48 | fraction << 28 | row in coset order).
// Only base values are evaluated: each chunk recomputes, as SSA values, what its fractions read (mask loads and a few base operations), so
// no register crosses a chunk.  Hash and bins are laid out by the caller; the source depends on this component alone.
std::string gen_count_source(const AirComponent& c, const std::vector<AirFrac>& fr) {
  std::ostringstream o;
  o << "// table multiplicities: build (table tuples -> bins) and probe (lookups -> counters)\n";
  o << kPrelude;
  o << coset_rows(c)
    << "__device__ __forceinline__ u32 canon(u32 v) { return v >= P31 ? v - P31 : v; }\n"
    << "#define NB_EMPTY 0xffffffffu\n"
    << "__device__ __forceinline__ u32 khash(u32 rel, u32 len, const u32* v) {\n"
    << "  u64 h = ((u64)rel << 32 | len) * 0x9E3779B97F4A7C15ull;\n"
    << "  for (u32 i = 0; i < len; ++i) { h = (h ^ v[i]) * 0x9E3779B97F4A7C15ull; h ^= h >> 31; }\n"
    << "  return (u32)(h >> 32);\n}\n"
    // a key is rel, len, values: kw words per bin
    // the build reads keys other threads of the same launch wrote (through L2: __ldcg); the probe reads a finished table (__ldg)
    << "__device__ __forceinline__ bool ksame_cg(const u32* k, u32 rel, u32 len, const u32* v) {\n"
    << "  if (__ldcg(k) != rel || __ldcg(k + 1) != len) return false;\n"
    << "  for (u32 i = 0; i < len; ++i) if (__ldcg(k + 2 + i) != v[i]) return false;\n  return true;\n}\n"
    << "__device__ __forceinline__ bool ksame(const u32* k, u32 rel, u32 len, const u32* v) {\n"
    << "  if (__ldg(k) != rel || __ldg(k + 1) != len) return false;\n"
    << "  for (u32 i = 0; i < len; ++i) if (__ldg(k + 2 + i) != v[i]) return false;\n  return true;\n}\n"
    << "__device__ __noinline__ void nb_insert(u32 rel, u32 len, const u32* v, u32 bin, u32* slots, u32* keys, u32 kw, u32 mask, u32* err) {\n"
    << "  u32* k = keys + (u64)bin * kw;\n"
    << "  k[0] = rel; k[1] = len; for (u32 i = 0; i < len; ++i) k[2 + i] = v[i];\n"
    << "  __threadfence();   // the key is visible before the slot that names it\n"
    << "  for (u32 s = khash(rel, len, v) & mask;; s = (s + 1) & mask) {\n"
    << "    const u32 prev = atomicCAS(slots + s, NB_EMPTY, bin);\n"
    << "    if (prev == NB_EMPTY) return;\n"
    << "    if (ksame_cg(keys + (u64)prev * kw, rel, len, v)) { atomicOr(err, 1u); return; }   // the same tuple in two rows: ambiguous\n"
    << "  }\n}\n"
    << "__device__ __noinline__ void nb_lookup(u32 rel, u32 len, const u32* v, u32 num, u64 tag, u32 pos, const u32* __restrict__ slots,\n"
    << "    const u32* __restrict__ keys, u32 kw, u32 mask, u64* cnt, u32* sh, u64* um) {\n"
    << "  u32 bin = NB_EMPTY;\n"
    << "  for (u32 s = khash(rel, len, v) & mask;; s = (s + 1) & mask) {\n"
    << "    const u32 e = __ldg(slots + s);\n"
    << "    if (e == NB_EMPTY) break;\n"
    << "    if (ksame(keys + (u64)e * kw, rel, len, v)) { bin = e; break; }\n"
    << "  }\n"
    << "  const bool bad = bin == NB_EMPTY;\n"
    // a private bin is two u32 words (low, high) in shared memory: a 64-bit shared add would be a CAS loop, a 32-bit one is one ATOMS.ADD;
    // the thread whose add wraps the low word carries into the high one
    << "  if (!bad) {\n"
    << "    if (sh) { if (atomicAdd(sh + 2 * bin, num) + num < num) atomicAdd(sh + 2 * bin + 1, 1u); }\n"
    << "    else atomicAdd(cnt + bin, (u64)num);\n  }\n"
    // the check kernel's warp aggregation; the 64-bit minimum as two 32-bit ones (threads of other call sites may share the warp)
    << "  const unsigned am = __activemask();\n"
    << "  const unsigned m = __ballot_sync(am, bad);\n"
    << "  if (m) {\n"
    << "    const u64 key = bad ? (tag | pos_to_row(pos)) : ~0ull;\n"
    << "    const u32 hi = __reduce_min_sync(am, (u32)(key >> 32));\n"
    << "    const u32 lo = __reduce_min_sync(am, (u32)(key >> 32) == hi ? (u32)key : 0xffffffffu);\n"
    << "    if ((threadIdx.x & 31u) == (u32)(__ffs(am) - 1)) { atomicAdd(um, (u64)__popc(m)); atomicMin(um + 1, (u64)hi << 32 | lo); }\n"
    << "  }\n}\n";
  o << ccols_decl(c);
  const std::vector<AirInstr>& prog = c.logup_prog;
  std::vector<int> da, db;
  prog_defs(prog, c.lg_base_regs, c.lg_ext_regs, da, db);
  auto x = [](int q) { return "x" + std::to_string(q); };
  // the statements computing the base values at positions `roots`, with everything they read, in program order
  auto emit_values = [&](std::ostringstream& s, const std::vector<int>& roots) {
    std::vector<char> need(prog.size(), 0);
    std::vector<int> st(roots.begin(), roots.end());
    while (!st.empty()) {
      const int q = st.back(); st.pop_back();
      if (q < 0 || need[q]) continue;
      need[q] = 1;
      st.push_back(da[q]);
      if (prog[q].op != OP_NEGB) st.push_back(db[q]);
    }
    for (size_t q = 0; q < prog.size(); ++q) {
      if (!need[q]) continue;
      const AirInstr& in = prog[q];
      s << "  const u32 " << x((int)q) << " = ";
      switch (in.op) {
        case OP_LOADM: s << "__ldg(ccols[" << in.a << "] + pos)"; break;
        case OP_CONSTB: s << in.a << "u"; break;
        case OP_ADDB: s << "add(" << x(da[q]) << ", " << x(db[q]) << ")"; break;
        case OP_SUBB: s << "sub(" << x(da[q]) << ", " << x(db[q]) << ")"; break;
        case OP_MULB: s << "mul(" << x(da[q]) << ", " << x(db[q]) << ")"; break;
        case OP_NEGB: s << "neg(" << x(da[q]) << ")"; break;
        default: s << "0u"; break;   // unreachable: air_lookup_tables takes tuples and numerators from base values only
      }
      s << ";\n";
    }
  };
  auto tuple = [&](const AirFrac& f) {
    std::ostringstream s;
    s << "const u32 v[" << f.tuple.size() << "] = {";
    for (size_t i = 0; i < f.tuple.size(); ++i) s << (i ? ", " : "") << "canon(" << x(f.tuple[i]) << ")";
    s << "};";
    return s.str();
  };
  const size_t CH = 64;   // fractions per __noinline__ chunk: NVVM's time grows faster than the function
  std::vector<size_t> tables, lookups;
  for (size_t i = 0; i < fr.size(); ++i) {
    if (fr[i].kind == FRAC_TABLE) tables.push_back(i);
    if (fr[i].kind == FRAC_LOOKUP) lookups.push_back(i);
  }
  u32 t_index = 0;
  std::map<size_t, u32> t_of;
  for (size_t i : tables) t_of[i] = t_index++;
  const size_t nbc = (tables.size() + CH - 1) / CH, npc = (lookups.size() + CH - 1) / CH;
  for (size_t ci = 0; ci < nbc; ++ci) {
    o << "__device__ __noinline__ void bchunk" << ci << "(u32 pos, const u32* __restrict__ tbase, u32* slots, u32* keys, u32 kw, u32 mask, u32* err) {\n";
    std::vector<int> roots;
    for (size_t j = ci * CH; j < std::min(tables.size(), (ci + 1) * CH); ++j) for (int v : fr[tables[j]].tuple) roots.push_back(v);
    emit_values(o, roots);
    for (size_t j = ci * CH; j < std::min(tables.size(), (ci + 1) * CH); ++j) {
      const AirFrac& f = fr[tables[j]];
      o << "  { " << tuple(f) << " nb_insert(" << f.rel << "u, " << f.tuple.size() << "u, v, __ldg(tbase + " << t_of[tables[j]] << ") + pos, slots, keys, kw, mask, err); }\n";
    }
    o << "}\n";
  }
  for (size_t ci = 0; ci < npc; ++ci) {
    o << "__device__ __noinline__ void pchunk" << ci << "(u32 pos, u64 ctag, const u32* __restrict__ slots, const u32* __restrict__ keys, u32 kw, u32 mask, u64* cnt, u32* sh, u64* um) {\n";
    std::vector<int> roots;
    for (size_t j = ci * CH; j < std::min(lookups.size(), (ci + 1) * CH); ++j) {
      for (int v : fr[lookups[j]].tuple) roots.push_back(v);
      roots.push_back(fr[lookups[j]].num);
    }
    emit_values(o, roots);
    for (size_t j = ci * CH; j < std::min(lookups.size(), (ci + 1) * CH); ++j) {
      const AirFrac& f = fr[lookups[j]];
      o << "  { const u32 n = canon(" << x(f.num) << "); if (n) { " << tuple(f) << " nb_lookup(" << f.rel << "u, " << f.tuple.size() << "u, v, n, ctag | "
        << lookups[j] << "ull << 28, pos, slots, keys, kw, mask, cnt, sh, um); } }\n";
    }
    o << "}\n";
  }
  // one launch per mode; rows by a grid-stride loop (the probe's private bins are zeroed and flushed once per CTA)
  o << "extern __shared__ u32 nbsh[];   // 2 words per private bin\n"
    << "extern \"C\" __global__ void __launch_bounds__(256) nbjit(u32 mode, u32 comp, const u32* __restrict__ tbase, u32* slots, u32* keys, u32 kw, u32 mask,\n"
    << "    u64* cnt, u32 nsh, u64* um, u32* err) {\n"
    << "  const u32 stride = gridDim.x * blockDim.x;\n"
    << "  if (mode == 0) {\n"
    << "    for (u32 pos = blockIdx.x * blockDim.x + threadIdx.x; pos < NB_N; pos += stride) {\n";
  for (size_t ci = 0; ci < nbc; ++ci) o << "      bchunk" << ci << "(pos, tbase, slots, keys, kw, mask, err);\n";
  o << "    }\n    return;\n  }\n"
    << "  u32* sh = nsh ? nbsh : nullptr;\n"
    << "  for (u32 i = threadIdx.x; i < 2 * nsh; i += blockDim.x) nbsh[i] = 0u;\n"
    << "  if (nsh) __syncthreads();\n"
    << "  const u64 ctag = (u64)comp << 48;\n"
    << "  for (u32 pos = blockIdx.x * blockDim.x + threadIdx.x; pos < NB_N; pos += stride) {\n";
  for (size_t ci = 0; ci < npc; ++ci) o << "    pchunk" << ci << "(pos, ctag, slots, keys, kw, mask, cnt, sh, um);\n";
  o << "  }\n"
    << "  if (nsh) {\n    __syncthreads();\n"
    << "    for (u32 i = threadIdx.x; i < nsh; i += blockDim.x) {\n"
    << "      const u64 v = (u64)nbsh[2 * i + 1] << 32 | nbsh[2 * i];\n"
    << "      if (v) atomicAdd(cnt + i, v);\n    }\n  }\n}\n";
  return o.str();
}
}  // namespace

bool jit_specialised(JitKind kind, const AirComponent& c, const std::vector<AirFrac>& fr) {
  switch (kind) {
    case JIT_CONSTRAINTS: return c.prog.size() >= JIT_MIN_INSTR;
    case JIT_LOGUP: return c.logup_prog.size() >= JIT_MIN_INSTR && c.n_logup_cols() > 0;
    case JIT_D2: return c.prog.size() >= JIT_MIN_INSTR && count_high(high_constraints(c)) > 0;
    case JIT_CHECK: return c.n_constraints > 0;
    case JIT_COUNT: return std::any_of(fr.begin(), fr.end(), [](const AirFrac& f) { return f.kind == FRAC_TABLE || f.kind == FRAC_LOOKUP; });
    default: return false;
  }
}

std::string jit_kernel_source(JitKind kind, const AirComponent& c, const std::vector<AirFrac>& fr) {
  switch (kind) {
    case JIT_LOGUP: return gen_logup_source(c);
    case JIT_CHECK: return gen_check_source(c);
    case JIT_COUNT: return gen_count_source(c, fr);
    default: return gen_source(c, kind == JIT_D2);
  }
}

bool jit_enabled() {
  const char* e = getenv("NB200_JIT");
  return !(e && e[0] == '0');   // libnvrtc itself is only opened when a kernel is missing from the cubin cache
}

void jit_release(JitKernel& jk) {
  if (jk.lib) cudaLibraryUnload((cudaLibrary_t)jk.lib);
  jk = JitKernel();
}

// ---- cubin cache: <directory of this library>/jit_cache/<key>.cubin (or $NB200_JIT_CACHE).  `python -m nexus_zkvm_b200.build`
// fills it for the shipped machines with nvcc, so a fresh box neither loads libnvrtc nor compiles; kernels compiled at run time are
// added when the directory is writable.  The key covers the generated source and the target; the D2 variant of a constraint kernel
// and the constraint check start with a line of their own, so they never share a key with the D1 variant.
uint64_t jit_source_key(const std::string& src) {
  uint64_t h = 1469598103934665603ull;
  auto mix = [&](const char* p, size_t n) { for (size_t i = 0; i < n; ++i) { h ^= (unsigned char)p[i]; h *= 1099511628211ull; } };
  mix(src.data(), src.size());
  const char* tgt = "|sm_90a|nb200-jit-4";
  mix(tgt, strlen(tgt));
  return h;
}
static std::string jit_cache_dir() {
  if (const char* e = getenv("NB200_JIT_CACHE")) return e;
  Dl_info info;
  if (dladdr((const void*)&jit_source_key, &info) && info.dli_fname) {
    std::string p = info.dli_fname;
    size_t k = p.rfind('/');
    return (k == std::string::npos ? std::string(".") : p.substr(0, k)) + "/jit_cache";
  }
  return "";
}
static std::string jit_cache_path(const std::string& src) {
  std::string d = jit_cache_dir();
  if (d.empty()) return "";
  char name[32]; snprintf(name, sizeof name, "/%016llx.cubin", (unsigned long long)jit_source_key(src));
  return d + name;
}
static bool read_file(const std::string& path, std::vector<char>& out) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  fseek(f, 0, SEEK_END); long n = ftell(f); fseek(f, 0, SEEK_SET);
  bool ok = n > 0;
  if (ok) { out.resize((size_t)n); ok = fread(out.data(), 1, (size_t)n, f) == (size_t)n; }
  fclose(f);
  return ok;
}
static void write_file_atomic(const std::string& path, const std::vector<char>& data) {
  std::string tmp = path + ".tmp" + std::to_string((long)getpid());
  FILE* f = fopen(tmp.c_str(), "wb");
  if (!f) return;
  bool ok = fwrite(data.data(), 1, data.size(), f) == data.size();
  ok = (fclose(f) == 0) && ok;
  if (!ok || rename(tmp.c_str(), path.c_str()) != 0) remove(tmp.c_str());
}
static nb200_status jit_load_cubin(nb200_ctx* ctx, const AirComponent& c, const std::vector<char>& cubin, JitKernel* out) {
  cudaLibrary_t lib;
  cudaError_t e = cudaLibraryLoadData(&lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0);
  if (e != cudaSuccess) return set_err(ctx, NB200_ERR_CUDA, std::string("jit: cudaLibraryLoadData: ") + cudaGetErrorString(e));
  cudaKernel_t k;
  e = cudaLibraryGetKernel(&k, lib, "nbjit");
  if (e != cudaSuccess) { cudaLibraryUnload(lib); return set_err(ctx, NB200_ERR_CUDA, std::string("jit: cudaLibraryGetKernel: ") + cudaGetErrorString(e)); }
  out->lib = (void*)lib; out->kernel = (void*)k; out->log_size = c.log_size; out->eval_log = c.eval_log();
  return NB200_OK;
}

nb200_status jit_compile(nb200_ctx* ctx, JitKind kind, const AirComponent& c, const std::vector<AirFrac>& fr, JitKernel* out) {
  out->lib = nullptr; out->kernel = nullptr; out->tried = true;
  const std::string src = jit_kernel_source(kind, c, fr);
  const std::string cache = jit_cache_path(src);
  if (!cache.empty()) {
    std::vector<char> cubin;
    if (read_file(cache, cubin) && jit_load_cubin(ctx, c, cubin, out) == NB200_OK) return NB200_OK;
    cudaGetLastError();  // a stale or foreign file: fall through to the compiler
  }
  Nvrtc& n = nvrtc();
  if (!n.ok) return set_err(ctx, NB200_ERR_STATE, "jit: libnvrtc not available");
  nvrtcProgram prog;
  if (n.CreateProgram(&prog, src.c_str(), "nb200_air.cu", 0, nullptr, nullptr) != NVRTC_SUCCESS) return set_err(ctx, NB200_ERR_STATE, "jit: nvrtcCreateProgram failed");
  const char* opts[] = {"--gpu-architecture=sm_90a", "--std=c++17", "-lineinfo"};
  nvrtcResult r = n.CompileProgram(prog, 3, opts);
  if (r != NVRTC_SUCCESS) {
    size_t ls = 0; n.GetProgramLogSize(prog, &ls);
    std::string log(ls, '\0'); if (ls) n.GetProgramLog(prog, &log[0]);
    n.DestroyProgram(&prog);
    return set_err(ctx, NB200_ERR_STATE, "jit: compile failed: " + log.substr(0, 2000));
  }
  size_t cs = 0; n.GetCUBINSize(prog, &cs);
  std::vector<char> cubin(cs);
  n.GetCUBIN(prog, cubin.data());
  n.DestroyProgram(&prog);
  if (!cache.empty()) write_file_atomic(cache, cubin);
  return jit_load_cubin(ctx, c, cubin, out);
}

// per constraint: y0 y1 y2 y3 | P-y1 P-y3 2y2-y3 y2+2y3 | P-(y2+2y3) 0 0 0   (the multipliers of qmac in the generated code)
void jit_coeff_table(const std::vector<qm31>& coeffs, std::vector<u32>& out) {
  out.assign(coeffs.size() * JIT_COEFF_WORDS, 0u);
  for (size_t k = 0; k < coeffs.size(); ++k) {
    const u32* y = coeffs[k].c;
    u32* t = &out[k * JIT_COEFF_WORDS];
    u32 gp = m31_add(m31_add(y[3], y[3]), y[2]), g = m31_sub(m31_add(y[2], y[2]), y[3]);
    t[0] = y[0]; t[1] = y[1]; t[2] = y[2]; t[3] = y[3];
    t[4] = P31 - y[1]; t[5] = P31 - y[3]; t[6] = g; t[7] = gp; t[8] = P31 - gp;
  }
}

// the kernel's column pointers (a host array, one per mask) into the module's __constant__ table, then the kernel, both in stream order
nb200_status jit_launch(nb200_ctx* ctx, const JitKernel& jk, const u32* const* cols, size_t n_cols, dim3 grid, dim3 block, void** args, size_t smem) {
  void* dptr = nullptr; size_t bytes = 0;
  cudaError_t e = cudaLibraryGetGlobal(&dptr, &bytes, (cudaLibrary_t)jk.lib, "ccols");
  if (e != cudaSuccess) return set_err(ctx, NB200_ERR_CUDA, std::string("jit: cudaLibraryGetGlobal(ccols): ") + cudaGetErrorString(e));
  if (n_cols) {
    e = cudaMemcpyAsync(dptr, cols, n_cols * sizeof(u32*), cudaMemcpyHostToDevice, ctx->stream);
    if (e != cudaSuccess) return set_err(ctx, NB200_ERR_CUDA, std::string("jit: ccols copy: ") + cudaGetErrorString(e));
  }
  e = cudaLaunchKernel((const void*)jk.kernel, grid, block, args, smem, ctx->stream);
  ctx->launches += 1;
  if (e != cudaSuccess) return set_err(ctx, NB200_ERR_CUDA, std::string("jit launch: ") + cudaGetErrorString(e));
  return NB200_OK;
}

}  // namespace nb
