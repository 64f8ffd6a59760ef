// NVRTC specialisation of AIR constraint programs (see jit.cu).
#pragma once
#include "common.cuh"
#include "air.h"
#include <string>
#include <vector>

namespace nb {

static const u32 JIT_BLOCK = 1024;       // the generated kernels are compiled for up to this many threads per CTA (<= 64 registers)
// threads per CTA at launch: two CTAs per SM, which sit in different phases of the program and share the pipes.  On H100, 256 / 512 / 1024
// gave the same whole-proof time within noise (profiles/README.md)
static const u32 JIT_LAUNCH_BLOCK = 512;
static const u32 JIT_MIN_INSTR = 64;      // shorter programs stay on the bytecode interpreter
static const u32 JIT_COEFF_WORDS = 12;   // words per constraint in the coefficient table the generated kernel reads

// The kernels generated for a component; 0-3 are the `which` of nb200_air_kernel_source.
//   JIT_CONSTRAINTS: every constraint (with the high-degree part on the side, jit.cu gen_source), on the LDE domain or a half of it;
//   JIT_LOGUP: the interaction trace; JIT_D2: the constraints of degree above AIR_LOW_DEGREE only, for the half coset D2;
//   JIT_CHECK: per constraint, the rows of the trace domain where it is non-zero and the first of them in coset order;
//   JIT_COUNT: the table-multiplicity count (mode 0 builds the hash of the component's table tuples, mode 1 counts its lookups).
enum JitKind { JIT_CONSTRAINTS, JIT_LOGUP, JIT_D2, JIT_CHECK, JIT_COUNT, JIT_KINDS };

struct JitKernel {
  void* lib = nullptr;     // cudaLibrary_t
  void* kernel = nullptr;  // cudaKernel_t
  u32 log_size = 0, eval_log = 0;
  bool tried = false;      // compilation attempted (failed attempts fall back to the interpreter)
  std::string err;         // why the attempt failed (empty: it did not, or was not made)
};

// the specialised kernel jk runs constraint_eval on 2^rows_log rows (else the bytecode interpreter does)
inline bool jit_usable(const JitKernel* jk, const AirComponent& c, u32 rows_log) {
  return jk && jk->kernel && jk->log_size == c.log_size && ((size_t)1 << rows_log) >= JIT_BLOCK;
}
bool jit_enabled();
// the library generates this kind for c: a constraint or LogUp program long enough to leave the interpreter, or a check or count with
// something to evaluate.  fr (air_lookup_tables) is read by JIT_COUNT only.
bool jit_specialised(JitKind kind, const AirComponent& c, const std::vector<AirFrac>& fr);
std::string jit_kernel_source(JitKind kind, const AirComponent& c, const std::vector<AirFrac>& fr);   // the CUDA C of the kernel
uint64_t jit_source_key(const std::string& src);   // name of the kernel's file in the cubin cache
nb200_status jit_compile(nb200_ctx* ctx, JitKind kind, const AirComponent& c, const std::vector<AirFrac>& fr, JitKernel* out);
// copies cols[0 .. n_cols) (host memory, one device column per mask) into the kernel's column table and launches it on ctx->stream
nb200_status jit_launch(nb200_ctx* ctx, const JitKernel& jk, const u32* const* cols, size_t n_cols, dim3 grid, dim3 block, void** args, size_t smem = 0);
void jit_release(JitKernel& jk);
void jit_coeff_table(const std::vector<qm31>& coeffs, std::vector<u32>& out);

}  // namespace nb
