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
uint64_t jit_source_key(const std::string& src);   // name of the kernel's file in the cubin cache
// the CUDA C the component's constraints are specialised to (inspection / offline ptxas checks): d2 = false every constraint (with the
// high-degree part on the side, jit.cu gen_source), d2 = true the constraints of degree above AIR_LOW_DEGREE only
std::string jit_source(const AirComponent& c, bool d2 = false);
nb200_status jit_compile_constraints(nb200_ctx* ctx, const AirComponent& c, bool d2, JitKernel* out);
nb200_status jit_compile_logup(nb200_ctx* ctx, const AirComponent& c, JitKernel* out);
nb200_status jit_launch_logup(nb200_ctx* ctx, const JitKernel& jk, const u32* const* d_cols, const u32* d_params, u32* d_out, u32 log_size);
std::string jit_logup_source(const AirComponent& c);
// the constraint check on the trace domain (jit.cu gen_check_source): per constraint, the count of rows where it is non-zero and the
// first such row in coset order, accumulated into d_nfail / d_first (zeros / 0xffffffff before the launch)
std::string jit_check_source(const AirComponent& c);
nb200_status jit_compile_check(nb200_ctx* ctx, const AirComponent& c, JitKernel* out);
nb200_status jit_launch_check(nb200_ctx* ctx, const JitKernel& jk, const u32* const* d_cols, const u32* d_params, u32* d_nfail, u32* d_first);
nb200_status jit_launch_constraints(nb200_ctx* ctx, const JitKernel& jk, const u32* const* d_cols, const u32* d_params, const u32* d_coeff,
                                    const u32* d_dinv, u32* const acc[4], u32 rows_log, u32 dom_log, u32 row0 = 0, size_t n_rows = 0,
                                    u32* const acc_high[4] = nullptr);
void jit_release(JitKernel& jk);
void jit_coeff_table(const std::vector<qm31>& coeffs, std::vector<u32>& out);

}  // namespace nb
