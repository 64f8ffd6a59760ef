// The v1 main component's main trace filled on the device from a program's step record (nb200_v1_main_trace for ADD / ADDI programs,
// nb200_v1_alu_trace for the 19 ALU opcodes, nb200_v1_control_trace for those and the 10 control-flow opcodes; one kernel behind three
// host checks): what add_chain.main_columns builds for the main
// component on the host, followed by finalize_columns, without the host columns or their upload.  The batch is cleared first (the columns
// no executed or padding row sets stay zero); then one thread per finalized row position writes its row's other columns (v1_trace.cuh),
// so consecutive threads write consecutive words of every column.
#include "common.cuh"
#include "v1_trace.cuh"
#include <algorithm>

namespace nb {
namespace {

constexpr u32 V1_BLOCK = 128;
static_assert(v1::STEP_FIELDS == NB200_V1_STEP_FIELDS, "the step record of include/nb200.h");

__global__ void __launch_bounds__(V1_BLOCK) v1_main_trace_kernel(const u32* __restrict__ steps, u32 n_steps, const u32* __restrict__ final_ctr,
                                                                 u32 n_prog, u32 log_size, u32* out) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (1u << log_size)) return;
  v1::main_row(steps, n_steps, final_ctr, n_prog, log_size, i, out + i, (size_t)1 << log_size);
}

// Which opcodes a fill entry takes: ADD and ADDI (nb200_v1_main_trace), the 19 ALU opcodes (nb200_v1_alu_trace) or all 29
// (nb200_v1_control_trace).
enum class Opcodes { ADD_ADDI, ALU, CONTROL };

// The host check of a step record and the fill: the opcodes of `ops` with their operand ranges.  The fill does not check that the pcs
// chain; the main component's next-row Pc constraint does.
nb200_status v1_fill(nb200_ctx* ctx, const char* who, Opcodes ops, size_t n_steps, const uint32_t* steps, size_t n_prog, const uint32_t* final_ctr,
                     uint32_t log_size, nb200_cols* out) {
  const std::string me = who;
  NB_ARG(ctx, out && (n_steps == 0 || steps) && (n_prog == 0 || final_ctr), me + ": null argument");
  NB_ARG(ctx, log_size >= 4 && log_size <= 28, me + ": log_size must be in [4, 28]");
  NB_ARG(ctx, out->n_cols == v1::MAIN_COLS && out->log_size == log_size, me + ": out must be a batch of 347 columns of 2^log_size rows");
  const size_t n = (size_t)1 << log_size;
  NB_ARG(ctx, n_steps <= n, me + ": more steps than 2^log_size rows");
  NB_ARG(ctx, n_prog <= n, me + ": more program rows than 2^log_size rows");
  auto f = [&](u32 field, size_t t) { return steps[field * n_steps + t]; };
  for (size_t t = 0; t < n_steps; ++t) {
    const u32 op = f(v1::OPCODE, t), op_c = f(v1::OP_C, t);
    if (ops != Opcodes::ADD_ADDI) {
      if (ops == Opcodes::ALU)
        NB_ARG(ctx, op < v1::N_OPCODES, me + ": step " + std::to_string(t) + " has an opcode above 18");
      else
        NB_ARG(ctx, op < v1::N_ALL_OPCODES, me + ": step " + std::to_string(t) + " has an opcode above 28");
      NB_ARG(ctx, !v1::is_type_i_shift(op) || op_c < 32, me + ": step " + std::to_string(t) + " has a shift amount above 31");
      NB_ARG(ctx, !(v1::is_type_i(op) || op == v1::OP_JALR) || op_c + 2048u < 4096u,
             me + ": step " + std::to_string(t) + " has an immediate that is not a sign-extended 12-bit value");
      NB_ARG(ctx, !v1::is_type_b(op) || (op_c + 4096u < 8192u && op_c % 2 == 0),
             me + ": step " + std::to_string(t) + " has a branch offset that is not an even sign-extended 13-bit value");
      NB_ARG(ctx, op != v1::OP_JAL || (op_c + (1u << 20) < (1u << 21) && op_c % 2 == 0),
             me + ": step " + std::to_string(t) + " has a JAL offset that is not an even sign-extended 21-bit value");
      NB_ARG(ctx, (op != v1::OP_LUI && op != v1::OP_AUIPC) || op_c < (1u << 20),
             me + ": step " + std::to_string(t) + " has a U-type immediate above 20 bits");
    } else {
      NB_ARG(ctx, op == v1::OP_ADD || op == v1::OP_ADDI, me + ": step " + std::to_string(t) + " is not ADD or ADDI");
    }
    NB_ARG(ctx, f(v1::RD, t) < 32 && f(v1::RS1, t) < 32 && (!v1::is_type_r(op) || op_c < 32),
           me + ": step " + std::to_string(t) + " has a register index above 31");
    const u64 clk = t + 1;
    for (u32 k = 0; k < 3; ++k)
      NB_ARG(ctx, f(v1::TS1_PREV + k, t) < 3 * clk + k + 1,
             me + ": step " + std::to_string(t) + " has a previous timestamp not below the current one");
    NB_ARG(ctx, f(v1::PC_CTR_PREV, t) != 0xFFFFFFFFu, me + ": a program counter of 2^32 - 1 has no successor");
  }
  // scratch, freed in stream order when the call returns: the step record and the final counters
  DevBuf d_steps, d_ctr;
  NB_TRY(alloc(ctx, d_steps, std::max<size_t>(n_steps * v1::STEP_FIELDS, 1)));
  NB_TRY(alloc(ctx, d_ctr, std::max<size_t>(n_prog, 1)));
  if (n_steps)
    NB_CUDA(ctx, cudaMemcpyAsync(d_steps.p, steps, n_steps * v1::STEP_FIELDS * 4, cudaMemcpyHostToDevice, ctx->stream));
  if (n_prog) NB_CUDA(ctx, cudaMemcpyAsync(d_ctr.p, final_ctr, n_prog * 4, cudaMemcpyHostToDevice, ctx->stream));
  NB_CUDA(ctx, cudaMemsetAsync(out->d, 0, (size_t)v1::MAIN_COLS * n * 4, ctx->stream));
  v1_main_trace_kernel<<<(u32)((n + V1_BLOCK - 1) / V1_BLOCK), V1_BLOCK, 0, ctx->stream>>>(d_steps.p, (u32)n_steps, d_ctr.p, (u32)n_prog, log_size,
                                                                                          out->d);
  NB_LAUNCH_CHECK(ctx);
  return NB200_OK;
}

}  // namespace

nb200_status v1_main_trace(nb200_ctx* ctx, size_t n_steps, const uint32_t* steps, size_t n_prog, const uint32_t* final_ctr, uint32_t log_size,
                           nb200_cols* out) {
  return v1_fill(ctx, "v1_main_trace", Opcodes::ADD_ADDI, n_steps, steps, n_prog, final_ctr, log_size, out);
}

nb200_status v1_alu_trace(nb200_ctx* ctx, size_t n_steps, const uint32_t* steps, size_t n_prog, const uint32_t* final_ctr, uint32_t log_size,
                          nb200_cols* out) {
  return v1_fill(ctx, "v1_alu_trace", Opcodes::ALU, n_steps, steps, n_prog, final_ctr, log_size, out);
}

nb200_status v1_control_trace(nb200_ctx* ctx, size_t n_steps, const uint32_t* steps, size_t n_prog, const uint32_t* final_ctr, uint32_t log_size,
                              nb200_cols* out) {
  return v1_fill(ctx, "v1_control_trace", Opcodes::CONTROL, n_steps, steps, n_prog, final_ctr, log_size, out);
}

}  // namespace nb
