// One row of the v1 main component's main trace (347 columns, prover/src/column.rs) for an ADD / ADDI program, filled from its step
// record (add_chain.STEP_FIELDS): the per-row fills of CpuChip (chips/cpu.rs:36-316), DecodingCheck types R and I (decoding/type_r.rs:25-60,
// type_i.rs:29-69), AddChip (instructions/i/add.rs:64-100), ProgramMemCheck (memory_check/program_mem_check.rs:44-100), RegisterMemCheck
// (register_mem_check.rs:53-117) and Timestamp (timestamp.rs:33-75), or the reference's padding row past the last step.
// The same code runs in v1_main_trace_kernel (v1_trace.cu) and, compiled as host C++, in tests/test_add_chain_cpu.py, which compares every
// row with AddChainMachine.fill_main_trace().  Rows are addressed by their finalized position (finalize_order.cuh).
#pragma once
#include "m31.cuh"
#include "finalize_order.cuh"

namespace nb {
namespace v1 {

constexpr u32 MAIN_COLS = 347;
// the step record, one array of n_steps words per field (include/nb200.h, nb200_v1_main_trace)
enum StepField : u32 { PC, WORD, OPCODE, RD, RS1, OP_C, VALUE_B, VALUE_C, RD_PREV, TS1_PREV, TS2_PREV, TS3_PREV, PC_CTR_PREV, STEP_FIELDS };
constexpr u32 OP_ADD = 0, OP_ADDI = 1;

// first column of each word this fill writes (MAIN_COLUMNS order, nexus_v1.py; tests/test_add_chain_cpu.py checks them against it).
// Every other column is zero on ADD, ADDI and padding rows.
namespace col {
constexpr u32 Pc = 0, PcNext = 4, OpA = 12, OpB = 13, OpC = 14, CarryFlag = 15, ImmC = 19, InstrVal = 20, ValueA = 28, ValueAEffective = 32,
              ValueB = 36, ValueC = 40, IsAdd = 44, IsPadding = 90, ValueAEffectiveFlag = 206, ValueAEffectiveFlagAux = 207,
              ValueAEffectiveFlagAuxInv = 208, Reg1Address = 209, Reg2Address = 210, Reg3Address = 211, Reg1ValPrev = 212, Reg2ValPrev = 216,
              Reg3ValPrev = 220, Reg1TsPrev = 224, ProgCtrPrev = 236, ProgCtrCur = 240, ProgCtrCarry = 244, FinalPrgMemoryCtr = 246,
              CReg1TsPrev = 250, CH1Minus = 262, OpC0_3 = 312, OpC4_7 = 315, OpC8_10 = 317, OpC11 = 318, OpA1_4 = 321, OpB1_4 = 323,
              OpC4 = 325, OpA0 = 326, OpB0 = 327, PcCarry = 333;
}  // namespace col

// carries out of the low and high 16 bits of x + y (limbs 1 and 3 of add_with_carries, add.rs:27-45)
NB_HD void carries16(u32 x, u32 y, u32& c0, u32& c1) {
  const u32 lo = (x & 0xFFFFu) + (y & 0xFFFFu);
  c0 = lo >> 16;
  c1 = ((x >> 16) + (y >> 16) + c0) >> 16;
}

// Row at finalized position i of 2^log_size rows into out[c * stride]: trace row r = finalized_src_row(i) is step r when r < n_steps and a
// padding row otherwise; FinalPrgMemoryCtr holds final_ctr[r] on the program's rows r < n_prog.  Writes the columns of `col` only.
// steps = STEP_FIELDS x n_steps words (field-major), already checked by the host (v1_main_trace).
NB_HD void main_row(const u32* steps, u32 n_steps, const u32* final_ctr, u32 n_prog, u32 log_size, u32 i, u32* out, size_t stride) {
  const u32 r = (u32)finalized_src_row(i, log_size);
  const bool exec = r < n_steps;
  auto put = [&](u32 c, u32 v) { out[(size_t)c * stride] = v; };
  auto put_word = [&](u32 c, u32 v) {
#pragma unroll
    for (u32 k = 0; k < 4; ++k) put(c + k, (v >> (8 * k)) & 255u);
  };
  auto field = [&](u32 f) { return exec ? steps[(size_t)f * n_steps + r] : 0u; };
  const u32 pc = field(PC), word = field(WORD), rd = field(RD), rs1 = field(RS1), op_c = field(OP_C);
  const u32 b = field(VALUE_B), c = field(VALUE_C);
  const bool is_add = exec && field(OPCODE) == OP_ADD, is_addi = exec && field(OPCODE) == OP_ADDI;
  u32 c0, c1;
  // CpuChip
  put(col::IsPadding, exec ? 0u : 1u);
  put(col::IsAdd, exec ? 1u : 0u);
  put(col::ImmC, is_addi ? 1u : 0u);
  put(col::ValueAEffectiveFlag, rd != 0);
  put(col::ValueAEffectiveFlagAux, rd ? m31_inv(rd) : 1u);
  put(col::ValueAEffectiveFlagAuxInv, rd ? rd : 1u);
  put_word(col::Pc, pc);
  put_word(col::PcNext, exec ? pc + 4 : 0u);
  carries16(pc, 4, c0, c1);
  put(col::PcCarry, exec ? c0 : 0u);
  put(col::PcCarry + 1, exec ? c1 : 0u);
  put_word(col::InstrVal, word);
  put_word(col::ValueB, b);
  put_word(col::ValueC, c);
  put(col::OpA, rd);
  put(col::OpB, rs1);
  put(col::OpC, is_addi ? op_c & 0xFFFu : op_c);
  put(col::Reg1Address, rs1);
  put(col::Reg2Address, is_add ? op_c : 0u);
  put(col::Reg3Address, rd);
  // DecodingCheck: type R (ADD) and type I without shift (ADDI)
  put(col::OpA0, rd & 1);
  put(col::OpA1_4, (rd >> 1) & 0xF);
  put(col::OpB0, rs1 & 1);
  put(col::OpB1_4, (rs1 >> 1) & 0xF);
  put(col::OpC0_3, op_c & 0xF);
  put(col::OpC4, is_add ? (op_c >> 4) & 1 : 0u);
  put(col::OpC4_7, is_addi ? (op_c >> 4) & 0xF : 0u);
  put(col::OpC8_10, is_addi ? (op_c >> 8) & 0x7 : 0u);
  put(col::OpC11, is_addi ? (op_c >> 11) & 1 : 0u);
  // AddChip
  const u32 a = b + c;
  put_word(col::ValueA, a);
  carries16(b, c, c0, c1);
  put(col::CarryFlag, c0);
  put(col::CarryFlag + 1, c1);
  // ProgramMemCheck
  const u32 ctr = field(PC_CTR_PREV);
  put_word(col::ProgCtrPrev, ctr);
  put_word(col::ProgCtrCur, exec ? ctr + 1 : 0u);
  carries16(ctr, 1, c0, c1);
  put(col::ProgCtrCarry, exec ? c0 : 0u);
  put(col::ProgCtrCarry + 1, exec ? c1 : 0u);
  put_word(col::FinalPrgMemoryCtr, r < n_prog ? final_ctr[r] : 0u);
  // RegisterMemCheck
  put_word(col::ValueAEffective, rd ? a : 0u);
  put_word(col::Reg1ValPrev, b);
  put_word(col::Reg2ValPrev, is_add ? c : 0u);
  put_word(col::Reg3ValPrev, field(RD_PREV));
  // Timestamp, every row: c = cur - 1 - prev against Reg{1,2,3}TsCur = 3 clk + {1,2,3}, the borrows out of the low and high 16 bits
  const u32 clk = r + 1;
#pragma unroll
  for (u32 k = 0; k < 3; ++k) {
    const u32 prev = field(TS1_PREV + k), cur = 3 * clk + k + 1;
    put_word(col::Reg1TsPrev + 4 * k, prev);
    put_word(col::CReg1TsPrev + 4 * k, cur - 1 - prev);
    put(col::CH1Minus + 2 * k, (cur & 0xFFFFu) < (prev & 0xFFFFu) + 1u ? 1u : 0u);
    put(col::CH1Minus + 2 * k + 1, 0u);
  }
}

}  // namespace v1
}  // namespace nb
