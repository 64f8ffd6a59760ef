// One row of the v1 main component's main trace (347 columns, prover/src/column.rs) for a program of RV32I's ALU instructions (ADD ...
// SRAI, add_chain.OPCODES), branches, JAL, JALR, LUI and AUIPC (add_chain.CONTROL_OPCODES), filled from its step record
// (add_chain.STEP_FIELDS): the per-row fills of CpuChip (chips/cpu.rs:36-316), DecodingCheck types R, I, I with a shift amount, B, U and J
// (decoding/type_r.rs:25-60, type_i.rs:29-69,288-330, type_b.rs:33-73, type_u.rs:29-51, type_j.rs:29-62), AddChip, SubChip, SltuChip,
// BitOpChip, SltChip, the branch chips, JalChip, LuiChip, AuipcChip, JalrChip, SllChip, SrlChip and SraChip (instructions/i/add.rs:64-100,
// sub.rs:66-100, sltu.rs:45-75, bit_op.rs:249-300, slt.rs:56-110, beq.rs:34-104, bne.rs, bltu.rs:28-55, blt.rs:38-86, bgeu.rs, bge.rs,
// jal.rs:33-73, lui.rs, auipc.rs:33-62, jalr.rs:38-101, sll.rs:72-112, srl.rs:79-119, sra.rs:93-139), ProgramMemCheck (memory_check/program_mem_check.rs:44-100),
// RegisterMemCheck (register_mem_check.rs:53-117) and Timestamp (timestamp.rs:33-75), or the reference's padding row past the last step.
// The same code runs in v1_main_trace_kernel (v1_trace.cu) and, compiled as host C++, in tests/test_add_chain_cpu.py and
// tests/test_alu_program_cpu.py and tests/test_control_program_cpu.py, which compare every row with add_chain.main_columns.  Rows are addressed by their finalized position
// (finalize_order.cuh).
#pragma once
#include "m31.cuh"
#include "finalize_order.cuh"

namespace nb {
namespace v1 {

constexpr u32 MAIN_COLS = 347;
// the step record, one array of n_steps words per field (include/nb200.h, nb200_v1_main_trace)
enum StepField : u32 { PC, WORD, OPCODE, RD, RS1, OP_C, VALUE_B, VALUE_C, RD_PREV, TS1_PREV, TS2_PREV, TS3_PREV, PC_CTR_PREV, STEP_FIELDS };
// opcode numbers of the step record (include/nb200.h): type R, type I, type I with a shift amount
enum Opcode : u32 { OP_ADD, OP_ADDI, OP_SUB, OP_SLL, OP_SLT, OP_SLTU, OP_XOR, OP_SRL, OP_SRA, OP_OR, OP_AND, OP_SLTI, OP_SLTIU, OP_XORI, OP_ORI,
                    OP_ANDI, OP_SLLI, OP_SRLI, OP_SRAI, N_OPCODES };
// the control-flow opcodes after them (nb200_v1_control_trace): type B, JAL (type J), JALR (type I), LUI and AUIPC (type U)
enum ControlOpcode : u32 { OP_BEQ = N_OPCODES, OP_BNE, OP_BLT, OP_BGE, OP_BLTU, OP_BGEU, OP_JAL, OP_JALR, OP_LUI, OP_AUIPC, N_ALL_OPCODES };
NB_HD bool is_type_b(u32 op) { return op >= OP_BEQ && op <= OP_BGEU; }
NB_HD bool is_type_r(u32 op) { return op == OP_ADD || (op >= OP_SUB && op <= OP_AND); }
NB_HD bool is_type_i(u32 op) { return op == OP_ADDI || (op >= OP_SLTI && op <= OP_ANDI); }
NB_HD bool is_type_i_shift(u32 op) { return op >= OP_SLLI && op <= OP_SRAI; }
// the register-register instruction an opcode computes (SLTIU: SLTU)
NB_HD u32 base_op(u32 op) {
  switch (op) {
    case OP_ADDI: return OP_ADD;
    case OP_SLTI: return OP_SLT;
    case OP_SLTIU: return OP_SLTU;
    case OP_XORI: return OP_XOR;
    case OP_ORI: return OP_OR;
    case OP_ANDI: return OP_AND;
    case OP_SLLI: return OP_SLL;
    case OP_SRLI: return OP_SRL;
    case OP_SRAI: return OP_SRA;
    default: return op;
  }
}

// first column of each word this fill writes (MAIN_COLUMNS order, nexus_v1.py; tests/test_add_chain_cpu.py checks them against it).
// Every other column is zero on ADD, ADDI and padding rows.
namespace col {
constexpr u32 Pc = 0, PcNext = 4, OpA = 12, OpB = 13, OpC = 14, CarryFlag = 15, ImmC = 19, InstrVal = 20, ValueA = 28, ValueAEffective = 32,
              ValueB = 36, ValueC = 40, IsAdd = 44, IsPadding = 90, ValueAEffectiveFlag = 206, ValueAEffectiveFlagAux = 207,
              ValueAEffectiveFlagAuxInv = 208, Reg1Address = 209, Reg2Address = 210, Reg3Address = 211, Reg1ValPrev = 212, Reg2ValPrev = 216,
              Reg3ValPrev = 220, Reg1TsPrev = 224, ProgCtrPrev = 236, ProgCtrCur = 240, ProgCtrCarry = 244, FinalPrgMemoryCtr = 246,
              CReg1TsPrev = 250, CH1Minus = 262, OpC0_3 = 312, OpC4_7 = 315, OpC8_10 = 317, OpC11 = 318, OpA1_4 = 321, OpB1_4 = 323,
              OpC4 = 325, OpA0 = 326, OpB0 = 327, PcCarry = 333;
// the instruction chips' columns beyond the ADD chain's
constexpr u32 IsOr = 45, IsAnd = 46, IsXor = 47, IsSub = 48, IsSltu = 49, IsSlt = 50, IsSll = 69, IsSrl = 70, IsSra = 71, Helper1 = 91,
              Helper2 = 95, Helper3 = 99, SgnB = 108, SgnC = 109, Rem = 115, Qt = 120, ShiftBit1 = 124, Exp1_3 = 129, Exp = 130, RemDiff = 131,
              SraDegreeAux = 139, ValueA4_7 = 335, ValueB4_7 = 339, ValueC4_7 = 343;
// the control-flow chips' and DecodingCheck B / U / J's columns
constexpr u32 PcNextAux = 8, BorrowFlag = 17, IsBne = 51, IsBeq = 52, IsBltu = 53, IsBlt = 54, IsBgeu = 55, IsBge = 56, IsJal = 57, IsLui = 66,
              IsAuipc = 67, IsJalr = 68, SgnA = 107, Neq = 110, Neq12 = 111, Neq34 = 112, LtFlag = 113, RemAux = 114, QtAux = 119, Neq12Aux = 135,
              Neq34Aux = 136, Neq12AuxInv = 137, Neq34AuxInv = 138, OpC1_3 = 313, OpC1_4 = 314, OpC5_7 = 316, OpC12 = 319, OpC20 = 320,
              OpB0_3 = 322, OpB4 = 328, OpC12_15 = 329, OpC16_23 = 330, OpC16_19 = 331, OpC24_31 = 332;
}  // namespace col

// carries out of the low and high 16 bits of x + y (limbs 1 and 3 of add_with_carries, add.rs:27-45)
NB_HD void carries16(u32 x, u32 y, u32& c0, u32& c1) {
  const u32 lo = (x & 0xFFFFu) + (y & 0xFFFFu);
  c0 = lo >> 16;
  c1 = ((x >> 16) + (y >> 16) + c0) >> 16;
}

// RV32I's result of the register-register instruction `base` on b and c (rs2's value, the immediate or the shift amount)
NB_HD u32 alu_result(u32 base, u32 b, u32 c) {
  switch (base) {
    case OP_SUB: return b - c;
    case OP_SLL: return b << (c & 31);
    case OP_SLT: return (int32_t)b < (int32_t)c ? 1u : 0u;
    case OP_SLTU: return b < c ? 1u : 0u;
    case OP_XOR: return b ^ c;
    case OP_SRL: return b >> (c & 31);
    case OP_SRA: return (u32)((int32_t)b >> (c & 31));
    case OP_OR: return b | c;
    case OP_AND: return b & c;
    default: return b + c;
  }
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
  const u32 op = field(OPCODE), base = base_op(op), rd_prev = field(RD_PREV);
  const bool is_r = exec && is_type_r(op), is_i = exec && (is_type_i(op) || op == OP_JALR), is_shift = exec && is_type_i_shift(op);
  const bool is_b = exec && is_type_b(op), jal = exec && op == OP_JAL, jalr = exec && op == OP_JALR, lui = exec && op == OP_LUI;
  const bool auipc = exec && op == OP_AUIPC, is_u = lui || auipc;
  // ValueA: the ALU result; a branch's op_a value (read through Reg3 and written back), the link pc + 4, LUI's ValueC, AUIPC's pc + ValueC
  const u32 a = is_b ? rd_prev : jal || jalr ? pc + 4 : lui ? c : auipc ? pc + c : alu_result(base, b, c);
  bool taken = false;
  switch (is_b ? op : 0u) {
    case OP_BEQ: taken = a == b; break;
    case OP_BNE: taken = a != b; break;
    case OP_BLT: taken = (int32_t)a < (int32_t)b; break;
    case OP_BGE: taken = (int32_t)a >= (int32_t)b; break;
    case OP_BLTU: taken = a < b; break;
    case OP_BGEU: taken = a >= b; break;
    default: break;
  }
  const u32 pc_next = taken || jal ? pc + c : jalr ? (b + c) & ~1u : pc + 4;
  u32 c0, c1;
  // CpuChip
  put(col::IsPadding, exec ? 0u : 1u);
  put(col::ImmC, exec && !is_r ? 1u : 0u);
  put(col::ValueAEffectiveFlag, rd != 0);
  put(col::ValueAEffectiveFlagAux, rd ? m31_inv(rd) : 1u);
  put(col::ValueAEffectiveFlagAuxInv, rd ? rd : 1u);
  put_word(col::Pc, pc);
  put_word(col::PcNext, exec ? pc_next : 0u);
  carries16(pc, 4, c0, c1);
  put(col::PcCarry, exec ? c0 : 0u);
  put(col::PcCarry + 1, exec ? c1 : 0u);
  put_word(col::InstrVal, word);
  put_word(col::ValueB, b);
  put_word(col::ValueC, c);
  put(col::OpA, rd);
  put(col::OpB, rs1);
  put(col::OpC, is_i ? op_c & 0xFFFu : is_b ? op_c & 0x1FFFu : jal ? op_c & 0x1FFFFFu : op_c);
  put(col::Reg1Address, rs1);
  put(col::Reg2Address, is_r ? op_c : 0u);
  put(col::Reg3Address, rd);
  // DecodingCheck: type R, type I without and with a shift amount; types B, U and J
  const bool r_or_i = is_r || is_i || is_shift;
  put(col::OpA0, rd & 1);
  put(col::OpA1_4, (rd >> 1) & 0xF);
  put(col::OpB0, r_or_i ? rs1 & 1 : 0u);
  put(col::OpB1_4, r_or_i ? (rs1 >> 1) & 0xF : 0u);
  put(col::OpC0_3, r_or_i ? op_c & 0xF : 0u);
  put(col::OpC4, is_r || is_shift ? (op_c >> 4) & 1 : 0u);
  put(col::OpC4_7, is_i || jal ? (op_c >> 4) & 0xF : 0u);
  put(col::OpC8_10, is_i || is_b || jal ? (op_c >> 8) & 0x7 : 0u);
  put(col::OpC11, is_i || is_b || jal ? (op_c >> 11) & 1 : 0u);
  put(col::OpC1_4, is_b ? (op_c >> 1) & 0xF : 0u);
  put(col::OpC5_7, is_b ? (op_c >> 5) & 0x7 : 0u);
  put(col::OpC12, is_b ? (op_c >> 12) & 1 : 0u);
  put(col::OpB0_3, is_b ? rs1 & 0xF : 0u);
  put(col::OpB4, is_b ? rs1 >> 4 : 0u);
  put(col::OpC1_3, jal ? (op_c >> 1) & 0x7 : 0u);
  put(col::OpC12_15, jal ? (op_c >> 12) & 0xF : is_u ? op_c & 0xF : 0u);
  put(col::OpC16_19, jal ? (op_c >> 16) & 0xF : 0u);
  put(col::OpC20, jal ? (op_c >> 20) & 1 : 0u);
  put(col::OpC16_23, is_u ? (op_c >> 4) & 0xFF : 0u);
  put(col::OpC24_31, is_u ? (op_c >> 12) & 0xFF : 0u);
  // the instruction chips: ValueA, and each chip's helpers, zero on the rows of other opcodes.  Every column is written by every thread,
  // so a warp over rows of mixed opcodes still writes whole 128-byte lines instead of one partial store per opcode.
  put_word(col::ValueA, a);
  const bool add = exec && base == OP_ADD, slt = exec && base == OP_SLT, sltx = slt || (exec && base == OP_SLTU);
  const bool sub = sltx || (exec && base == OP_SUB), bit = exec && (base == OP_XOR || base == OP_OR || base == OP_AND);
  const bool sll = exec && base == OP_SLL, sra = exec && base == OP_SRA, srx = sra || (exec && base == OP_SRL), shift = sll || srx;
  // CarryFlag: AddChip's carries of b + c, the carries of the branches' PcNext = pc + (c or 4), of JAL / JALR's ValueA = pc + 4 and of
  // AUIPC's pc + c; SubChip, SltuChip, SltChip: the borrows of b - c
  const bool cmp = is_b && op != OP_BEQ && op != OP_BNE, lt = exec && (op == OP_BLT || op == OP_BGE);
  const bool carry = add || is_b || jal || jalr || auipc;
  carries16(add ? b : pc, add ? c : is_b ? (taken ? c : 4u) : jal || jalr ? 4u : c, c0, c1);
  put(col::CarryFlag, carry ? c0 : sub && (b & 0xFFFFu) < (c & 0xFFFFu) ? 1u : 0u);
  put(col::CarryFlag + 1, carry ? c1 : sub && b < c ? 1u : 0u);
  // BorrowFlag: the compare branches' borrows of a - b, the carries of JAL's PcNext = pc + c and of JALR's PcNextAux = b + c
  carries16(jal ? pc : b, c, c0, c1);
  put(col::BorrowFlag, cmp ? ((a & 0xFFFFu) < (b & 0xFFFFu) ? 1u : 0u) : jal || jalr ? c0 : 0u);
  put(col::BorrowFlag + 1, cmp ? (a < b ? 1u : 0u) : jal || jalr ? c1 : 0u);
  put_word(col::PcNextAux, jalr ? b + c : 0u);
  put(col::RemAux, jalr ? (b + c) & 1 : 0u);
  put(col::QtAux, jalr ? ((b + c) & 0xFFu) >> 1 : 0u);
  // Helper1: b - c for SltuChip / SltChip, the shift amount's bits 5..7 for the shift chips, a - b for the compare branches; Helper2 /
  // Helper3: SltChip's b and c without their sign bits, SraChip's top byte of b without it and the logical shift, BLT / BGE's a and b
  // without their sign bits
  const u32 s3 = c & 7, e = 1u << s3, sh = c & 31, sgn_b = b >> 31;
  put_word(col::Helper1, sltx ? b - c : shift ? (c & 0xFFu) >> 5 : cmp ? a - b : 0u);
  put_word(col::Helper2, slt ? b & 0x7FFFFFFFu : sra ? (b >> 24) & 0x7Fu : lt ? a & 0x7FFFFFFFu : 0u);
  put_word(col::Helper3, slt ? c & 0x7FFFFFFFu : sra ? b >> sh : lt ? b & 0x7FFFFFFFu : 0u);
  put(col::SgnB, slt || sra || (exec && op == OP_BGE) ? sgn_b : 0u);
  put(col::SgnC, slt ? c >> 31 : 0u);
  put(col::SgnA, exec && op == OP_BGE ? a >> 31 : 0u);
  put(col::LtFlag, lt && (int32_t)a < (int32_t)b ? 1u : 0u);
  // BeqChip / BneChip: whether the 16-bit halves of a and b differ, and the inverse of their difference, or of pc's half read big-endian
  // (beq.rs:41-42) when they are equal
  const bool eq = exec && (op == OP_BEQ || op == OP_BNE);
  put(col::Neq, eq && a != b ? 1u : 0u);
#pragma unroll
  for (u32 k = 0; k < 2; ++k) {
    const u32 ah = (a >> (16 * k)) & 0xFFFFu, bh = (b >> (16 * k)) & 0xFFFFu;
    const u32 pc_be = ((pc >> (16 * k)) & 0xFFu) << 8 | ((pc >> (16 * k + 8)) & 0xFFu);
    const u32 aux_inv = ah != bh ? (ah + P31 - bh) % P31 : (pc_be ? pc_be : 1u);
    put(col::Neq12 + k, eq && ah != bh ? 1u : 0u);
    put(col::Neq12Aux + k, eq ? m31_inv(aux_inv) : 0u);
    put(col::Neq12AuxInv + k, eq ? aux_inv : 0u);
  }
#pragma unroll
  for (u32 k = 0; k < 4; ++k) {                                                 // BitOpChip: the high nibbles
    put(col::ValueA4_7 + k, bit ? (a >> (8 * k + 4)) & 15u : 0u);
    put(col::ValueB4_7 + k, bit ? (b >> (8 * k + 4)) & 15u : 0u);
    put(col::ValueC4_7 + k, bit ? (c >> (8 * k + 4)) & 15u : 0u);
  }
  // SllChip, SrlChip, SraChip: Exp1_3 = 2^(low three bits of the amount); SLL multiplies b by it byte by byte (Rem, carries Qt), SRL / SRA
  // divide b by it from the top byte (quotients Qt, remainders Rem, RemDiff = Exp1_3 - 1 - Rem); SRA's Exp = 2^8 / Exp1_3
#pragma unroll
  for (u32 k = 0; k < 5; ++k) put(col::ShiftBit1 + k, shift ? (c >> k) & 1 : 0u);
  put(col::Exp1_3, shift ? e : 0u);
#pragma unroll
  for (u32 k = 0; k < 4; ++k) {
    const u32 rem = (b >> (8 * k)) & (e - 1);
    put(col::Rem + k, sll ? ((b << s3) >> (8 * k)) & 255u : srx ? rem : 0u);
    put(col::Qt + k, sll ? (u32)(((u64)b >> (8 * k + 8 - s3)) & (e - 1)) : srx ? ((b >> s3) >> (8 * k)) & 255u : 0u);
    put(col::RemDiff + k, srx ? e - 1 - rem : 0u);
  }
  put(col::Exp, sra ? 256u >> s3 : 0u);
  put(col::SraDegreeAux, sra ? sgn_b * (e - 1) * (256u >> s3) : 0u);
  // CpuChip's opcode flags
  put(col::IsAdd, add);
  put(col::IsSub, exec && base == OP_SUB);
  put(col::IsSltu, exec && base == OP_SLTU);
  put(col::IsSlt, slt);
  put(col::IsXor, exec && base == OP_XOR);
  put(col::IsOr, exec && base == OP_OR);
  put(col::IsAnd, exec && base == OP_AND);
  put(col::IsSll, sll);
  put(col::IsSrl, exec && base == OP_SRL);
  put(col::IsSra, sra);
  put(col::IsBeq, exec && op == OP_BEQ);
  put(col::IsBne, exec && op == OP_BNE);
  put(col::IsBlt, exec && op == OP_BLT);
  put(col::IsBge, exec && op == OP_BGE);
  put(col::IsBltu, exec && op == OP_BLTU);
  put(col::IsBgeu, exec && op == OP_BGEU);
  put(col::IsJal, jal);
  put(col::IsJalr, jalr);
  put(col::IsLui, lui);
  put(col::IsAuipc, auipc);
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
  put_word(col::Reg2ValPrev, is_r ? c : 0u);
  put_word(col::Reg3ValPrev, rd_prev);
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
