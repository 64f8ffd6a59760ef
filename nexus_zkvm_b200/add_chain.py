"""The reference's ADD-chain benchmark proven as an executing v1 trace: the shape of `Machine::prove` (nexus-zkvm prover/src/machine.rs:126-297,
`prove_with_extensions(&[])`) on the program of prover-benches/benches/stark_prove.rs (common-testing/src/lib.rs:5-30):

    addi x1, x0, 1
    add  x_k, x_j, x_i          i, j, k = 0, 1, 2 at first, each + 1 mod 32 per instruction

2^n instructions, each executed once, so 2^n executed steps and no padding rows; `n_steps < 2^log_size` runs the first n_steps
instructions and pads the rest with the reference's padding rows.  The program is laid out as HarvardEmulator::from_basic_blocks lays it out
(vm/src/emulator/executor.rs:501-524): base address and entry point ELF_TEXT_START = 136, every register 0, the global clock 1 at the first
step; the view has no initial, input, exit-code or output memory, so RamInitFinal is empty (its 2^4 rows are padding).

Components, in the reference's order:
   0 main component              nexus_v1.record_main_component with DecodingCheck's types R and I (decoding=True)
   1 FinalReg                    the final register file: (index, final timestamp, final value) per register
   2 BitOpMultiplicity           no bit-op lookup in the ADD chain: zero
   3 RamInitFinal                2^4 zero rows
   4-8 Multiplicity8/16/32/128/256
Relations: BitOp, LoadStore, ProgramCheck, RegisterCheck, Range8, 16, 32, 128, 256 (draw_lookup_elements over BaseComponent).

AluMachine runs a straight-line program of every RV32I register-register and register-immediate instruction but LUI / AUIPC (OPCODES,
alu_program) on the same components, its main component also recorded with SltuChip, SltChip, SllChip, SrlChip and SraChip (alu=True); its
bit-op instructions make BitOpMultiplicity nonzero.

ControlMachine runs a looping program (control_program) that adds RV32I's branches, JAL, JALR, LUI and AUIPC (CONTROL_OPCODES) through the
pc-driven emulator `run`, its main component also recorded with DecodingCheck's types B, U and J and the ten control-flow chips
(control=True); its program rows run many times or never, and FinalPrgMemoryCtr holds the counts.

The step record (`STEP_FIELDS`, one uint32 row per field, one column per step) is what the device fill (nb200_v1_main_trace for ADD / ADDI,
nb200_v1_alu_trace for the 19 ALU opcodes, nb200_v1_control_trace for all 29, csrc/v1_trace.{cu,cuh}) takes; `fill_main_trace` is its numpy
reference, a port of the per-row fills of CpuChip (cpu.rs:36-316), DecodingCheck R / I / I with a shift amount / B / U / J (type_r.rs:25-60,
type_i.rs:29-69,288-330, type_b.rs, type_u.rs, type_j.rs), AddChip (add.rs:64-100), SubChip, SltuChip, BitOpChip, SltChip, the branch chips,
JalChip, LuiChip, AuipcChip, JalrChip, SllChip, SrlChip, SraChip, ProgramMemCheck (program_mem_check.rs:44-100), RegisterMemCheck
(register_mem_check.rs:53-117) and Timestamp (timestamp.rs:33-75) for executed and padding rows."""
import numpy as np

from . import air as A
from . import nexus_v1 as V
from . import whole_machine as W

P = (1 << 31) - 1
ELF_TEXT_START = 136                       # PUBLIC_OUTPUT_ADDRESS_LOCATION + 4 (common/src/constants/mod.rs:8-10)
NUM_REGISTERS = 32
# the step record's opcode numbers (include/nb200.h): (mnemonic, instruction type, funct3, funct7, the main component's flag column);
# type "R" reads rs2, "I" takes a 12-bit immediate, "IShift" a 5-bit shift amount (SLLI / SRLI / SRAI, funct7 in the immediate's top bits)
OPCODES = [("ADD", "R", 0b000, 0, "IsAdd"), ("ADDI", "I", 0b000, 0, "IsAdd"), ("SUB", "R", 0b000, 0b0100000, "IsSub"),
           ("SLL", "R", 0b001, 0, "IsSll"), ("SLT", "R", 0b010, 0, "IsSlt"), ("SLTU", "R", 0b011, 0, "IsSltu"), ("XOR", "R", 0b100, 0, "IsXor"),
           ("SRL", "R", 0b101, 0, "IsSrl"), ("SRA", "R", 0b101, 0b0100000, "IsSra"), ("OR", "R", 0b110, 0, "IsOr"), ("AND", "R", 0b111, 0, "IsAnd"),
           ("SLTI", "I", 0b010, 0, "IsSlt"), ("SLTIU", "I", 0b011, 0, "IsSltu"), ("XORI", "I", 0b100, 0, "IsXor"), ("ORI", "I", 0b110, 0, "IsOr"),
           ("ANDI", "I", 0b111, 0, "IsAnd"), ("SLLI", "IShift", 0b001, 0, "IsSll"), ("SRLI", "IShift", 0b101, 0, "IsSrl"),
           ("SRAI", "IShift", 0b101, 0b0100000, "IsSra")]
(OP_ADD, OP_ADDI, OP_SUB, OP_SLL, OP_SLT, OP_SLTU, OP_XOR, OP_SRL, OP_SRA, OP_OR, OP_AND, OP_SLTI, OP_SLTIU, OP_XORI, OP_ORI, OP_ANDI,
 OP_SLLI, OP_SRLI, OP_SRAI) = range(len(OPCODES))
OP_TYPE = [ty for _n, ty, _f3, _f7, _flag in OPCODES]
R_TWIN = ["SLTU" if n == "SLTIU" else n if ty == "R" else n[:-1] for n, ty, _f3, _f7, _flag in OPCODES]   # what each opcode computes
# the step record, field by field (nb200_v1_main_trace's and nb200_v1_alu_trace's `steps`): op_c is rs2 for type R, the sign-extended
# 12-bit immediate for type I and the shift amount for SLLI / SRLI / SRAI, value_c is rs2's value or op_c; the three previous timestamps
# are those of the rs1 read, the rs2 read and the rd write (0 when the access does not happen); pc_ctr_prev is how often the instruction at
# pc was executed before
STEP_FIELDS = ["pc", "word", "opcode", "rd", "rs1", "op_c", "value_b", "value_c", "rd_prev", "ts1_prev", "ts2_prev", "ts3_prev", "pc_ctr_prev"]


# the control-flow opcodes, numbers 19-28 of the step record (include/nb200.h): (mnemonic, instruction type, funct3, the main component's
# flag column).  Their (opcode, rd, rs1, c) operands are the step record's: a branch's rd is its op_a (the instruction's rs1 field, read
# through Reg3) and its rs1 is its op_b (the instruction's rs2 field, read through Reg1), c the even offset in [-4096, 4094]; JAL's c is the
# even offset in [-2^20, 2^20 - 2] and its rs1 is 0; JALR's c is a 12-bit immediate as ADDI's; LUI's and AUIPC's c is the 20-bit
# immediate (ValueC = c << 12) and their rs1 is 0
CONTROL_OPCODES = [("BEQ", "B", 0b000, "IsBeq"), ("BNE", "B", 0b001, "IsBne"), ("BLT", "B", 0b100, "IsBlt"), ("BGE", "B", 0b101, "IsBge"),
                   ("BLTU", "B", 0b110, "IsBltu"), ("BGEU", "B", 0b111, "IsBgeu"), ("JAL", "J", 0, "IsJal"), ("JALR", "I", 0b000, "IsJalr"),
                   ("LUI", "U", 0, "IsLui"), ("AUIPC", "U", 0, "IsAuipc")]
(OP_BEQ, OP_BNE, OP_BLT, OP_BGE, OP_BLTU, OP_BGEU, OP_JAL, OP_JALR, OP_LUI, OP_AUIPC) = range(len(OPCODES), len(OPCODES) + len(CONTROL_OPCODES))
ALL_OPCODES = OPCODES + [(n, ty, f3, 0, flag) for n, ty, f3, flag in CONTROL_OPCODES]
ALL_OP_TYPE = [ty for _n, ty, _f3, _f7, _flag in ALL_OPCODES]
BRANCHES = [OP_BEQ, OP_BNE, OP_BLT, OP_BGE, OP_BLTU, OP_BGEU]
N_OPCODES = len(ALL_OPCODES)


def encode(op, rd, rs1, c):
    """The RV32I instruction word of opcode number `op` with rd, rs1 and c = rs2, the immediate or the shift amount (CONTROL_OPCODES: the
    step record's operands)."""
    if op >= len(OPCODES):
        return _encode_control(op, rd, rs1, c)
    _name, ty, f3, f7, _flag = OPCODES[op]
    if ty == "R":
        return (f7 << 25) | (c << 20) | (rs1 << 15) | (f3 << 12) | (rd << 7) | 0b0110011
    if ty == "I":
        return ((c & 0xFFF) << 20) | (rs1 << 15) | (f3 << 12) | (rd << 7) | 0b0010011
    return (f7 << 25) | ((c & 31) << 20) | (rs1 << 15) | (f3 << 12) | (rd << 7) | 0b0010011


def _encode_control(op, a, b, c):
    name, ty, f3, _flag = CONTROL_OPCODES[op - len(OPCODES)]
    if ty == "B":
        assert -4096 <= c < 4096 and c % 2 == 0
        i = c & 0x1FFF
        return (((i >> 12) & 1) << 31) | (((i >> 5) & 0x3F) << 25) | (b << 20) | (a << 15) | (f3 << 12) | (((i >> 1) & 0xF) << 8) \
            | (((i >> 11) & 1) << 7) | 0b1100011
    if ty == "J":
        assert -(1 << 20) <= c < 1 << 20 and c % 2 == 0 and b == 0
        i = c & 0x1FFFFF
        return (((i >> 20) & 1) << 31) | (((i >> 1) & 0x3FF) << 21) | (((i >> 11) & 1) << 20) | (((i >> 12) & 0xFF) << 12) | (a << 7) | 0b1101111
    if ty == "I":
        assert -2048 <= c < 2048
        return ((c & 0xFFF) << 20) | (b << 15) | (f3 << 12) | (a << 7) | 0b1100111
    assert 0 <= c < 1 << 20 and b == 0
    return (c << 12) | (a << 7) | (0b0110111 if name == "LUI" else 0b0010111)


def encode_beq(rs1, rs2, offset):
    return encode(OP_BEQ, rs1, rs2, offset)


def encode_bne(rs1, rs2, offset):
    return encode(OP_BNE, rs1, rs2, offset)


def encode_blt(rs1, rs2, offset):
    return encode(OP_BLT, rs1, rs2, offset)


def encode_bge(rs1, rs2, offset):
    return encode(OP_BGE, rs1, rs2, offset)


def encode_bltu(rs1, rs2, offset):
    return encode(OP_BLTU, rs1, rs2, offset)


def encode_bgeu(rs1, rs2, offset):
    return encode(OP_BGEU, rs1, rs2, offset)


def encode_jal(rd, offset):
    return encode(OP_JAL, rd, 0, offset)


def encode_jalr(rd, rs1, imm):
    return encode(OP_JALR, rd, rs1, imm)


def encode_lui(rd, imm20):
    return encode(OP_LUI, rd, 0, imm20)


def encode_auipc(rd, imm20):
    return encode(OP_AUIPC, rd, 0, imm20)


def encode_add(rd, rs1, rs2):
    return encode(OP_ADD, rd, rs1, rs2)


def encode_addi(rd, rs1, imm):
    return encode(OP_ADDI, rd, rs1, imm)


def encode_sub(rd, rs1, rs2):
    return encode(OP_SUB, rd, rs1, rs2)


def encode_sll(rd, rs1, rs2):
    return encode(OP_SLL, rd, rs1, rs2)


def encode_slt(rd, rs1, rs2):
    return encode(OP_SLT, rd, rs1, rs2)


def encode_sltu(rd, rs1, rs2):
    return encode(OP_SLTU, rd, rs1, rs2)


def encode_xor(rd, rs1, rs2):
    return encode(OP_XOR, rd, rs1, rs2)


def encode_srl(rd, rs1, rs2):
    return encode(OP_SRL, rd, rs1, rs2)


def encode_sra(rd, rs1, rs2):
    return encode(OP_SRA, rd, rs1, rs2)


def encode_or(rd, rs1, rs2):
    return encode(OP_OR, rd, rs1, rs2)


def encode_and(rd, rs1, rs2):
    return encode(OP_AND, rd, rs1, rs2)


def encode_slti(rd, rs1, imm):
    return encode(OP_SLTI, rd, rs1, imm)


def encode_sltiu(rd, rs1, imm):
    return encode(OP_SLTIU, rd, rs1, imm)


def encode_xori(rd, rs1, imm):
    return encode(OP_XORI, rd, rs1, imm)


def encode_ori(rd, rs1, imm):
    return encode(OP_ORI, rd, rs1, imm)


def encode_andi(rd, rs1, imm):
    return encode(OP_ANDI, rd, rs1, imm)


def encode_slli(rd, rs1, shamt):
    return encode(OP_SLLI, rd, rs1, shamt)


def encode_srli(rd, rs1, shamt):
    return encode(OP_SRLI, rd, rs1, shamt)


def encode_srai(rd, rs1, shamt):
    return encode(OP_SRAI, rd, rs1, shamt)


def add_chain_program(log_size, n_instructions=None):
    """The ADD chain's first `n_instructions` (default 2^log_size) instructions: (words uint32, [(opcode, rd, rs1, rs2 or imm)])."""
    n = (1 << log_size) if n_instructions is None else int(n_instructions)
    ops, (i, j, k) = [(OP_ADDI, 1, 0, 1)], (0, 1, 2)
    while len(ops) < n:
        ops.append((OP_ADD, k, j, i))
        i, j, k = (i + 1) % NUM_REGISTERS, (j + 1) % NUM_REGISTERS, (k + 1) % NUM_REGISTERS
    ops = ops[:n]
    words = np.array([encode(*op) for op in ops], np.uint32)
    return words, ops


# alu_program's fixed prefix: registers driven through 0, 1, -1, 0x7FFFFFFF and 0x80000000, then the edge cases of each instruction
ALU_PREFIX = [
    (OP_ADDI, 1, 0, 1), (OP_ADDI, 2, 0, -1), (OP_SRLI, 3, 2, 1), (OP_SLLI, 4, 1, 31), (OP_ADDI, 5, 0, 0),   # x1..x5 = 1, -1, max, min, 0
    (OP_SLT, 6, 3, 3), (OP_SLTU, 7, 4, 4), (OP_SLT, 8, 4, 3), (OP_SLTU, 9, 3, 4), (OP_SLT, 10, 2, 5),     # equal operands, both signs
    (OP_SRA, 11, 4, 2), (OP_SRAI, 12, 4, 31), (OP_SRL, 13, 2, 5), (OP_SLLI, 14, 2, 0), (OP_SLL, 15, 3, 2),  # rs2 = -1: bits above 4 set
    (OP_ADDI, 16, 0, 33), (OP_SLL, 17, 3, 16), (OP_SRL, 18, 4, 16), (OP_SRA, 19, 4, 16),                 # rs2 = 33: shift by 1
    (OP_ADDI, 20, 3, -2048), (OP_SLTIU, 21, 2, -2048), (OP_SLTI, 22, 4, -2048), (OP_SLTIU, 23, 5, 1),    # immediate -2048, seqz
    (OP_XORI, 24, 3, -1), (OP_ORI, 25, 4, -2048), (OP_ANDI, 26, 2, -2048), (OP_SLTI, 27, 1, 1),
    (OP_SUB, 28, 4, 1), (OP_SUB, 29, 0, 4), (OP_SUB, 30, 5, 2), (OP_ADD, 31, 3, 1),                      # min - 1, -min, 0 - (-1), max + 1
    (OP_XOR, 1, 3, 4), (OP_OR, 2, 4, 5), (OP_AND, 3, 2, 4), (OP_SRAI, 4, 3, 31),
    (OP_ADD, 0, 2, 2), (OP_XOR, 0, 3, 4), (OP_SRAI, 0, 2, 31), (OP_SLTU, 0, 0, 2),                       # writes to x0
]
IMM_EDGES = [-2048, -2047, -1, 0, 1, 2, 15, 16, 255, 256, 2046, 2047]


def alu_program(log_size, n_instructions=None, seed=0):
    """A seeded straight-line program of `n_instructions` (default 2^log_size) instructions over all 19 opcodes: ALU_PREFIX, then each
    instruction drawn uniformly with random registers, immediates (a quarter of them from IMM_EDGES) and shift amounts.
    (words uint32, [(opcode, rd, rs1, rs2 / imm / shift amount)])."""
    n = (1 << log_size) if n_instructions is None else int(n_instructions)
    rng = np.random.default_rng(seed)
    m = max(0, n - len(ALU_PREFIX))
    op = rng.integers(0, len(OPCODES), m)
    rd, rs1, rs2 = (rng.integers(0, NUM_REGISTERS, m) for _ in range(3))
    imm = np.where(rng.integers(0, 4, m) == 0, np.array(IMM_EDGES)[rng.integers(0, len(IMM_EDGES), m)], rng.integers(-2048, 2048, m))
    shamt = rng.integers(0, 32, m)
    c = np.select([np.array(OP_TYPE)[op] == "R", np.array(OP_TYPE)[op] == "I"], [rs2, imm], shamt)
    ops = (ALU_PREFIX + [tuple(int(x) for x in row) for row in zip(op, rd, rs1, c)])[:n]
    return np.array([encode(*o) for o in ops], np.uint32), ops


def alu(op, b, c):
    """RV32I's result of opcode number `op` on the u32 operands b and c (rs2's value, the sign-extended immediate or the shift amount)."""
    sb, sc, sh = b - ((b >> 31) << 32), c - ((c >> 31) << 32), c & 31
    r = {"ADD": b + c, "SUB": b - c, "SLL": b << sh, "SLT": int(sb < sc), "SLTU": int(b < c), "XOR": b ^ c, "SRL": b >> sh, "SRA": sb >> sh,
         "OR": b | c, "AND": b & c}[R_TWIN[op]]
    return r & 0xFFFFFFFF


def execute(ops, base=ELF_TEXT_START):
    """Run a straight-line program of the 19 opcodes once from the all-zero register file.  Returns (steps, final registers) where steps is
    (len(STEP_FIELDS), n_steps) uint32 in STEP_FIELDS order and final registers = (values, timestamps) of the 32 registers after the last
    step (FinalReg's rows).  Step t (clk = t + 1) reads rs1 at 3 clk + 1, rs2 at 3 clk + 2 and writes rd at 3 clk + 3 (preprocessed.rs:75-100);
    a write to x0 stores 0 (ValueAEffective)."""
    val, ts = [0] * NUM_REGISTERS, [0] * NUM_REGISTERS
    pc_ctr = {}
    cols = [[] for _ in STEP_FIELDS]
    for t, (op, rd, rs1, c) in enumerate(ops):
        assert 0 <= op < len(OPCODES) and 0 <= rd < 32 and 0 <= rs1 < 32
        word = encode(op, rd, rs1, c)
        clk = t + 1
        pc = base + 4 * t
        b, ts1 = val[rs1], ts[rs1]
        ts[rs1] = 3 * clk + 1
        if OP_TYPE[op] == "R":
            assert 0 <= c < 32
            cv, ts2 = val[c], ts[c]
            ts[c] = 3 * clk + 2
            op_c = c
        elif OP_TYPE[op] == "I":
            op_c = (c & 0xFFF) - ((c & 0x800) << 1) & 0xFFFFFFFF                # the 12-bit immediate, sign-extended
            cv, ts2 = op_c, 0
        else:
            assert 0 <= c < 32
            op_c = cv = c
            ts2 = 0
        a = alu(op, b, cv)
        rd_prev, ts3 = val[rd], ts[rd]
        val[rd], ts[rd] = (a if rd else 0), 3 * clk + 3
        ctr = pc_ctr.get(pc, 0)
        pc_ctr[pc] = ctr + 1
        for col, v in zip(cols, (pc, word, op, rd, rs1, op_c, b, cv, rd_prev, ts1, ts2, ts3, ctr)):
            col.append(v)
    steps = np.array(cols, dtype=np.uint32).reshape(len(STEP_FIELDS), len(ops))
    return steps, (np.array(val, np.uint32), np.array(ts, np.uint32))


def _sext(x, bits):
    x &= (1 << bits) - 1
    return x - ((x >> (bits - 1)) << bits)


def _taken(op, a, b):
    """Whether branch opcode `op` is taken on op_a's value a and op_b's value b (u32)."""
    sa, sb = _sext(a, 32), _sext(b, 32)
    return {OP_BEQ: a == b, OP_BNE: a != b, OP_BLT: sa < sb, OP_BGE: sa >= sb, OP_BLTU: a < b, OP_BGEU: a >= b}[op]


def run(ops, n_steps, base=ELF_TEXT_START):
    """Execute the program `ops` = [(opcode, rd, rs1, c)] over all 29 opcodes (OPCODES, CONTROL_OPCODES), laid out from `base`, for exactly
    n_steps steps from pc = base and the all-zero register file.  Returns (steps, final registers, final_ctr) as `execute` does, final_ctr
    being how often each program row ran (0 for a row that never ran).  A branch reads op_b through Reg1 and op_a through Reg3 (which
    writes its value back); JAL, LUI and AUIPC read no register.  Raises ValueError when pc leaves the program or is not 4-aligned."""
    words = [encode(*o) for o in ops]
    val, ts = [0] * NUM_REGISTERS, [0] * NUM_REGISTERS
    final_ctr = np.zeros(len(ops), np.uint32)
    cols = [[] for _ in STEP_FIELDS]
    pc = base
    for t in range(n_steps):
        row, off = divmod(pc - base, 4)
        if off or not 0 <= row < len(ops):
            raise ValueError(f"step {t}: pc {pc:#x} is outside the program or not 4-aligned")
        op, rd, rs1, c = ops[row]
        assert 0 <= op < N_OPCODES and 0 <= rd < 32 and 0 <= rs1 < 32
        ty, clk = ALL_OP_TYPE[op], t + 1
        b = ts1 = ts2 = 0
        if ty not in ("J", "U"):                                              # Reg1: rs1, or a branch's op_b
            b, ts1 = val[rs1], ts[rs1]
            ts[rs1] = 3 * clk + 1
        nxt = pc + 4
        if ty == "R":
            assert 0 <= c < 32
            cv, ts2 = val[c], ts[c]
            ts[c] = 3 * clk + 2
            op_c = c
        elif ty == "I":
            op_c = cv = _sext(c, 12) & 0xFFFFFFFF
        elif ty == "IShift":
            assert 0 <= c < 32
            op_c = cv = c
        elif ty == "B":
            op_c = cv = c & 0xFFFFFFFF
        elif ty == "J":
            op_c = cv = c & 0xFFFFFFFF
        else:
            op_c, cv = c, (c << 12) & 0xFFFFFFFF
        rd_prev, ts3 = val[rd], ts[rd]
        if op < len(OPCODES):
            a = alu(op, b, cv)
        elif ty == "B":
            a = rd_prev
            if _taken(op, rd_prev, b):
                nxt = pc + cv
        elif op == OP_JAL:
            a, nxt = pc + 4, pc + cv
        elif op == OP_JALR:
            a, nxt = pc + 4, (b + cv) & 0xFFFFFFFE
        else:
            a = cv if op == OP_LUI else pc + cv
        a &= 0xFFFFFFFF
        val[rd], ts[rd] = (a if rd else 0), 3 * clk + 3
        for col, v in zip(cols, (pc, words[row], op, rd, rs1, op_c, b, cv, rd_prev, ts1, ts2, ts3, final_ctr[row])):
            col.append(v)
        final_ctr[row] += 1
        pc = nxt & 0xFFFFFFFF
    steps = np.array(cols, dtype=np.uint32).reshape(len(STEP_FIELDS), n_steps)
    return steps, (np.array(val, np.uint32), np.array(ts, np.uint32)), final_ctr


# control_program's fixed prefix (runs once): registers driven through 1, -1, 0x7FFFFFFF, 0x80000000, 0, equal halves, then every branch on
# each operand pair with a marker instruction it skips when taken, the extreme offsets (not taken), a backward counted branch, JAL forward
# and backward with rd = x0 and not, JALR to an odd target and with rd == rs1, LUI 0xFFFFF / 0, AUIPC with negative immediates and each
# ALU opcode once
def _control_prefix():
    ops = [(OP_ADDI, 1, 0, 1), (OP_ADDI, 2, 0, -1), (OP_SRLI, 3, 2, 1), (OP_SLLI, 4, 1, 31), (OP_ADDI, 5, 0, 0), (OP_ADDI, 6, 0, 1),
           (OP_LUI, 8, 0, 0x10), (OP_LUI, 9, 0, 0xFFFFF), (OP_LUI, 10, 0, 0), (OP_ADDI, 9, 9, 0x7FF)]   # x8 = 0x10000, x9 = 0xFFFFF7FF
    pairs = [(1, 6), (5, 2), (2, 5), (3, 4), (4, 3), (8, 5), (1, 5), (9, 2), (3, 3), (0, 5), (5, 0)]
    for op in BRANCHES:
        for a, b in pairs:
            ops += [(op, a, b, 8), (OP_ADDI, 7, 7, 1)]
    ops += [(OP_BNE, 1, 6, 4094), (OP_BEQ, 1, 5, -4096), (OP_BLTU, 2, 1, -4096), (OP_BLT, 3, 4, 4094)]
    ops += [(OP_ADDI, 11, 0, 3), (OP_ADDI, 11, 11, -1), (OP_BNE, 11, 0, -4)]                   # a backward branch, taken twice
    ops += [(OP_JAL, 0, 0, 8), (OP_JAL, 12, 0, 8), (OP_JAL, 13, 0, -4), (OP_ADDI, 7, 7, 100)]  # JAL forward (x0), backward (x13), forward (x12)
    ops += [(OP_AUIPC, 14, 0, 0), (OP_JALR, 15, 14, 13), (OP_ADDI, 7, 7, 1000)]                # JALR to an odd target: bit 0 cleared
    ops += [(OP_AUIPC, 16, 0, 0), (OP_JALR, 16, 16, 12), (OP_ADDI, 7, 7, 1000)]                # JALR with rd == rs1
    ops += [(OP_AUIPC, 17, 0, 0xFFFFF), (OP_AUIPC, 18, 0, 0x80000), (OP_LUI, 19, 0, 0xFFFFF), (OP_LUI, 0, 0, 0x12345)]
    ops += [(k, 20 + k % 8, 1 + k % 5, 1 + k % 4 if OP_TYPE[k] == "R" else k) for k in range(len(OPCODES))]   # every ALU opcode once
    return ops


def control_program(log_size, n_steps=None, seed=0):
    """A looping program over all 29 opcodes: the fixed prefix (_control_prefix), then a seeded body of random ALU instructions (registers
    x1..x27) among forward branches on random registers, a counted inner loop (counter x28) and a call of a function through JAL / JALR
    (link x29), the body closed by a JAL back to its first instruction so that any number of steps is valid.  The body has max(64,
    2^log_size / 16) instructions.  Returns (words uint32, [(opcode, rd, rs1, c)], n_steps), n_steps defaulting to 2^log_size."""
    n_steps = (1 << log_size) if n_steps is None else int(n_steps)
    rng = np.random.default_rng(seed)
    ops = _control_prefix()
    body = len(ops)

    def random_alu():
        op = int(rng.integers(0, len(OPCODES)))
        ty = OP_TYPE[op]
        c = int(rng.integers(0, 28)) if ty == "R" else int(rng.integers(-2048, 2048)) if ty == "I" else int(rng.integers(0, 32))
        return (op, int(rng.integers(1, 28)), int(rng.integers(0, 28)), c)

    n_body = max(64, (1 << log_size) // 16)
    call_at = body + n_body // 2
    while len(ops) < body + n_body:
        k = int(rng.integers(0, 16))
        if k == 0:
            ops += [(int(rng.choice(BRANCHES)), int(rng.integers(0, 28)), int(rng.integers(0, 28)), 4 * int(rng.integers(2, 4)))]
        elif k == 1:
            n = int(rng.integers(1, 4))
            ops += [(OP_ADDI, 28, 0, int(rng.integers(2, 6)))] + [random_alu() for _ in range(n)]
            ops += [(OP_ADDI, 28, 28, -1), (OP_BNE, 28, 0, -4 * (n + 1))]
        elif len(ops) >= call_at:
            ops += [("call",)]
            call_at = 1 << 62
        else:
            ops.append(random_alu())
    ops = ops[:body + n_body] + [random_alu() for _ in range(3)]
    ops.append((OP_JAL, 0, 0, -4 * (len(ops) - body)))
    func = len(ops)
    ops += [random_alu(), random_alu(), (OP_LUI, 30, 0, int(rng.integers(0, 1 << 20))), (OP_JALR, 0, 29, 0)]
    ops = [(OP_JAL, 29, 0, 4 * (func - i)) if o == ("call",) else o for i, o in enumerate(ops)]
    assert ("call",) not in ops
    return np.array([encode(*o) for o in ops], np.uint32), ops, n_steps


def _le(x, k=4):
    x = np.asarray(x, dtype=np.uint64)
    return [((x >> np.uint64(8 * i)) & np.uint64(255)).astype(np.uint32) for i in range(k)]


def _carries16(x, y):
    """The carries out of the low and the high 16 bits of x + y (the limbs 1 and 3 of add_with_carries, add.rs:27-45)."""
    x, y = np.asarray(x, np.uint64), np.asarray(y, np.uint64)
    lo = (x & 0xFFFF) + (y & 0xFFFF)
    c0 = lo >> 16
    c1 = ((x >> 16) + (y >> 16) + c0) >> 16
    return [c0.astype(np.uint32), c1.astype(np.uint32)]


def _borrows16(x, y):
    """The borrows out of the low and the high 16 bits of x - y (subtract_with_borrow's limbs 1 and 3, sub.rs:26-63)."""
    x, y = np.asarray(x, np.uint64), np.asarray(y, np.uint64)
    return [((x & 0xFFFF) < (y & 0xFFFF)).astype(np.uint32), (x < y).astype(np.uint32)]


def _signed(x):
    x = np.asarray(x, np.uint64).astype(np.int64)
    return x - ((x >> 31) << 32)


def alu_np(op, b, c):
    """`alu` over arrays: the u32 results of the opcode numbers `op` on the operands b and c."""
    b, c = np.asarray(b, np.uint64), np.asarray(c, np.uint64)
    sh = c & np.uint64(31)
    sb, sc = _signed(b), _signed(c)
    by_name = {"ADD": b + c, "SUB": b - c, "SLL": b << sh, "SLT": (sb < sc).astype(np.uint64), "SLTU": (b < c).astype(np.uint64),
               "XOR": b ^ c, "SRL": b >> sh, "SRA": (sb >> sh.astype(np.int64)).astype(np.uint64), "OR": b | c, "AND": b & c}
    return np.select([op == k for k in range(len(OPCODES))], [by_name[n] for n in R_TWIN], 0) & np.uint64(0xFFFFFFFF)


def _inv_m31(x):
    """x^(P-2) mod P elementwise: the inverse in M31 of each nonzero x < P."""
    x, r = np.asarray(x, np.uint64) % np.uint64(P), None
    e, p2 = P - 2, None
    while e:
        p2 = x if p2 is None else (p2 * p2) % np.uint64(P)
        if e & 1:
            r = p2 if r is None else (r * p2) % np.uint64(P)
        e >>= 1
    return r


def main_columns(steps, final_ctr, log_size):
    """The main component's 347 columns in trace order ({column name: its limbs}) for the step record `steps` (rows past n_steps are padding
    rows) and the final access counters of the program's rows (FinalPrgMemoryCtr)."""
    n = 1 << log_size
    s = {f: np.asarray(steps[i], np.uint64) for i, f in enumerate(STEP_FIELDS)}
    m = s["pc"].size
    assert m <= n and len(final_ctr) <= n
    t = {name: [np.zeros(n, np.uint32) for _ in range(size)] for name, size in V.MAIN_COLUMNS}

    def put(name, limbs, rows=slice(0, m)):
        for dst, v in zip(t[name], limbs):
            dst[rows] = v

    def put_on(ops, name, limbs):
        """Write `limbs` (arrays over the steps) on the steps whose opcode is in `ops` only."""
        rows = np.nonzero(np.isin(op, ops))[0]
        for dst, v in zip(t[name], limbs):
            dst[rows] = np.broadcast_to(np.asarray(v, np.uint64), (m,))[rows]

    op = s["opcode"]
    ty = np.array(ALL_OP_TYPE)[op.astype(np.int64)]
    is_r, is_i, is_shift, is_b, is_j, is_u = (ty == k for k in ("R", "I", "IShift", "B", "J", "U"))
    rd, rs1, b, c = s["rd"], s["rs1"], s["value_b"], s["value_c"]
    pc, mask = s["pc"], np.uint64(0xFFFFFFFF)
    # ValueA: the ALU result; a branch's op_a value (read through Reg3 and written back), the link pc + 4, LUI's ValueC, AUIPC's pc + ValueC
    a = np.select([is_b, np.isin(op, [OP_JAL, OP_JALR]), op == OP_LUI, op == OP_AUIPC],
                  [s["rd_prev"], (pc + 4) & mask, c, (pc + c) & mask], alu_np(op, b, c))
    sa, sb = _signed(a), _signed(b)
    taken = np.select([op == k for k in BRANCHES], [a == b, a != b, sa < sb, sa >= sb, a < b, a >= b], False)
    pc_next = np.select([taken | (op == OP_JAL), op == OP_JALR], [(pc + c) & mask, (b + c) & np.uint64(0xFFFFFFFE)], (pc + 4) & mask)
    flag = (rd != 0).astype(np.uint32)
    # CpuChip (cpu.rs:36-316)
    put("IsPadding", [np.zeros(m, np.uint32)])
    t["IsPadding"][0][m:] = 1
    put("ValueAEffectiveFlag", [flag])
    inv = np.array([1] + [pow(r, P - 2, P) for r in range(1, 32)], np.uint64)
    t["ValueAEffectiveFlagAux"][0][:] = 1
    t["ValueAEffectiveFlagAuxInv"][0][:] = 1
    put("ValueAEffectiveFlagAux", [np.where(rd != 0, inv[rd.astype(np.int64) % 32], 1)])
    put("ValueAEffectiveFlagAuxInv", [np.where(rd != 0, rd, 1)])
    put("Pc", _le(s["pc"]))
    put("PcCarry", _carries16(s["pc"], 4))
    put("PcNext", _le(pc_next))
    put("InstrVal", _le(s["word"]))
    for name in dict.fromkeys(f for _n, _ty, _f3, _f7, f in ALL_OPCODES):
        put(name, [np.isin(op, [k for k, o in enumerate(ALL_OPCODES) if o[4] == name]).astype(np.uint32)])
    put("ValueB", _le(b))
    put("ValueC", _le(c))
    put("OpA", [rd])
    put("OpB", [rs1])
    put("OpC", [np.select([is_i, is_b, is_j], [s["op_c"] & 0xFFF, s["op_c"] & 0x1FFF, s["op_c"] & 0x1FFFFF], s["op_c"])])
    put("ImmC", [(~is_r).astype(np.uint32)])
    put("Reg1Address", [rs1])
    put("Reg2Address", [np.where(is_r, s["op_c"], 0)])
    put("Reg3Address", [rd])
    # DecodingCheck, types R, I without and I with a shift amount: type_r.rs:43-59, type_i.rs:46-68 and 288-330; types B, U and J:
    # type_b.rs:33-73, type_u.rs:29-51, type_j.rs:29-62
    oc = s["op_c"]
    r_or_i = is_r | is_i | is_shift
    put("OpA0", [rd & 1]); put("OpA1_4", [(rd >> 1) & 0xF])
    put("OpB0", [np.where(r_or_i, rs1 & 1, 0)]); put("OpB1_4", [np.where(r_or_i, (rs1 >> 1) & 0xF, 0)])
    put("OpC0_3", [np.where(r_or_i, oc & 0xF, 0)])
    put("OpC4", [np.where(is_r | is_shift, (oc >> 4) & 1, 0)])
    put("OpC4_7", [np.where(is_i | is_j, (oc >> 4) & 0xF, 0)])
    put("OpC8_10", [np.where(is_i | is_b | is_j, (oc >> 8) & 0x7, 0)])
    put("OpC11", [np.where(is_i | is_b | is_j, (oc >> 11) & 1, 0)])
    put("OpC1_4", [np.where(is_b, (oc >> 1) & 0xF, 0)])
    put("OpC5_7", [np.where(is_b, (oc >> 5) & 0x7, 0)])
    put("OpC12", [np.where(is_b, (oc >> 12) & 1, 0)])
    put("OpB0_3", [np.where(is_b, rs1 & 0xF, 0)])
    put("OpB4", [np.where(is_b, rs1 >> 4, 0)])
    put("OpC1_3", [np.where(is_j, (oc >> 1) & 0x7, 0)])
    put("OpC12_15", [np.select([is_j, is_u], [(oc >> 12) & 0xF, oc & 0xF], 0)])
    put("OpC16_19", [np.where(is_j, (oc >> 16) & 0xF, 0)])
    put("OpC20", [np.where(is_j, (oc >> 20) & 1, 0)])
    put("OpC16_23", [np.where(is_u, (oc >> 4) & 0xFF, 0)])
    put("OpC24_31", [np.where(is_u, (oc >> 12) & 0xFF, 0)])
    # the instruction chips: ValueA = the result, and each chip's helpers on its own rows
    put("ValueA", _le(a))
    put_on([OP_ADD, OP_ADDI], "CarryFlag", _carries16(b, c))                        # AddChip (add.rs:64-100)
    slt, sltu = [OP_SLT, OP_SLTI], [OP_SLTU, OP_SLTIU]
    put_on([OP_SUB] + slt + sltu, "CarryFlag", _borrows16(b, c))                     # SubChip (sub.rs:66-100), and CarryFlag as the borrows
    put_on(slt + sltu, "Helper1", _le((b - c) & 0xFFFFFFFF))                         # SltuChip (sltu.rs:45-75), SltChip (slt.rs:56-110)
    put_on(slt, "Helper2", _le(b & 0x7FFFFFFF))
    put_on(slt, "Helper3", _le(c & 0x7FFFFFFF))
    put_on(slt, "SgnC", [c >> 31])
    bit_ops = [OP_XOR, OP_OR, OP_AND, OP_XORI, OP_ORI, OP_ANDI]                      # BitOpChip (bit_op.rs:249-300): the high nibbles
    for name, v in (("ValueA4_7", a), ("ValueB4_7", b), ("ValueC4_7", c)):
        put_on(bit_ops, name, [x >> 4 for x in _le(v)])
    # SllChip, SrlChip, SraChip (sll.rs:72-112, srl.rs:79-119, sra.rs:93-139): the shift amount's bits from ValueC's low byte, Exp1_3 = 2^(its
    # low three bits); SLL multiplies ValueB by Exp1_3 byte by byte (Rem, carries Qt), SRL / SRA divide it from the top byte (quotients Qt
    # = the bytes of b >> those bits, remainders Rem)
    sll, srl, sra = [OP_SLL, OP_SLLI], [OP_SRL, OP_SRLI], [OP_SRA, OP_SRAI]
    c0 = c & 0xFF
    e = np.uint64(1) << (c0 & 7)
    put_on(sll + srl + sra, "Helper1", [c0 >> 5, 0, 0, 0])
    for k in range(5):
        put_on(sll + srl + sra, f"ShiftBit{k + 1}", [(c0 >> k) & 1])
    put_on(sll + srl + sra, "Exp1_3", [e])
    put_on(sll, "Rem", _le((b * e) & 0xFFFFFFFF))
    put_on(sll, "Qt", [((b & ((1 << (8 * i + 8)) - 1)) * e) >> (8 * i + 8) for i in range(4)])
    rem = [x & (e - 1) for x in _le(b)]
    put_on(srl + sra, "Rem", rem)
    put_on(srl + sra, "Qt", _le(b >> (c0 & 7)))
    put_on(srl + sra, "RemDiff", [e - 1 - r for r in rem])
    sgn_b = b >> 31
    exp = np.uint64(256) // e
    put_on(sra, "Helper2", [(b >> 24) & 0x7F, 0, 0, 0])
    put_on(sra, "Helper3", _le(b >> (c & 31)))
    put_on(slt + sra, "SgnB", [sgn_b])
    put_on(sra, "Exp", [exp])
    put_on(sra, "SraDegreeAux", [sgn_b * (e - 1) * exp])
    # the branch chips (beq.rs:34-104, bne.rs, bltu.rs:28-55, blt.rs:38-86, bgeu.rs, bge.rs): CarryFlag = the carries of PcNext = Pc +
    # (ValueC or 4); BEQ / BNE: the halves' inequality flags and their aux / inverse pairs, the fallback pair from pc's halves read
    # big-endian (u16::from_be_bytes, beq.rs:41-42); the others: Helper1 = ValueA - ValueB with BorrowFlag its borrows, BLT / BGE's Helper2 /
    # Helper3 = ValueA / ValueB without the sign bit, LtFlag the signed comparison, BGE's SgnA / SgnB
    put_on(BRANCHES, "CarryFlag", _carries16(pc, np.where(taken, c, 4)))
    eq_ops, cmp_ops, lt_ops = [OP_BEQ, OP_BNE], [OP_BLT, OP_BGE, OP_BLTU, OP_BGEU], [OP_BLT, OP_BGE]
    put_on(eq_ops, "Neq", [(a != b).astype(np.uint32)])
    pc_be = [((pc >> np.uint64(16 * k)) & 0xFF) * 256 + ((pc >> np.uint64(16 * k + 8)) & 0xFF) for k in (0, 1)]
    for k, name in enumerate(("Neq12", "Neq34")):
        ah, bh = (a >> np.uint64(16 * k)) & 0xFFFF, (b >> np.uint64(16 * k)) & 0xFFFF
        aux_inv = np.where(ah != bh, (ah + P - bh) % P, np.maximum(pc_be[k], 1))
        put_on(eq_ops, name, [(ah != bh).astype(np.uint32)])
        put_on(eq_ops, name + "Aux", [_inv_m31(aux_inv)])
        put_on(eq_ops, name + "AuxInv", [aux_inv])
    put_on(cmp_ops, "Helper1", _le((a - b) & mask))
    put_on(cmp_ops, "BorrowFlag", _borrows16(a, b))
    put_on(lt_ops, "Helper2", _le(a & 0x7FFFFFFF))
    put_on(lt_ops, "Helper3", _le(b & 0x7FFFFFFF))
    put_on(lt_ops, "LtFlag", [(sa < sb).astype(np.uint32)])
    put_on([OP_BGE], "SgnA", [a >> 31])
    put_on([OP_BGE], "SgnB", [b >> 31])
    # JalChip (jal.rs:33-73), JalrChip (jalr.rs:38-101), AuipcChip (auipc.rs:33-62): CarryFlag = the carries of ValueA = Pc + 4 (Pc +
    # ValueC for AUIPC); BorrowFlag = those of JAL's PcNext = Pc + ValueC and JALR's PcNextAux = ValueB + ValueC, whose bit 0 is RemAux and
    # whose low byte less it is 2 QtAux
    put_on([OP_JAL, OP_JALR], "CarryFlag", _carries16(pc, 4))
    put_on([OP_AUIPC], "CarryFlag", _carries16(pc, c))
    put_on([OP_JAL], "BorrowFlag", _carries16(pc, c))
    put_on([OP_JALR], "BorrowFlag", _carries16(b, c))
    put_on([OP_JALR], "PcNextAux", _le((b + c) & mask))
    put_on([OP_JALR], "RemAux", [(b + c) & 1])
    put_on([OP_JALR], "QtAux", [((b + c) & 0xFF) >> 1])
    # ProgramMemCheck (program_mem_check.rs:44-100): the counters of this access; FinalPrgMemoryCtr on the program's rows
    put("ProgCtrPrev", _le(s["pc_ctr_prev"]))
    put("ProgCtrCur", _le(s["pc_ctr_prev"] + 1))
    put("ProgCtrCarry", _carries16(s["pc_ctr_prev"], 1))
    put("FinalPrgMemoryCtr", _le(final_ctr), slice(0, len(final_ctr)))
    # RegisterMemCheck (register_mem_check.rs:53-117): ValueAEffective and the previous values / timestamps of the accessed registers
    put("ValueAEffective", _le(a * flag))
    put("Reg1ValPrev", _le(b))
    put("Reg2ValPrev", _le(np.where(is_r, c, 0)))
    put("Reg3ValPrev", _le(s["rd_prev"]))
    for k in (1, 2, 3):
        put(f"Reg{k}TsPrev", _le(s[f"ts{k}_prev"]))
    # Timestamp (timestamp.rs:33-75), every row: c = cur - 1 - prev with the borrows out of the low and high 16 bits
    clk = np.arange(1, n + 1, dtype=np.uint64)
    for k in (1, 2, 3):
        cur = 3 * clk + k
        prev = np.zeros(n, np.uint64)
        prev[:m] = s[f"ts{k}_prev"]
        assert np.all(prev < cur)
        cc = cur - 1 - prev
        b0 = ((cur & 0xFFFF) < (prev & 0xFFFF) + 1).astype(np.uint32)
        t[f"CReg{k}TsPrev"] = _le(cc)
        t[f"CH{k}Minus"] = [b0, np.zeros(n, np.uint32)]
    return t


def _count(hist, values, weights=None):
    """Add each value to the histogram, with its numerator when `weights` are given (rows of numerator 0 look nothing up)."""
    v = np.asarray(values, np.int64)
    if weights is None:
        hist += np.bincount(v, minlength=hist.size)
    else:
        keep = weights != 0
        hist += np.bincount(v[keep], weights[keep], minlength=hist.size).astype(np.int64)


def table_counts(t, ram_cols):
    """The multiplicities of BitOp (And, Or, Xor: one per row b nibble * 16 + c nibble), Range8, 16, 32, 128, 256 as the main component's
    lookups (nexus_v1.record_main_component's bit-op lookups and range checks with their numerators, the instruction types B, J and U and
    JALR's among them) and RamInitFinal's nine Range256 lookups per row count them."""
    h = {r: np.zeros(length, np.int64) for r, length, _ls in W.MULTIPLICITY_TABLES}
    f = lambda *names: sum(t[nm][0].astype(np.int64) for nm in names)
    imm_c = f("ImmC")
    vtype = {"R": (1 - imm_c) * f(*V.TYPE_R_OPS), "INoShift": imm_c * f(*V.ALU_IMM_NO_SHIFT) + f("IsJalr"), "IShift": imm_c * f(*V.ALU_IMM_SHIFT),
             "B": f(*V.IS_TYPE_B), "J": f("IsJal"), "U": f(*V.IS_TYPE_U)}
    for w in V.R256_WORDS + V.R256_HALF_WORDS + V.R256_BYTES:
        for limb in t[w]:
            _count(h["Range256"], limb)
    for w in V.R256_TYPE_U_BYTES:
        _count(h["Range256"], t[w][0], vtype["U"])
    for v in ram_cols[[0, 1, 2, 3, 5, 6, 7, 8, 9]]:
        _count(h["Range256"], v)
    for w in V.R32:
        _count(h["Range32"], t[w][0])
    for ty, names in V.R16:
        for nm in names:
            if ty in vtype:
                _count(h["Range16"], t[nm][0], vtype[ty])
    for ty, names in V.R8:
        for nm in names:
            if ty in vtype:
                _count(h["Range8"], t[nm][0], vtype[ty])
    _count(h["Range8"], t["Helper1"][0], f(*V.ALU_IMM_SHIFT))
    for nm in ("Helper2", "Helper3"):
        _count(h["Range128"], t[nm][3], f("IsSlt", "IsBge", "IsBlt"))
    _count(h["Range128"], t["QtAux"][0], f("IsJalr"))
    _count(h["Range128"], t["Helper2"][0], f("IsSra"))
    h["BitOp"] = [np.zeros(256, np.int64) for _ in range(3)]
    for hist, flag in zip(h["BitOp"], ("IsAnd", "IsOr", "IsXor")):
        for k in range(4):
            b_hi, c_hi = t["ValueB4_7"][k].astype(np.int64), t["ValueC4_7"][k].astype(np.int64)
            b_lo, c_lo = t["ValueB"][k] - 16 * b_hi, t["ValueC"][k] - 16 * c_hi
            _count(hist, b_lo * 16 + c_lo, f(flag))
            _count(hist, b_hi * 16 + c_hi, f(flag))
    return h


class AddChainMachine:
    """The ADD chain of the module docstring at 2^log_size rows, `n_steps` executed steps (default 2^log_size); `ops` = [(opcode, rd, rs1,
    rs2 or imm)] runs another straight-line program instead.  Same interface as the other
    machines: `air`, `words`, `relations`, `log_sizes`, `preprocessed_columns()`, `fill_main_trace()` (tree 1 in commitment order, the
    multiplicity columns counted on the host), `column_log_sizes()`, and `device_trees(ctx)` (the main trace filled on the device by
    nb200_v1_main_trace, the multiplicities counted there)."""
    ALU = False                                          # record_main_component's `alu`: the machine constrains SLT, SLTU and the shifts
    CONTROL = False                                      # record_main_component's `control`: branches, jumps, LUI and AUIPC

    def __init__(self, log_size, n_steps=None, ops=None):
        assert log_size >= 8
        self.log_size = self.log_size_main = log_size
        if ops is None:
            self.n_steps = (1 << log_size) if n_steps is None else int(n_steps)
            self.program, ops = self.default_program(log_size, self.n_steps)
        else:                                                                 # another straight-line program
            self.n_steps = len(ops)
        assert 1 <= self.n_steps <= 1 << log_size
        self.steps, (self.final_values, self.final_timestamps) = execute(ops)
        self.program = self.steps[STEP_FIELDS.index("word")].copy()
        # every instruction runs once: the final counter of each program row (program_mem_check.rs:88-99)
        self.final_ctr = np.ones(self.program.size, np.uint32)
        self._record(log_size)

    def _record(self, log_size):
        """Record the nine components and the relations at 2^log_size main rows."""
        self.ram_log_size = W.ram_log_size(0)
        air = A.Air()
        names = [("BitOp", 4), ("LoadStore", 5), ("ProgramCheck", 8), ("RegisterCheck", 9), ("Range8", 1), ("Range16", 1), ("Range32", 1),
                 ("Range128", 1), ("Range256", 1)]
        self.relations = [air.relation(n, s) for n, s in names]
        rel = {r.name: r for r in self.relations}
        self.main, _col = V.record_main_component(air, log_size, rel, decoding=True, alu=self.ALU, control=self.CONTROL)
        self.final_reg = W._final_reg_component(air, rel["RegisterCheck"])
        self.bit_op = W._bit_op_component(air, rel["BitOp"])
        self.ram = W._ram_init_final_component(air, self.ram_log_size, rel["LoadStore"], rel["Range256"])
        self.tables = [W._multiplicity_component(air, rel[r], length, ls) for r, length, ls in W.MULTIPLICITY_TABLES]
        self.air = air
        self.log_sizes = [log_size, W.FINAL_REG_LOG_SIZE, W.BIT_OP_LOG_SIZE, self.ram_log_size] + [ls for _r, _l, ls in W.MULTIPLICITY_TABLES]
        self.words = air.serialize()
        self._main = None

    def default_program(self, log_size, n_steps):
        return add_chain_program(log_size, n_steps)

    def device_fill(self, ctx, out=None):
        """The main component's 347 columns filled on the device from the step record (nb200_v1_main_trace)."""
        return ctx.v1_main_trace(self.steps, self.final_ctr, self.log_size, out=out)

    # ---- tree 0
    def program_columns(self):
        """The program trace (program_trace.rs:48-100): PrgMemoryPc / PrgMemoryWord as 16-bit halves and PrgMemoryFlag on the program's rows,
        PrgInitialPc's bytes on row 0.  {column id: (2^log_size,) uint32}."""
        n, m = 1 << self.log_size, self.program.size
        out = {}
        pcs = ELF_TEXT_START + 4 * np.arange(m, dtype=np.uint64)
        for name, halves in (("PrgMemoryPc", pcs), ("PrgMemoryWord", self.program.astype(np.uint64))):
            for k, v in enumerate(((halves & 0xFFFF), halves >> 16)):
                out[f"{name}_{k}"] = np.zeros(n, np.uint32)
                out[f"{name}_{k}"][:m] = v
        out["PrgMemoryFlag_0"] = np.zeros(n, np.uint32)
        out["PrgMemoryFlag_0"][:m] = 1
        for k, b in enumerate(_le(ELF_TEXT_START)):
            out[f"PrgInitialPc_{k}"] = np.zeros(n, np.uint32)
            out[f"PrgInitialPc_{k}"][0] = b
        return out

    def preprocessed_columns(self):
        ids = self.air.preprocessed_ids
        by_id = dict(V.main_preprocessed_columns(self.log_size))
        by_id.update(self.program_columns())
        by_id[f"preprocessed_register_idx_{W.FINAL_REG_LOG_SIZE}"] = np.arange(32, dtype=np.uint32)
        r = np.arange(256, dtype=np.uint32)
        b, c = r >> 4, r & 15
        for name, v in zip(W.BITOP_PREPROCESSED, [b, c, b & c, b | c, b ^ c]):
            by_id[name] = v
        for name in W.RAM_PREPROCESSED:                                       # no initial memory, exit code or output
            by_id[name] = np.zeros(1 << self.ram_log_size, np.uint32)
        for _r, length, ls in W.MULTIPLICITY_TABLES:
            v = np.zeros(1 << ls, np.uint32)
            v[:length] = np.arange(length, dtype=np.uint32)
            by_id[f"preprocessed_range_values_{length}"] = v
        cols = [None] * self.air.n_columns()[0]
        for name, i in ids.items():
            cols[i] = by_id[name]
        return cols

    # ---- tree 1
    def final_reg_columns(self):
        """FinalReg's 8 columns: each register's final timestamp bytes, then its final value bytes (final_reg.rs:80-116)."""
        return _le(self.final_timestamps) + _le(self.final_values)

    def main_columns(self):
        return main_columns(self.steps, self.final_ctr, self.log_size)

    def fill_main_trace(self):
        """Tree 1 in commitment order: the 347 main columns, FinalReg, BitOpMultiplicity, RamInitFinal, then Multiplicity8 ... 256.
        Built once and cached."""
        if self._main is None:
            t = self.main_columns()
            ram = np.zeros((W.RAM_COLS, 1 << self.ram_log_size), np.uint32)
            h = table_counts(t, ram)
            cols = [limb for name, _ in V.MAIN_COLUMNS for limb in t[name]]
            cols += self.final_reg_columns()
            cols += [(v % P).astype(np.uint32) for v in h["BitOp"]]
            cols += list(ram)
            for r, length, ls in W.MULTIPLICITY_TABLES:
                v = np.zeros(1 << ls, np.int64)
                v[:length] = h[r]
                cols.append((v % P).astype(np.uint32))
            assert len(cols) == self.air.n_columns()[1]
            self._main = cols
        return list(self._main)

    def column_log_sizes(self):
        return self.air.column_log_sizes()

    def device_trees(self, ctx, out=None):
        """(tree-0 device batches, tree-1 device batches), finalized order, for machine.prove(..., resident=...): tree 0 and FinalReg's
        columns uploaded, the main component filled on the device from the step record (device_fill; `out` = a batch of 347 columns of
        2^log_size rows to reuse), RamInitFinal zero, and every table column (BitOpMultiplicity's among them) counted on the device from the
        filled trace (nb200_table_multiplicities_first_row)."""
        from .machine import fill_table_multiplicities

        def upload_runs(cols):
            res, i = [], 0
            while i < len(cols):
                j = i
                while j < len(cols) and len(cols[j]) == len(cols[i]):
                    j += 1
                res.append(ctx.upload(np.stack(cols[i:j]), coset_order=True))
                i = j
            return res

        tree0 = upload_runs(self.preprocessed_columns())
        tree1 = [self.device_fill(ctx, out=out)]
        tree1 += upload_runs(self.final_reg_columns())
        tree1.append(ctx.alloc(3, W.BIT_OP_LOG_SIZE))
        ram = ctx.alloc(W.RAM_COLS, self.ram_log_size)
        ram.upload(np.zeros((W.RAM_COLS, 1 << self.ram_log_size), np.uint32))
        tree1.append(ram)
        i = 0
        while i < len(W.MULTIPLICITY_TABLES):
            j = i
            while j < len(W.MULTIPLICITY_TABLES) and W.MULTIPLICITY_TABLES[j][2] == W.MULTIPLICITY_TABLES[i][2]:
                j += 1
            tree1.append(ctx.alloc(j - i, W.MULTIPLICITY_TABLES[i][2]))
            i = j
        fill_table_multiplicities(self, ctx, tree0, tree1, first_row=True)
        return tree0, tree1


class AluMachine(AddChainMachine):
    """A straight-line program over every RV32I register-register and register-immediate instruction but LUI / AUIPC (OPCODES) at
    2^log_size rows: alu_program(log_size, n_steps, seed) by default (n_steps defaults to 2^log_size), or `ops` = [(opcode, rd, rs1, rs2 /
    imm / shift amount)].  AddChainMachine's components, relations, draw order and interface, with the main component recorded with
    `alu=True` (SltuChip, SltChip, SllChip, SrlChip and SraChip constrained) and filled on the device by nb200_v1_alu_trace.  Its bit-op
    lookups make BitOpMultiplicity nonzero."""
    ALU = True

    def __init__(self, log_size, n_steps=None, ops=None, seed=0):
        self.seed = seed
        super().__init__(log_size, n_steps, ops)

    def default_program(self, log_size, n_steps):
        return alu_program(log_size, n_steps, self.seed)

    def device_fill(self, ctx, out=None):
        """The main component's 347 columns filled on the device from the step record (nb200_v1_alu_trace)."""
        return ctx.v1_alu_trace(self.steps, self.final_ctr, self.log_size, out=out)


class ControlMachine(AluMachine):
    """A looping program over all 29 opcodes of the step record (OPCODES and CONTROL_OPCODES) run for n_steps steps by `run`:
    control_program(log_size, n_steps, seed) by default, or `ops` = [(opcode, rd, rs1, c)] run for n_steps (default 2^log_size) steps.  The
    main component has max(8, ceil(log2 n_steps), ceil(log2 program length)) rows and is recorded with `control=True` (DecodingCheck's types
    B, U and J and the branch, JAL, LUI, AUIPC and JALR chips constrained); tree 0's program columns hold the program, and
    FinalPrgMemoryCtr how often each of its rows ran (0 for a row that never ran).  AluMachine's components, relations, draw order and
    interface; the main trace is filled on the device by nb200_v1_control_trace."""
    CONTROL = True

    def __init__(self, log_size=8, n_steps=None, ops=None, seed=0):
        self.seed = seed
        if ops is None:
            self.program, ops, n_steps = control_program(log_size, n_steps, seed)
        else:
            n_steps = (1 << log_size) if n_steps is None else int(n_steps)
            self.program = np.array([encode(*o) for o in ops], np.uint32)
        self.ops, self.n_steps = ops, n_steps
        assert n_steps >= 1
        ceil_log2 = lambda x: max(0, int(x - 1).bit_length())
        log_size = max(8, ceil_log2(n_steps), ceil_log2(len(ops)))
        self.log_size = self.log_size_main = log_size
        self.steps, (self.final_values, self.final_timestamps), self.final_ctr = run(ops, n_steps)
        self._record(log_size)

    def device_fill(self, ctx, out=None):
        """The main component's 347 columns filled on the device from the step record (nb200_v1_control_trace)."""
        return ctx.v1_control_trace(self.steps, self.final_ctr, self.log_size, out=out)
