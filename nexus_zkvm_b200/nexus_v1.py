"""The reference's v1 main component as data: real column layout + an exact transcription of a subset of its chips (class docstring).
Column tables generated from nexus-zkvm prover/src/column.rs (names and #[size] attributes, enum order) — layout data, not code."""
import numpy as np

from . import air as A

P = (1 << 31) - 1

MAIN_COLUMNS = [
    ("Pc", 4), ("PcNext", 4), ("PcNextAux", 4), ("OpA", 1), ("OpB", 1), ("OpC", 1), ("CarryFlag", 2), ("BorrowFlag", 2), ("ImmC", 1),
    ("InstrVal", 4), ("PrevCtr", 4), ("ValueA", 4), ("ValueAEffective", 4), ("ValueB", 4), ("ValueC", 4), ("IsAdd", 1), ("IsOr", 1), ("IsAnd", 1),
    ("IsXor", 1), ("IsSub", 1), ("IsSltu", 1), ("IsSlt", 1), ("IsBne", 1), ("IsBeq", 1), ("IsBltu", 1), ("IsBlt", 1), ("IsBgeu", 1), ("IsBge", 1),
    ("IsJal", 1), ("IsSb", 1), ("IsSh", 1), ("IsSw", 1), ("IsLb", 1), ("IsLh", 1), ("IsLbu", 1), ("IsLhu", 1), ("IsLw", 1), ("IsLui", 1),
    ("IsAuipc", 1), ("IsJalr", 1), ("IsSll", 1), ("IsSrl", 1), ("IsSra", 1), ("IsMul", 1), ("IsMulhu", 1), ("IsMulh", 1), ("IsMulhsu", 1),
    ("IsDivu", 1), ("IsDiv", 1), ("IsRemu", 1), ("IsRem", 1), ("IsEcall", 1), ("IsEbreak", 1), ("IsSysDebug", 1), ("IsSysMemoryAdvise", 1),
    ("IsSysHalt", 1), ("IsSysPrivInput", 1), ("IsSysCycleCount", 1), ("IsSysStackReset", 1), ("IsSysHeapReset", 1), ("IsCustomKeccak", 1),
    ("IsPadding", 1), ("Helper1", 4), ("Helper2", 4), ("Helper3", 4), ("Helper4", 4), ("SgnA", 1), ("SgnB", 1), ("SgnC", 1), ("Neq", 1),
    ("Neq12", 1), ("Neq34", 1), ("LtFlag", 1), ("RemAux", 1), ("Rem", 4), ("QtAux", 1), ("Qt", 4), ("ShiftBit1", 1), ("ShiftBit2", 1),
    ("ShiftBit3", 1), ("ShiftBit4", 1), ("ShiftBit5", 1), ("Exp1_3", 1), ("Exp", 1), ("RemDiff", 4), ("Neq12Aux", 1), ("Neq34Aux", 1),
    ("Neq12AuxInv", 1), ("Neq34AuxInv", 1), ("SraDegreeAux", 1), ("MulP1", 2), ("MulC1", 1), ("MulP3Prime", 2), ("MulC3Prime", 1),
    ("MulP3PrimePrime", 2), ("MulC3PrimePrime", 1), ("MulP5", 2), ("MulC5", 1), ("MulCarry0", 1), ("MulCarry1", 1), ("MulCarry2_0", 1),
    ("MulCarry2_1", 1), ("MulCarry3", 1), ("IsDivideByZero", 1), ("IsAZero", 1), ("IsOverflow", 1), ("Quotient", 4), ("HelperT", 4),
    ("Remainder", 4), ("HelperU", 4), ("RemainderBorrow", 1), ("HelperUBorrow", 1), ("ValueALow", 4), ("ValueAAbsBorrow", 2),
    ("ValueAAbsBorrowHigh", 2), ("ValueBAbsBorrow", 2), ("ValueCAbsBorrow", 2), ("ValueAAbs", 4), ("ValueAAbsHigh", 4), ("ValueBAbs", 4),
    ("ValueCAbs", 4), ("ValueAEffectiveFlag", 1), ("ValueAEffectiveFlagAux", 1), ("ValueAEffectiveFlagAuxInv", 1), ("Reg1Address", 1),
    ("Reg2Address", 1), ("Reg3Address", 1), ("Reg1ValPrev", 4), ("Reg2ValPrev", 4), ("Reg3ValPrev", 4), ("Reg1TsPrev", 4), ("Reg2TsPrev", 4),
    ("Reg3TsPrev", 4), ("ProgCtrPrev", 4), ("ProgCtrCur", 4), ("ProgCtrCarry", 2), ("FinalPrgMemoryCtr", 4), ("CReg1TsPrev", 4), ("CReg2TsPrev", 4),
    ("CReg3TsPrev", 4), ("CH1Minus", 2), ("CH2Minus", 2), ("CH3Minus", 2), ("RamBaseAddr", 4), ("Ram1ValCur", 1), ("Ram2ValCur", 1),
    ("Ram3ValCur", 1), ("Ram4ValCur", 1), ("Ram1ValPrev", 1), ("Ram2ValPrev", 1), ("Ram3ValPrev", 1), ("Ram4ValPrev", 1), ("Ram1TsPrev", 4),
    ("Ram2TsPrev", 4), ("Ram3TsPrev", 4), ("Ram4TsPrev", 4), ("Ram1TsPrevAux", 4), ("Ram2TsPrevAux", 4), ("Ram3TsPrevAux", 4), ("Ram4TsPrevAux", 4),
    ("OpC0_3", 1), ("OpC1_3", 1), ("OpC1_4", 1), ("OpC4_7", 1), ("OpC5_7", 1), ("OpC8_10", 1), ("OpC11", 1), ("OpC12", 1), ("OpC20", 1),
    ("OpA1_4", 1), ("OpB0_3", 1), ("OpB1_4", 1), ("OpC0", 1), ("OpC4", 1), ("OpA0", 1), ("OpB0", 1), ("OpB4", 1), ("OpC12_15", 1), ("OpC16_23", 1),
    ("OpC16_19", 1), ("OpC24_31", 1), ("PcCarry", 2), ("ValueA4_7", 4), ("ValueB4_7", 4), ("ValueC4_7", 4),
]
PREPROCESSED_COLUMNS = [
    ("IsFirst", 1), ("IsLast", 1), ("Clk", 4), ("Reg1TsCur", 4), ("Reg2TsCur", 4), ("Reg3TsCur", 4),
]
PROGRAM_COLUMNS = [
    ("PrgMemoryPc", 2), ("PrgMemoryWord", 2), ("PrgMemoryFlag", 1), ("PrgInitialPc", 4),
]


# ---- chip data transcribed from the reference (column lists are the reference's const arrays) --------------------------------
# virtual columns: prover/src/virtual_column.rs
TYPE_R_OPS = ["IsAdd", "IsSub", "IsSlt", "IsSltu", "IsXor", "IsOr", "IsAnd", "IsSll", "IsSrl", "IsSra", "IsMul", "IsMulhu", "IsDiv", "IsDivu",
              "IsRem", "IsRemu", "IsMulh", "IsMulhsu"]
IS_ALU = TYPE_R_OPS
IS_LOAD = ["IsLb", "IsLh", "IsLw", "IsLbu", "IsLhu"]
IS_TYPE_S = ["IsSb", "IsSh", "IsSw"]
IS_TYPE_SYS = ["IsEcall", "IsEbreak"]
IS_TYPE_U = ["IsLui", "IsAuipc"]
IS_TYPE_B = ["IsBeq", "IsBne", "IsBlt", "IsBge", "IsBltu", "IsBgeu"]
ALU_IMM_NO_SHIFT = ["IsAdd", "IsSlt", "IsSltu", "IsXor", "IsOr", "IsAnd"]
ALU_IMM_SHIFT = ["IsSll", "IsSrl", "IsSra"]
OP_B_FLAG = ["IsSb", "IsSh", "IsSw", "IsLb", "IsLh", "IsLw", "IsLbu", "IsLhu", "IsJalr", "IsAdd", "IsSub", "IsSlt", "IsSltu", "IsXor", "IsOr", "IsAnd",
             "IsSll", "IsSrl", "IsSra", "IsBeq", "IsBne", "IsBlt", "IsBge", "IsBltu", "IsBgeu", "IsMul", "IsEcall", "IsEbreak", "IsMulhu", "IsDivu",
             "IsRemu", "IsDiv", "IsRem", "IsMulh", "IsMulhsu"]
# cpu.rs:379-420: the flags whose sum (plus IsPadding, IsCustomKeccak) must be one
CPU_OP_FLAGS = ["IsAdd", "IsSub", "IsAnd", "IsOr", "IsXor", "IsSlt", "IsSltu", "IsBne", "IsBeq", "IsBltu", "IsBgeu", "IsBlt", "IsBge", "IsJal", "IsSb",
                "IsSh", "IsSw", "IsLui", "IsAuipc", "IsJalr", "IsLb", "IsLbu", "IsLh", "IsLhu", "IsLw", "IsSll", "IsSrl", "IsSra", "IsMul", "IsMulh",
                "IsMulhsu", "IsMulhu", "IsDiv", "IsDivu", "IsRem", "IsRemu", "IsEcall", "IsEbreak"]
# range_check/range_bool.rs:30-124
BOOL_SINGLE = ["ValueAEffectiveFlag", "ImmC", "IsAdd", "IsOr", "IsAnd", "IsXor", "IsSub", "IsSltu", "IsSlt", "IsBltu", "IsBlt", "IsBgeu", "IsBge", "IsBne",
               "IsBeq", "IsJal", "IsSb", "IsSh", "IsSw", "IsLb", "IsLh", "IsLbu", "IsLhu", "IsLw", "IsLui", "IsAuipc", "IsJalr", "IsSll", "IsSrl", "IsSra",
               "IsMul", "IsMulhu", "IsMulh", "IsMulhsu", "IsDivu", "IsRemu", "IsDiv", "IsRem", "IsEcall", "IsEbreak", "IsSysCycleCount", "IsSysDebug",
               "IsSysHalt", "IsSysHeapReset", "IsSysPrivInput", "IsSysStackReset", "IsPadding", "LtFlag", "RemAux", "SgnA", "SgnB", "SgnC", "ShiftBit1",
               "ShiftBit2", "ShiftBit3", "ShiftBit4", "ShiftBit5"]
BOOL_HALF_WORD = ["CarryFlag", "PcCarry", "CH1Minus", "CH2Minus", "CH3Minus", "ProgCtrCarry", "BorrowFlag", "ValueAAbsBorrow", "ValueBAbsBorrow",
                  "ValueCAbsBorrow", "ValueAAbsBorrowHigh"]
BOOL_TYPE_R = ["OpC4", "OpA0", "OpB0", "MulCarry0", "MulCarry2_0", "MulCarry2_1", "MulCarry3", "MulC1", "MulC3Prime", "MulC3PrimePrime", "MulC5",
               "IsDivideByZero", "IsOverflow", "IsAZero", "RemainderBorrow", "HelperUBorrow"]
BOOL_TYPE_I_NO_SHIFT = ["OpC11", "OpA0", "OpB0"]
BOOL_TYPE_I_SHIFT = ["OpC4", "OpA0", "OpB0"]
BOOL_TYPE_J = ["OpC11", "OpC20", "OpA0"]
BOOL_TYPE_B = ["OpC11", "OpC12", "OpA0", "OpB4"]
BOOL_TYPE_S = ["OpC0", "OpC11", "OpA0", "OpB4"]
# range_check/range256.rs:41-95
R256_WORDS = ["Pc", "PcNextAux", "InstrVal", "PrevCtr", "ValueA", "ValueB", "ValueC", "Reg1TsPrev", "Reg2TsPrev", "Reg3TsPrev", "Helper1", "ProgCtrCur",
              "ProgCtrPrev", "FinalPrgMemoryCtr", "CReg1TsPrev", "CReg2TsPrev", "CReg3TsPrev", "RamBaseAddr", "Ram1TsPrev", "Ram2TsPrev", "Ram3TsPrev",
              "Ram4TsPrev", "Ram1TsPrevAux", "Ram2TsPrevAux", "Ram3TsPrevAux", "Ram4TsPrevAux", "Rem", "Qt", "RemDiff", "HelperT", "HelperU", "Quotient",
              "Remainder", "ValueBAbs", "ValueCAbs", "ValueAAbs", "ValueAAbsHigh", "ValueALow"]
R256_BYTES = ["Ram1ValCur", "Ram2ValCur", "Ram3ValCur", "Ram4ValCur", "Ram1ValPrev", "Ram2ValPrev", "Ram3ValPrev", "Ram4ValPrev"]
R256_HALF_WORDS = ["MulP1", "MulP3Prime", "MulP3PrimePrime", "MulP5"]
R256_TYPE_U_BYTES = ["OpC16_23", "OpC24_31"]
# range_check/range16.rs:34-40, range8.rs:46-50, range32.rs:30
R16 = [("R", ["OpC0_3", "OpA1_4", "OpB1_4"]), ("U", ["OpC12_15", "OpA1_4"]), ("INoShift", ["OpC0_3", "OpC4_7", "OpA1_4", "OpB1_4"]),
       ("IShift", ["OpC0_3", "OpA1_4", "OpB1_4"]), ("J", ["OpC4_7", "OpC12_15", "OpC16_19", "OpA1_4"]), ("B", ["OpC1_4", "OpA1_4", "OpB0_3"]),
       ("S", ["OpC1_4", "OpA1_4", "OpB0_3"])]
R8 = [("INoShift", ["OpC8_10"]), ("J", ["OpC1_3", "OpC8_10"]), ("B", ["OpC5_7", "OpC8_10"]), ("S", ["OpC5_7", "OpC8_10"]), ("R", ["MulCarry1"])]
R32 = ["OpA", "OpB", "Reg1Address", "Reg2Address", "Reg3Address"]


def main_preprocessed_columns(log_size):
    """The main component's 18 preprocessed and 9 program columns for an empty program: {column id: (2^log_size,) uint32}."""
    n = 1 << log_size
    out = {}

    def put(name, limbs):
        for i, v in enumerate(limbs):
            out[f"{name}_{i}"] = v

    z = np.zeros(n, np.uint32)
    first, last = z.copy(), z.copy()
    first[0], last[n - 1] = 1, 1
    put("IsFirst", [first]); put("IsLast", [last])
    clk = np.arange(1, n + 1, dtype=np.uint64)                              # preprocessed.rs:75-100
    le = lambda x: [((x >> (8 * k)) & 0xFF).astype(np.uint32) for k in range(4)]
    put("Clk", le(clk)); put("Reg1TsCur", le(3 * clk + 1)); put("Reg2TsCur", le(3 * clk + 2)); put("Reg3TsCur", le(3 * clk + 3))
    for name, size in PROGRAM_COLUMNS:                                      # empty program: the program trace is all zero
        put(name, [z] * size)
    return out


def padding_witness(log_size, seed=0):
    """The main component's padding-only witness (NexusV1Machine's docstring): {column name: its limbs, (2^log_size,) uint32 each}."""
    n = 1 << log_size
    rng = np.random.default_rng(seed)
    t = {name: [np.zeros(n, np.uint32) for _ in range(size)] for name, size in MAIN_COLUMNS}
    t["IsPadding"][0][:] = 1
    t["ValueAEffectiveFlagAux"][0][:] = 1
    t["ValueAEffectiveFlagAuxInv"][0][:] = 1
    rb = lambda: rng.integers(0, 256, n, dtype=np.uint64).astype(np.uint32)
    free_words = [w for w in R256_WORDS if w not in ("Reg1TsPrev", "Reg2TsPrev", "Reg3TsPrev", "CReg1TsPrev", "CReg2TsPrev", "CReg3TsPrev")]
    for w in free_words + R256_HALF_WORDS + R256_BYTES + ["ValueAEffective", "Reg1ValPrev", "Reg2ValPrev", "Reg3ValPrev", "PcNext"]:
        if w == "ValueAEffective":
            continue                                                    # = ValueA * flag = 0 (register_mem_check.rs:129-136)
        for limb in t[w]:
            limb[:] = rb()
    for limb in t["Pc"]:
        limb[0] = 0                                                    # is_first * (pc - PrgInitialPc) with an empty program
    for w in ("ValueA4_7", "ValueB4_7", "ValueC4_7"):                   # high nibbles of the (free) values; only looked up when a bit-op flag is set
        src = {"ValueA4_7": "ValueA", "ValueB4_7": "ValueB", "ValueC4_7": "ValueC"}[w]
        for k in range(4):
            t[w][k][:] = t[src][k] >> 4
    for w in ("OpB", "Reg1Address", "Reg2Address", "Reg3Address"):       # Range32-checked; OpA = ValueAEffectiveFlag / aux = 0
        t[w][0][:] = rng.integers(0, 32, n, dtype=np.uint64).astype(np.uint32)
    # timestamps: prev < cur = 3 clk + k, c = cur - 1 - prev with the chip's per-16-bit borrows (timestamp.rs:101-150)
    clk = np.arange(1, n + 1, dtype=np.uint64)
    for k in (1, 2, 3):
        cur = 3 * clk + k
        prev = (rng.integers(0, 1 << 62, n, dtype=np.uint64) % cur).astype(np.uint64)
        cc = cur - 1 - prev
        lo = (cc & 0xFFFF) + (prev & 0xFFFF) + 1
        b0 = (lo >> 16).astype(np.uint32)
        hi = (cc >> 16) + (prev >> 16) + b0
        assert np.all(lo - (b0.astype(np.uint64) << 16) == (cur & 0xFFFF)) and np.all(hi == (cur >> 16))
        for i in range(4):
            t[f"Reg{k}TsPrev"][i][:] = ((prev >> (8 * i)) & 0xFF).astype(np.uint32)
            t[f"CReg{k}TsPrev"][i][:] = ((cc >> (8 * i)) & 0xFF).astype(np.uint32)
        t[f"CH{k}Minus"][0][:] = b0
    return t


def _record_decoding_r_i(m, c, col, is_type_r, is_load, alu_imm_no_shift, alu_imm_shift, is_type_i_no_shift):
    """DecodingCheckChip's TypeRChip and TypeIChip = (TypeINoShiftChip, TypeIShiftChip) constraints, in the reference's order: the register
    and immediate fields of OpA / OpB / OpC and ValueC against their bit pieces, and the instruction word's bytes (InstrVal) against the
    opcode, funct3 and funct7 of each instruction."""
    one_m_imm, imm_c = 1 - c("ImmC"), c("ImmC")
    a0, a14, b0, b14 = c("OpA0"), c("OpA1_4"), c("OpB0"), c("OpB1_4")
    c03, c4, c47, c810, c11 = c("OpC0_3"), c("OpC4"), c("OpC4_7"), c("OpC8_10"), c("OpC11")
    op_a, op_b, op_c = c("OpA"), c("OpB"), c("OpC")
    iv, vc = col["InstrVal"], col["ValueC"]
    funct3 = lambda f: a14 + f * 16 + b0 * 128 - iv[1]                    # op_a1_4 + funct3 2^4 + op_b0 2^7 - instr_val_2
    # type R (type_r.rs:67-408)
    m.add_constraint(is_type_r * (c03 + c4 * 16 - op_c))
    m.add_constraint(is_type_r * (a0 + a14 * 2 - op_a))
    m.add_constraint(is_type_r * (b0 + b14 * 2 - op_b))
    m.add_constraint(is_type_r * (0b0110011 + a0 * 128 - iv[0]))
    r_funct3 = [("IsAdd", 0b000), ("IsSub", 0b000), ("IsSll", 0b001), ("IsSlt", 0b010), ("IsSltu", 0b011), ("IsXor", 0b100), ("IsSrl", 0b101),
                ("IsSra", 0b101), ("IsOr", 0b110), ("IsAnd", 0b111), ("IsMul", 0b000), ("IsMulhu", 0b011), ("IsDivu", 0b101), ("IsRemu", 0b111),
                ("IsDiv", 0b100), ("IsRem", 0b110), ("IsMulhsu", 0b010), ("IsMulh", 0b001)]
    for flag, f in r_funct3:
        m.add_constraint(c(flag) * one_m_imm * funct3(f))
    m.add_constraint(is_type_r * (b14 + c03 * 16 - iv[2]))
    for flag, f7 in (("IsAdd", 0), ("IsSub", 0b0100000), ("IsSll", 0), ("IsSlt", 0), ("IsSltu", 0), ("IsXor", 0), ("IsSrl", 0),
                     ("IsSra", 0b0100000), ("IsOr", 0), ("IsAnd", 0)):
        m.add_constraint(c(flag) * one_m_imm * (c4 + f7 * 2 - iv[3]))
    m_ops = c("IsMul") + c("IsMulhu") + c("IsDivu") + c("IsRemu") + c("IsDiv") + c("IsRem") + c("IsMulhsu") + c("IsMulh")
    m.add_constraint(m_ops * one_m_imm * (c4 + 0b0000001 * 2 - iv[3]))
    # type I without shift (type_i.rs:77-283)
    t = is_type_i_no_shift
    m.add_constraint(t * (c03 + c47 * 16 + c810 * 256 + c11 * 2048 - op_c))
    m.add_constraint(t * (c03 + c47 * 16 - vc[0]))
    m.add_constraint(t * (c810 + c11 * ((1 << 5) - 1) * 8 - vc[1]))
    m.add_constraint(t * (c11 * 255 - vc[2]))
    m.add_constraint(t * (c11 * 255 - vc[3]))
    m.add_constraint(t * (a0 + a14 * 2 - op_a))
    m.add_constraint(t * (b0 + b14 * 2 - op_b))
    m.add_constraint(is_load * (0b0000011 + a0 * 128 - iv[0]))
    m.add_constraint(alu_imm_no_shift * (0b0010011 + a0 * 128 - iv[0]))
    m.add_constraint(c("IsJalr") * (0b1100111 + a0 * 128 - iv[0]))
    for flag, f in (("IsLb", 0b000), ("IsLh", 0b001), ("IsLw", 0b010), ("IsLbu", 0b100), ("IsLhu", 0b101)):
        m.add_constraint(c(flag) * funct3(f))
    for flag, f in (("IsAdd", 0b000), ("IsSlt", 0b010), ("IsSltu", 0b011), ("IsXor", 0b100), ("IsOr", 0b110), ("IsAnd", 0b111)):
        m.add_constraint(c(flag) * imm_c * funct3(f))
    m.add_constraint(c("IsJalr") * funct3(0b000))
    m.add_constraint(t * (b14 + c03 * 16 - iv[2]))
    m.add_constraint(t * (c47 + c810 * 16 + c11 * 128 - iv[3]))
    # type I with a shift amount (type_i.rs:335-441)
    s = alu_imm_shift
    m.add_constraint(s * (c03 + c4 * 16 - op_c))
    m.add_constraint(s * (c03 + c4 * 16 - vc[0]))
    for k in (1, 2, 3):
        m.add_constraint(s * vc[k])
    m.add_constraint(s * (a0 + a14 * 2 - op_a))
    m.add_constraint(s * (b0 + b14 * 2 - op_b))
    m.add_constraint(s * (0b0010011 + a0 * 128 - iv[0]))
    for flag, f in (("IsSll", 0b001), ("IsSrl", 0b101), ("IsSra", 0b101)):
        m.add_constraint(c(flag) * imm_c * funct3(f))
    m.add_constraint(s * (b14 + c03 * 16 - iv[2]))
    for flag, f7 in (("IsSll", 0), ("IsSrl", 0), ("IsSra", 0b0100000)):
        m.add_constraint(c(flag) * imm_c * (c4 + f7 * 2 - iv[3]))


def _record_sltu(m, c, col):
    """SltuChip (sltu.rs:79-131): a = b - c with CarryFlag as the two 16-bit borrows into Helper1, and ValueA = the high borrow."""
    is_sltu, bf, vb, vc, va, h1 = c("IsSltu"), col["CarryFlag"], col["ValueB"], col["ValueC"], col["ValueA"], col["Helper1"]
    m.add_constraint(is_sltu * (bf[1] - va[0]))
    m.add_constraint(is_sltu * (h1[0] + h1[1] * 256 - bf[0] * 65536 - (vb[0] + vb[1] * 256 - vc[0] - vc[1] * 256)))
    m.add_constraint(is_sltu * (h1[2] + h1[3] * 256 - bf[1] * 65536 - (vb[2] + vb[3] * 256 - vc[2] - vc[3] * 256 - bf[0])))
    for k in (1, 2, 3):
        m.add_constraint(is_sltu * va[k])


def _record_slt(m, c, col):
    """SltChip (slt.rs:118-199): the unsigned borrow as SLTU's, combined with the sign bits SgnB / SgnC split off ValueB / ValueC's top
    bytes (their low seven bits in Helper2[3] / Helper3[3])."""
    is_slt, bf, vb, vc, va, h1 = c("IsSlt"), col["CarryFlag"], col["ValueB"], col["ValueC"], col["ValueA"], col["Helper1"]
    sgn_b, sgn_c = c("SgnB"), c("SgnC")
    m.add_constraint(is_slt * (h1[0] + h1[1] * 256 - bf[0] * 65536 - (vb[0] + vb[1] * 256 - vc[0] - vc[1] * 256)))
    m.add_constraint(is_slt * (h1[2] + h1[3] * 256 - bf[1] * 65536 - (vb[2] + vb[3] * 256 - vc[2] - vc[3] * 256 - bf[0])))
    m.add_constraint(is_slt * (sgn_b * (1 - sgn_c) + bf[1] * (sgn_b * sgn_c + (1 - sgn_b) * (1 - sgn_c)) - va[0]))
    for k in (1, 2, 3):
        m.add_constraint(is_slt * va[k])
    m.add_constraint(is_slt * (sgn_b * 128 + col["Helper2"][3] - vb[3]))
    m.add_constraint(is_slt * (sgn_c * 128 + col["Helper3"][3] - vc[3]))


def _shift_amount(m, flag, col):
    """The first two constraints of SllChip, SrlChip and SraChip: ValueC's low byte = ShiftBit1..5 + 32 Helper1[0], and Exp1_3 = 2^(its
    low three bits).  Returns ShiftBit1..5."""
    sh = [col[f"ShiftBit{k}"][0] for k in range(1, 6)]
    m.add_constraint(flag * (sh[0] + sh[1] * 2 + sh[2] * 4 + sh[3] * 8 + sh[4] * 16 + col["Helper1"][0] * 32 - col["ValueC"][0]))
    m.add_constraint(flag * ((sh[0] + 1) * (sh[1] * 3 + 1) * (sh[2] * 15 + 1) - col["Exp1_3"][0]))
    return sh


def _right_shift_by_exp(m, flag, col):
    """SrlChip's and SraChip's byte-wise division of ValueB by Exp1_3: quotients Qt, remainders Rem carried down from the top byte."""
    vb, rem, qt, e = col["ValueB"], col["Rem"], col["Qt"], col["Exp1_3"][0]
    m.add_constraint(flag * (vb[3] - rem[3] - qt[3] * e))
    for i in (2, 1, 0):
        m.add_constraint(flag * (vb[i] + rem[i + 1] * 256 - rem[i] - qt[i] * e))


def _byte_moves(sh4, sh5):
    """The byte-shift selectors of ShiftBit4 / ShiftBit5 for a move by 0, 1, 2 and 3 bytes."""
    return [(1 - sh4) * (1 - sh5), sh4 * (1 - sh5), (1 - sh4) * sh5, sh4 * sh5]


def _record_sll(m, c, col):
    """SllChip (sll.rs:114-199): ValueB times Exp1_3 byte by byte (Rem, carries Qt), then moved up by ShiftBit4 + 2 ShiftBit5 bytes."""
    is_sll, vb, va, rem, qt, e = c("IsSll"), col["ValueB"], col["ValueA"], col["Rem"], col["Qt"], col["Exp1_3"][0]
    sh = _shift_amount(m, is_sll, col)
    m.add_constraint(is_sll * (rem[0] + qt[0] * 256 - vb[0] * e))
    for i in (1, 2, 3):
        m.add_constraint(is_sll * (rem[i] + qt[i] * 256 - qt[i - 1] - vb[i] * e))
    sel = _byte_moves(sh[3], sh[4])
    for i in range(4):
        acc = va[i]
        for j in range(i + 1):
            acc = acc - rem[i - j] * sel[j]
        m.add_constraint(is_sll * acc)


def _record_srl(m, c, col):
    """SrlChip (srl.rs:121-232): ValueB divided by Exp1_3 byte by byte, the quotients moved down by ShiftBit4 + 2 ShiftBit5 bytes, and
    RemDiff = Exp1_3 - 1 - Rem (Range256-checked, so Rem < Exp1_3)."""
    is_srl, va, qt, rem, e = c("IsSrl"), col["ValueA"], col["Qt"], col["Rem"], col["Exp1_3"][0]
    sh = _shift_amount(m, is_srl, col)
    _right_shift_by_exp(m, is_srl, col)
    sel = _byte_moves(sh[3], sh[4])
    for i in (3, 2, 1, 0):
        acc = va[i]
        for j in range(4 - i):
            acc = acc - qt[i + j] * sel[j]
        m.add_constraint(is_srl * acc)
    for i in range(4):
        m.add_constraint(is_srl * (e - 1 - rem[i] - col["RemDiff"][i]))


def _record_sra(m, c, col):
    """SraChip (sra.rs:141-347): SRL's quotients into Helper3 (the logical shift), SgnB split off ValueB's top byte (low seven bits in
    Helper2[0]), Exp = 2^8 / Exp1_3, SraDegreeAux = SgnB (Exp1_3 - 1) Exp (the sign bits the byte the shift lands in gets), and ValueA =
    the logical shift with the sign replicated into the vacated bytes."""
    is_sra, vb, va, qt, rem, e = c("IsSra"), col["ValueB"], col["ValueA"], col["Qt"], col["Rem"], col["Exp1_3"][0]
    srl, exp, sgn_b, aux = col["Helper3"], c("Exp"), c("SgnB"), c("SraDegreeAux")
    sh = _shift_amount(m, is_sra, col)
    _right_shift_by_exp(m, is_sra, col)
    m.add_constraint(is_sra * (col["Helper2"][0] + sgn_b * 128 - vb[3]))
    sel = _byte_moves(sh[3], sh[4])
    for i in (3, 2, 1, 0):
        acc = srl[i]
        for j in range(4 - i):
            acc = acc - qt[i + j] * sel[j]
        m.add_constraint(is_sra * acc)
    sh1, sh2, sh3, sh4, sh5 = sh
    m.add_constraint(is_sra * (2 * (2 - sh1) * (4 - sh2 * 3) * (16 - sh3 * 15) - exp))
    m.add_constraint(is_sra * (sgn_b * (e - 1) * exp - aux))
    m.add_constraint(is_sra * (va[3] - (1 - sh4) * (1 - sh5) * (srl[3] + aux) - (sh4 + sh5 - sh4 * sh5) * sgn_b * 255))
    m.add_constraint(is_sra * (va[2] - (1 - sh4) * (1 - sh5) * srl[2] - sh4 * (1 - sh5) * (srl[2] + aux) - sh5 * sgn_b * 255))
    m.add_constraint(is_sra * (va[1] - (1 - sh5) * srl[1] - (1 - sh4) * sh5 * (srl[1] + aux) - sh4 * sh5 * sgn_b * 255))
    m.add_constraint(is_sra * (va[0] - (1 - sh4 * sh5) * srl[0] - sh4 * sh5 * (srl[0] + aux)))
    for i in range(4):
        m.add_constraint(is_sra * (e - 1 - rem[i] - col["RemDiff"][i]))


# the instruction chips that alu=True records, in BaseComponent's order (SltuChip before BitOpChip, the others after it)
ALU_CHIPS_BEFORE_BIT_OP = [("SltuChip", _record_sltu)]
ALU_CHIPS_AFTER_BIT_OP = [("SltChip", _record_slt), ("SllChip", _record_sll), ("SrlChip", _record_srl), ("SraChip", _record_sra)]


def _record_type_b(m, c, col):
    """DecodingCheck's TypeBChip (type_b.rs:75-233): OpC is the raw 13-bit offset (OpC1_4, OpC5_7, OpC8_10, OpC11, OpC12), ValueC its
    sign extension; OpA is the instruction's rs1 field, OpB its rs2 field (OpB0_3, OpB4); the instruction word's bytes."""
    t = sum_of(c, IS_TYPE_B)
    c14, c57, c810, c11, c12 = c("OpC1_4"), c("OpC5_7"), c("OpC8_10"), c("OpC11"), c("OpC12")
    a0, a14, b03, b4 = c("OpA0"), c("OpA1_4"), c("OpB0_3"), c("OpB4")
    vc, iv = col["ValueC"], col["InstrVal"]
    m.add_constraint(t * (c14 * 2 + c57 * 32 + c810 * 256 + c11 * 2048 + c12 * 4096 - c("OpC")))
    m.add_constraint(t * (c14 * 2 + c57 * 32 - vc[0]))
    m.add_constraint(t * (c810 + c11 * 8 + c12 * 15 * 16 - vc[1]))
    m.add_constraint(t * (c12 * 255 - vc[2]))
    m.add_constraint(t * (c12 * 255 - vc[3]))
    m.add_constraint(t * (a0 + a14 * 2 - c("OpA")))
    m.add_constraint(t * (b03 + b4 * 16 - c("OpB")))
    m.add_constraint(t * (0b1100011 + c11 * 128 - iv[0]))
    for flag, f3 in (("IsBeq", 0b000), ("IsBne", 0b001), ("IsBlt", 0b100), ("IsBge", 0b101), ("IsBltu", 0b110), ("IsBgeu", 0b111)):
        m.add_constraint(c(flag) * (c14 + f3 * 16 + a0 * 128 - iv[1]))
    m.add_constraint(t * (a14 + b03 * 16 - iv[2]))
    m.add_constraint(t * (b4 + c57 * 2 + c810 * 16 + c12 * 128 - iv[3]))


def _record_type_u(m, c, col):
    """DecodingCheck's TypeUChip (type_u.rs:53-138): OpC is the 20-bit immediate (OpC12_15, OpC16_23, OpC24_31), ValueC = OpC << 12,
    OpB = ValueB = 0; the instruction word's bytes."""
    t = sum_of(c, IS_TYPE_U)
    c1215, c1623, c2431, a0, a14 = c("OpC12_15"), c("OpC16_23"), c("OpC24_31"), c("OpA0"), c("OpA1_4")
    vb, vc, iv = col["ValueB"], col["ValueC"], col["InstrVal"]
    m.add_constraint(t * (c1215 + c1623 * 16 + c2431 * 4096 - c("OpC")))
    m.add_constraint(t * vc[0])
    m.add_constraint(t * (c1215 * 16 - vc[1]))
    m.add_constraint(t * (c1623 - vc[2]))
    m.add_constraint(t * (c2431 - vc[3]))
    m.add_constraint(t * (a0 + a14 * 2 - c("OpA")))
    m.add_constraint(t * c("OpB"))
    for k in range(4):
        m.add_constraint(t * vb[k])
    m.add_constraint(c("IsLui") * (0b0110111 + a0 * 128 - iv[0]))
    m.add_constraint(c("IsAuipc") * (0b0010111 + a0 * 128 - iv[0]))
    m.add_constraint(t * (a14 + c1215 * 16 - iv[1]))
    m.add_constraint(t * (c1623 - iv[2]))
    m.add_constraint(t * (c2431 - iv[3]))


def _record_type_j(m, c, col):
    """DecodingCheck's TypeJChip (type_j.rs:64-193): OpC is the raw 21-bit offset (OpC1_3, OpC4_7, OpC8_10, OpC11, OpC12_15, OpC16_19,
    OpC20), ValueC its sign extension, OpB = ValueB = 0; the instruction word's bytes."""
    t = c("IsJal")
    c13, c47, c810, c11, c1215, c1619, c20 = (c(n) for n in ("OpC1_3", "OpC4_7", "OpC8_10", "OpC11", "OpC12_15", "OpC16_19", "OpC20"))
    a0, a14 = c("OpA0"), c("OpA1_4")
    vb, vc, iv = col["ValueB"], col["ValueC"], col["InstrVal"]
    m.add_constraint(t * (c13 * 2 + c47 * 16 + c810 * 256 + c11 * 2048 + c1215 * 4096 + c1619 * 65536 + c20 * (1 << 20) - c("OpC")))
    m.add_constraint(t * (c13 * 2 + c47 * 16 - vc[0]))
    m.add_constraint(t * (c810 + c11 * 8 + c1215 * 16 - vc[1]))
    m.add_constraint(t * (c1619 + c20 * 15 * 16 - vc[2]))
    m.add_constraint(t * (c20 * 255 - vc[3]))
    m.add_constraint(t * (a0 + a14 * 2 - c("OpA")))
    m.add_constraint(t * c("OpB"))
    for k in range(4):
        m.add_constraint(t * vb[k])
    m.add_constraint(t * (0b1101111 + a0 * 128 - iv[0]))
    m.add_constraint(t * (a14 + c1215 * 16 - iv[1]))
    m.add_constraint(t * (c1619 + c11 * 16 + c13 * 32 - iv[2]))
    m.add_constraint(t * (c47 + c810 * 16 + c20 * 128 - iv[3]))


def _next_pc(m, flag, col, taken):
    """The two 16-bit halves of PcNext = Pc + (taken ? ValueC : 4) with CarryFlag as the carries (the branch chips' last two constraints)."""
    vc, pc, pn, cf = col["ValueC"], col["Pc"], col["PcNext"], col["CarryFlag"]
    m.add_constraint(flag * (taken * (vc[0] + vc[1] * 256) + (1 - taken) * 4 + pc[0] + pc[1] * 256 - cf[0] * 65536 - pn[0] - pn[1] * 256))
    m.add_constraint(flag * (taken * (vc[2] + vc[3] * 256) + pc[2] + pc[3] * 256 + cf[0] - cf[1] * 65536 - pn[2] - pn[3] * 256))


def _record_beq_bne(flag_name, equal_taken):
    """BeqChip / BneChip (beq.rs:152-260, bne.rs): Neq12 / Neq34 = the 16-bit halves of ValueA and ValueB differ, through the inverses
    Neq12Aux / Neq34Aux of their differences (any nonzero value with its inverse when they are equal), Neq = either differs, and PcNext."""
    def record(m, c, col):
        flag, va, vb = c(flag_name), col["ValueA"], col["ValueB"]
        neq, n12, n34 = c("Neq"), c("Neq12"), c("Neq34")
        m.add_constraint(flag * ((va[0] + va[1] * 256 - vb[0] - vb[1] * 256) * c("Neq12Aux") - n12))
        m.add_constraint(flag * ((va[2] + va[3] * 256 - vb[2] - vb[3] * 256) * c("Neq34Aux") - n34))
        m.add_constraint(flag * n12 * (1 - n12))
        m.add_constraint(flag * n34 * (1 - n34))
        m.add_constraint(flag * (c("Neq12Aux") * c("Neq12AuxInv") - 1))
        m.add_constraint(flag * (c("Neq34Aux") * c("Neq34AuxInv") - 1))
        m.add_constraint(flag * ((1 - n12) * (1 - n34) - (1 - neq)))
        _next_pc(m, flag, col, 1 - neq if equal_taken else neq)
    return record


def _sub_borrows(m, flag, col):
    """Helper1 = ValueA - ValueB with BorrowFlag as the borrows out of the 16-bit halves (the compare branches' first two constraints)."""
    va, vb, h1, bf = col["ValueA"], col["ValueB"], col["Helper1"], col["BorrowFlag"]
    m.add_constraint(flag * (va[0] + va[1] * 256 - vb[0] - vb[1] * 256 - h1[0] - h1[1] * 256 + bf[0] * 65536))
    m.add_constraint(flag * (va[2] + va[3] * 256 - vb[2] - vb[3] * 256 - h1[2] - h1[3] * 256 + bf[1] * 65536 - bf[0]))


def _record_bltu_bgeu(flag_name, less_taken):
    """BltuChip / BgeuChip (bltu.rs:111-185, bgeu.rs): the unsigned borrow of ValueA - ValueB decides the branch."""
    def record(m, c, col):
        flag, ltu = c(flag_name), col["BorrowFlag"][1]
        _sub_borrows(m, flag, col)
        _next_pc(m, flag, col, ltu if less_taken else 1 - ltu)
    return record


def _record_blt(m, c, col):
    """BltChip (blt.rs:138-241): LtFlag = the signed comparison, from the unsigned borrow and the sign bits (ValueA / ValueB's top bytes less
    Helper2[3] / Helper3[3], over 128)."""
    flag, va, vb, lt, ltu = c("IsBlt"), col["ValueA"], col["ValueB"], c("LtFlag"), col["BorrowFlag"][1]
    inv128 = pow(128, P - 2, P)
    sgn_a, sgn_b = (va[3] - col["Helper2"][3]) * inv128, (vb[3] - col["Helper3"][3]) * inv128
    _sub_borrows(m, flag, col)
    m.add_constraint(flag * (sgn_a * (1 - sgn_b) + ltu * (sgn_a * sgn_b + (1 - sgn_a) * (1 - sgn_b)) - lt))
    _next_pc(m, flag, col, lt)
    m.add_constraint(flag * (sgn_a * (1 - sgn_a)))
    m.add_constraint(flag * (sgn_b * (1 - sgn_b)))


def _record_bge(m, c, col):
    """BgeChip (bge.rs:143-268): BLT's comparison with the sign bits in SgnA / SgnB, the branch taken when LtFlag is 0."""
    flag, va, vb, lt, ltu = c("IsBge"), col["ValueA"], col["ValueB"], c("LtFlag"), col["BorrowFlag"][1]
    sgn_a, sgn_b = c("SgnA"), c("SgnB")
    _sub_borrows(m, flag, col)
    m.add_constraint(flag * (col["Helper2"][3] + sgn_a * 128 - va[3]))
    m.add_constraint(flag * (col["Helper3"][3] + sgn_b * 128 - vb[3]))
    m.add_constraint(flag * (sgn_a * (1 - sgn_b) + ltu * (sgn_a * sgn_b + (1 - sgn_a) * (1 - sgn_b)) - lt))
    _next_pc(m, flag, col, 1 - lt)


def _link(m, flag, col):
    """ValueA = Pc + 4 with CarryFlag as the carries (JalChip's and JalrChip's first two constraints)."""
    pc, va, cf = col["Pc"], col["ValueA"], col["CarryFlag"]
    m.add_constraint(flag * (4 + pc[0] + pc[1] * 256 - cf[0] * 65536 - va[0] - va[1] * 256))
    m.add_constraint(flag * (pc[2] + pc[3] * 256 + cf[0] - cf[1] * 65536 - va[2] - va[3] * 256))


def _add_halves(m, flag, x, y, carries, out):
    """out = x + y over 16-bit halves of bytes, with `carries` the carries out of the low and the high half."""
    m.add_constraint(flag * (x[0] + x[1] * 256 + y[0] + y[1] * 256 - carries[0] * 65536 - out[0] - out[1] * 256))
    m.add_constraint(flag * (x[2] + x[3] * 256 + y[2] + y[3] * 256 + carries[0] - carries[1] * 65536 - out[2] - out[3] * 256))


def _record_jal(m, c, col):
    """JalChip (jal.rs:94-160): ValueA = Pc + 4, PcNext = Pc + ValueC with BorrowFlag as its carries."""
    flag = c("IsJal")
    _link(m, flag, col)
    _add_halves(m, flag, col["ValueC"], col["Pc"], col["BorrowFlag"], col["PcNext"])


def _record_lui(m, c, col):
    """LuiChip (lui.rs:59-76): ValueA = ValueC (the immediate << 12)."""
    for k in range(4):
        m.add_constraint(c("IsLui") * (col["ValueC"][k] - col["ValueA"][k]))


def _record_auipc(m, c, col):
    """AuipcChip (auipc.rs:66-110): ValueA = Pc + ValueC with CarryFlag as the carries."""
    _add_halves(m, c("IsAuipc"), col["Pc"], col["ValueC"], col["CarryFlag"], col["ValueA"])


def _record_jalr(m, c, col):
    """JalrChip (jalr.rs:108-213): ValueA = Pc + 4; PcNextAux = ValueB + ValueC with BorrowFlag as its carries; PcNext = PcNextAux with
    bit 0 (RemAux) cleared, its low byte 2 QtAux."""
    flag, pn, aux, qt = c("IsJalr"), col["PcNext"], col["PcNextAux"], c("QtAux")
    _link(m, flag, col)
    _add_halves(m, flag, col["ValueC"], col["ValueB"], col["BorrowFlag"], aux)
    m.add_constraint(flag * (aux[0] - qt * 2 - c("RemAux")))
    m.add_constraint(flag * (qt * 2 - pn[0]))
    for k in (1, 2, 3):
        m.add_constraint(flag * (aux[k] - pn[k]))


# the decoding types and instruction chips that control=True records, in DecodingCheckChip's and BaseComponent's order (the instruction
# chips between SltChip and SllChip)
CONTROL_DECODING = [("TypeBChip", _record_type_b), ("TypeUChip", _record_type_u), ("TypeJChip", _record_type_j)]
CONTROL_CHIPS = [("BneChip", _record_beq_bne("IsBne", False)), ("BeqChip", _record_beq_bne("IsBeq", True)),
                 ("BltuChip", _record_bltu_bgeu("IsBltu", True)), ("BltChip", _record_blt), ("BgeuChip", _record_bltu_bgeu("IsBgeu", False)),
                 ("BgeChip", _record_bge), ("JalChip", _record_jal), ("LuiChip", _record_lui), ("AuipcChip", _record_auipc),
                 ("JalrChip", _record_jalr)]


def sum_of(c, names):
    """The sum of the named single-limb columns (record_main_component's ssum, for the chips recorded outside it)."""
    acc = c(names[0])
    for n in names[1:]:
        acc = acc + c(n)
    return acc


def record_main_component(air, log_size, rel, keccak=False, decoding=False, alu=False, control=False):
    """Record the main component (`MachineEval<BaseComponent>`, NexusV1Machine's docstring) into `air`: the chips in BaseComponent's order
    against the relations `rel` (name -> air.Relation: BitOp, LoadStore, ProgramCheck, RegisterCheck, Range8/16/32/128/256), then
    `finalize_logup()`.  `keccak`: the keccak extension is enabled, so KeccakChip (CustomInstructionChip, after LoadStoreChip) adds its
    booleanity constraint on IsCustomKeccak (chips/custom.rs:178-196).  `decoding`: DecodingCheckChip's type R and type I constraints
    (_record_decoding_r_i) follow CpuChip's, as DecodingCheckChip follows CpuChip in BaseComponent; its types B, J, S, U and SYS are not
    recorded.  `alu`: the arithmetic of SltuChip, SltChip, SllChip, SrlChip and SraChip (ALU_CHIPS_*) in their places among the chips, so
    that every RV32I register-register and register-immediate instruction but LUI / AUIPC is constrained.  `control` (with `alu`):
    DecodingCheck's types B, U and J (CONTROL_DECODING) after types R and I, and the arithmetic of the branch, JAL, LUI, AUIPC and JALR
    chips (CONTROL_CHIPS) between SltChip and SllChip, so that programs may branch, jump and call.  Returns (component, {column name: its
    masks})."""
    m = air.component(log_size, 2)
    pre, col = {}, {}
    for name, size in PREPROCESSED_COLUMNS + PROGRAM_COLUMNS:           # TraceEval::new: preprocessed ids, then program ids
        pre[name] = [m.get_preprocessed_column(f"{name}_{i}") for i in range(size)]
    nxt = {}
    for name, size in MAIN_COLUMNS:
        if name in ("Pc", "IsPadding"):                                 # Column::reads_next_row_mask
            pairs = [m.next_interaction_mask(A.ORIGINAL_TRACE_IDX, [0, 1]) for _ in range(size)]
            col[name], nxt[name] = [p[0] for p in pairs], [p[1] for p in pairs]
        else:
            col[name] = [m.next_trace_mask() for _ in range(size)]

    def ssum(names):
        acc = col[names[0]][0]
        for n in names[1:]:
            acc = acc + col[n][0]
        return acc

    c = lambda n: col[n][0]
    imm_c = c("ImmC")
    is_type_r = (1 - imm_c) * ssum(TYPE_R_OPS)
    is_load, is_type_s, is_type_sys, is_type_u = ssum(IS_LOAD), ssum(IS_TYPE_S), ssum(IS_TYPE_SYS), ssum(IS_TYPE_U)
    is_type_b, is_type_j = ssum(IS_TYPE_B), c("IsJal")
    alu_imm_no_shift, alu_imm_shift = imm_c * ssum(ALU_IMM_NO_SHIFT), imm_c * ssum(ALU_IMM_SHIFT)
    is_type_i_no_shift = is_load + alu_imm_no_shift + c("IsJalr")
    is_type_i = is_load + c("IsJalr") + alu_imm_no_shift + alu_imm_shift
    op_b_flag = ssum(OP_B_FLAG)
    is_pc_incremented = ssum(IS_ALU) + is_load + is_type_s + is_type_sys * (1 - c("IsSysHalt")) + is_type_u + c("IsCustomKeccak")
    reg3_accessed = (is_type_s + is_type_b + is_type_r + is_type_i + is_type_u + is_type_j
                     + is_type_sys * (c("IsSysPrivInput") + c("IsSysHeapReset") + c("IsSysStackReset")))
    vtype = {"R": is_type_r, "U": is_type_u, "INoShift": is_type_i_no_shift, "IShift": alu_imm_shift, "J": is_type_j, "B": is_type_b, "S": is_type_s}

    # ---------------- CpuChip (cpu.rs:318-566) ----------------
    is_padding, next_is_padding = c("IsPadding"), nxt["IsPadding"][0]
    next_is_first = pre["IsLast"][0]
    m.add_constraint((1 - next_is_first) * is_padding * (1 - next_is_padding))
    m.add_constraint(c("ValueAEffectiveFlagAux") * c("ValueAEffectiveFlagAuxInv") - 1)
    op_a, op_b, op_c = c("OpA"), c("OpB"), c("OpC")
    m.add_constraint(op_a * c("ValueAEffectiveFlagAux") - c("ValueAEffectiveFlag"))
    m.add_constraint(ssum(CPU_OP_FLAGS) + is_padding + c("IsCustomKeccak") - 1)
    r1a, r2a, r3a = c("Reg1Address"), c("Reg2Address"), c("Reg3Address")
    m.add_constraint((is_type_r + is_type_i) * (op_b - r1a))
    m.add_constraint(is_type_r * (op_c - r2a))
    m.add_constraint((is_type_r + is_type_i) * (op_a - r3a))
    r1v, r2v, r3v = col["Reg1ValPrev"], col["Reg2ValPrev"], col["Reg3ValPrev"]
    va, vb, vc = col["ValueA"], col["ValueB"], col["ValueC"]
    for k in (0, 2):
        m.add_constraint(op_b_flag * (r1v[k] + r1v[k + 1] * 256 - (vb[k] + vb[k + 1] * 256)))
        m.add_constraint(is_type_r * (r2v[k] + r2v[k + 1] * 256 - (vc[k] + vc[k + 1] * 256)))
    is_type_b_s = is_type_b + is_type_s
    m.add_constraint(is_type_b_s * (op_b - r1a))
    m.add_constraint(is_type_b_s * (op_a - r3a))
    for k in (0, 2):
        m.add_constraint(is_type_b_s * (r3v[k] + r3v[k + 1] * 256 - va[k] - va[k + 1] * 256))
    is_sys_halt = c("IsSysHalt")
    m.add_constraint(is_type_sys * (op_b - r1a))
    m.add_constraint(is_type_sys * (op_c - r2a))
    m.add_constraint(is_type_sys * (op_a - r3a))
    pc, pc_next, pc_carry, pc_on_next_row = col["Pc"], col["PcNext"], col["PcCarry"], nxt["Pc"]
    for k in (0, 2):
        m.add_constraint((1 - next_is_first) * (1 - next_is_padding)
                         * (pc_next[k] + pc_next[k + 1] * 256 - (pc_on_next_row[k] + pc_on_next_row[k + 1] * 256)))
    m.add_constraint(is_pc_incremented * (pc_next[0] + pc_next[1] * 256 + pc_carry[0] * 65536 - (pc[0] + pc[1] * 256) - 4))
    m.add_constraint(is_pc_incremented * (pc_next[2] + pc_next[3] * 256 + pc_carry[1] * 65536 - (pc[2] + pc[3] * 256) - pc_carry[0]))
    for k in (0, 2):
        m.add_constraint(is_type_sys * is_sys_halt * (pc[k] + pc[k + 1] * 256 - (pc_next[k] + pc_next[k + 1] * 256)))
    # ---------------- DecodingCheckChip, types R and I (chips/decoding/type_r.rs:61-409, type_i.rs:71-442) ----------------
    if decoding:
        _record_decoding_r_i(m, c, col, is_type_r, is_load, alu_imm_no_shift, alu_imm_shift, is_type_i_no_shift)
    assert not control or (alu and decoding)
    if control:
        for _name, record in CONTROL_DECODING:
            record(m, c, col)
    # ---------------- AddChip / SubChip, and SltuChip (sltu.rs) with `alu` ----------------
    cf = col["CarryFlag"]
    is_add, is_sub = c("IsAdd"), c("IsSub")
    m.add_constraint(is_add * (va[0] + va[1] * 256 + cf[0] * 65536 - (vb[0] + vb[1] * 256 + vc[0] + vc[1] * 256)))
    m.add_constraint(is_add * (va[2] + va[3] * 256 + cf[1] * 65536 - (vb[2] + vb[3] * 256 + vc[2] + vc[3] * 256 + cf[0])))
    m.add_constraint(is_sub * (va[0] + va[1] * 256 - cf[0] * 65536 - (vb[0] + vb[1] * 256 - vc[0] - vc[1] * 256)))
    m.add_constraint(is_sub * (va[2] + va[3] * 256 - cf[1] * 65536 - (vb[2] + vb[3] * 256 - vc[2] - vc[3] * 256 - cf[0])))
    if alu:
        for _name, record in ALU_CHIPS_BEFORE_BIT_OP:
            record(m, c, col)
    # ---------------- BitOpChip: lookup structure (bit_op.rs:380-431; 4 limbs x {And, Or, Xor} x {low, high nibble} = 24 fractions) ----------------
    va47, vb47, vc47 = col["ValueA4_7"], col["ValueB4_7"], col["ValueC4_7"]
    for k in range(4):
        for op_code, flag in ((1, c("IsAnd")), (2, c("IsOr")), (3, c("IsXor"))):
            m.add_to_relation(rel["BitOp"], flag, [m.const(op_code), vb[k] - vb47[k] * 16, vc[k] - vc47[k] * 16, va[k] - va47[k] * 16])
            m.add_to_relation(rel["BitOp"], flag, [m.const(op_code), vb47[k], vc47[k], va47[k]])
    # ---------------- SltChip, SllChip, SrlChip, SraChip (slt.rs, sll.rs, srl.rs, sra.rs); between SltChip and SllChip the branch, jump,
    # LUI and AUIPC chips with `control` ----------------
    if alu:
        after = list(ALU_CHIPS_AFTER_BIT_OP)
        if control:
            k = [n for n, _r in after].index("SltChip") + 1
            after = after[:k] + CONTROL_CHIPS + after[k:]
        for _name, record in after:
            record(m, c, col)
    # ---------------- LoadStoreChip: lookup structure (load_store.rs:650-685,788-903; 4 bytes x {subtract prev, add cur} = 8 fractions) ----------------
    ram1 = ssum(["IsSb", "IsSh", "IsSw", "IsLb", "IsLh", "IsLbu", "IsLhu", "IsLw"])
    ram2 = ssum(["IsSh", "IsSw", "IsLh", "IsLhu", "IsLw"])
    ram34 = ssum(["IsSw", "IsLw"])
    base, clk = col["RamBaseAddr"], pre["Clk"]
    for off, acc in ((0, ram1), (1, ram2), (2, ram34), (3, ram34)):
        addr_lo, addr_hi = base[0] + off + base[1] * 256, base[2] + base[3] * 256
        ts = col[f"Ram{off + 1}TsPrev"]
        m.add_to_relation(rel["LoadStore"], -acc, [addr_lo, addr_hi, c(f"Ram{off + 1}ValPrev"), ts[0] + ts[1] * 256, ts[2] + ts[3] * 256])
        m.add_to_relation(rel["LoadStore"], acc, [addr_lo, addr_hi, c(f"Ram{off + 1}ValCur"), clk[0] + clk[1] * 256, clk[2] + clk[3] * 256])
    # ---------------- KeccakChip in CustomInstructionChip (chips/custom.rs:178-196), with the keccak extension enabled ----------------
    if keccak:
        m.add_constraint(c("IsCustomKeccak") * (1 - c("IsCustomKeccak")))
    # ---------------- ProgramMemCheckChip (program_mem_check.rs:152-200 and the four constrain_* helpers :255-537) ----------------
    is_first = pre["IsFirst"][0]
    for k in range(4):
        m.add_constraint(is_first * (pc[k] - pre["PrgInitialPc"][k]))
    pcur, pprev, pcarry = col["ProgCtrCur"], col["ProgCtrPrev"], col["ProgCtrCarry"]
    m.add_constraint((1 - is_padding) * (pcur[0] + pcur[1] * 256 + pcarry[0] * 65536 - (pprev[0] + pprev[1] * 256 + 1)))
    m.add_constraint((1 - is_padding) * (pcur[2] + pcur[3] * 256 + pcarry[1] * 65536 - (pprev[2] + pprev[3] * 256 + pcarry[0])))
    m.add_constraint(pcarry[1])
    pm_pc, pm_word, pm_flag = pre["PrgMemoryPc"], pre["PrgMemoryWord"], pre["PrgMemoryFlag"][0]
    zero = m.const(0)
    m.add_to_relation(rel["ProgramCheck"], pm_flag, pm_pc + pm_word + [zero] * 4)                       # add_initial_digest
    m.add_to_relation(rel["ProgramCheck"], -pm_flag, pm_pc + pm_word + col["FinalPrgMemoryCtr"])        # subtract_final_digest
    iv = col["InstrVal"]
    acc_tuple = [pc[0] + pc[1] * 256, pc[2] + pc[3] * 256, iv[0] + iv[1] * 256, iv[2] + iv[3] * 256]
    m.add_to_relation(rel["ProgramCheck"], -(1 - is_padding), acc_tuple + pprev)                         # subtract_access
    m.add_to_relation(rel["ProgramCheck"], 1 - is_padding, acc_tuple + pcur)                             # add_access
    # ---------------- RegisterMemCheckChip ----------------
    vae, vaef = col["ValueAEffective"], c("ValueAEffectiveFlag")
    for k in range(4):
        m.add_constraint(vae[k] - va[k] * vaef)
    for flag, addr, ts, val in ((op_b_flag, "Reg1Address", col["Reg1TsPrev"], r1v), (is_type_r, "Reg2Address", col["Reg2TsPrev"], r2v),
                                (reg3_accessed, "Reg3Address", col["Reg3TsPrev"], r3v)):
        m.add_to_relation(rel["RegisterCheck"], -flag, [c(addr)] + ts + val)
    for flag, addr, ts, val in ((op_b_flag, "Reg1Address", pre["Reg1TsCur"], vb), (is_type_r, "Reg2Address", pre["Reg2TsCur"], vc),
                                (reg3_accessed, "Reg3Address", pre["Reg3TsCur"], vae)):
        m.add_to_relation(rel["RegisterCheck"], flag, [c(addr)] + ts + val)
    # ---------------- TimestampChip ----------------
    chm = [col["CH1Minus"], col["CH2Minus"], col["CH3Minus"]]
    for k in range(3):
        m.add_constraint(chm[k][1])
    for k, (cprev, cur, prev) in enumerate(((col["CReg1TsPrev"], pre["Reg1TsCur"], col["Reg1TsPrev"]),
                                            (col["CReg2TsPrev"], pre["Reg2TsCur"], col["Reg2TsPrev"]),
                                            (col["CReg3TsPrev"], pre["Reg3TsCur"], col["Reg3TsPrev"]))):
        m.add_constraint(cprev[0] + cprev[1] * 256 + prev[0] + prev[1] * 256 + 1 - (chm[k][0] * 65536 + cur[0] + cur[1] * 256))
        m.add_constraint(cprev[2] + cprev[3] * 256 + prev[2] + prev[3] * 256 + chm[k][0] - (chm[k][1] * 65536 + cur[2] + cur[3] * 256))
    # ---------------- RangeCheckChip = (Range8, Range16, Range32, Range128, Range256, RangeBool) ----------------
    for t, cols_ in R8:
        for n in cols_:
            m.add_to_relation(rel["Range8"], vtype[t], [c(n)])
    m.add_to_relation(rel["Range8"], ssum(ALU_IMM_SHIFT), [col["Helper1"][0]])          # Helper1MsbChecked = IsSll + IsSrl + IsSra
    for t, cols_ in R16:
        for n in cols_:
            m.add_to_relation(rel["Range16"], vtype[t], [c(n)])
    for n in R32:
        m.add_to_relation(rel["Range32"], 1, [c(n)])
    num = c("IsSlt") + c("IsBge") + c("IsBlt")
    for n in ("Helper2", "Helper3"):
        m.add_to_relation(rel["Range128"], num, [col[n][3]])
    m.add_to_relation(rel["Range128"], c("IsJalr"), [c("QtAux")])
    m.add_to_relation(rel["Range128"], c("IsSra"), [col["Helper2"][0]])
    m.add_to_relation(rel["Range128"], c("IsLh") + c("IsLb"), [c("QtAux")])
    for n in R256_WORDS:
        for limb in col[n]:
            m.add_to_relation(rel["Range256"], 1, [limb])
    for n in R256_HALF_WORDS:
        for limb in col[n]:
            m.add_to_relation(rel["Range256"], 1, [limb])
    for n in R256_BYTES:
        m.add_to_relation(rel["Range256"], 1, [c(n)])
    for n in R256_TYPE_U_BYTES:
        m.add_to_relation(rel["Range256"], is_type_u, [c(n)])
    for n in BOOL_SINGLE:
        m.add_constraint(c(n) * (c(n) - 1))
    for n in BOOL_HALF_WORD:
        for limb in col[n]:
            m.add_constraint(limb * (limb - 1))
    for t, names in (("R", BOOL_TYPE_R), ("INoShift", BOOL_TYPE_I_NO_SHIFT), ("IShift", BOOL_TYPE_I_SHIFT), ("J", BOOL_TYPE_J),
                     ("B", BOOL_TYPE_B), ("S", BOOL_TYPE_S)):
        for n in names:
            m.add_constraint(vtype[t] * c(n) * (c(n) - 1))
    m.finalize_logup()                                                     # components/mod.rs:52-54
    return m, col


class NexusV1Machine:
    """The reference's v1 main component (`MachineEval<BaseComponent>`, nexus-zkvm prover/src/components/mod.rs:39-57) recorded as data —
    the REAL trace layout (all 347 main columns of prover/src/column.rs:22-604 in enum order, `Pc` and `IsPadding` with the [0, 1] mask of
    column.rs:17-19; the 18 preprocessed + 9 program columns of column.rs:617-662 requested in TraceEval::new's order, trace/eval.rs:22-50) and an
    exact transcription of these chips, in BaseComponent's order (machine.rs:49-79):
      CpuChip               chips/cpu.rs:318-566            (padding rule, ValueAEffectiveFlag, one-hot opcode sum, register wiring for types R/I/B/S/SYS,
                                                             next-row Pc, Pc increment with carries, halt)
      AddChip, SubChip      chips/instructions/i/add.rs:98-139, sub.rs:104-146
      BitOpChip             chips/instructions/i/bit_op.rs:380-431      (its 24 four-tuple lookups; the chip has no other constraint)
      LoadStoreChip         chips/instructions/i/load_store.rs:650-685,788-903   (its 8 five-tuple RAM lookups; NOT its 39 arithmetic constraint sites)
      ProgramMemCheckChip   chips/memory_check/program_mem_check.rs:152-200,255-537   (7 constraints + 4 eight-tuple lookups)
      RegisterMemCheckChip  chips/memory_check/register_mem_check.rs:120-200,325-395   (ValueAEffective + 6 nine-tuple lookups)
      TimestampChip         chips/memory_check/timestamp.rs:73-150
      Range8/16/32/128/256  chips/range_check/*.rs          (9 + 22 + 5 + 5 + 170 = 211 lookup fractions, numerators as upstream)
    — all 253 logup fractions of the reference's main component = 1012 interaction columns (SURVEY §8), 27 / 347 / 1012 committed columns —
      RangeBoolChip         chips/range_check/range_bool.rs:143-188   (112 booleanity constraints)
    with `finalize_logup()` (one secure column per fraction) and LOG_CONSTRAINT_DEGREE = 2 (components/mod.rs:12).  NOT transcribed (their
    columns are present and committed, their arithmetic constraints are not): DecodingCheck, LoadStore's arithmetic, and the other instruction chips
    (slt, branches, jumps, lui/auipc, shifts, M extension, syscalls, custom).  Of the 8 base extensions (machine.rs:82-91) the two
    multiplicity tables the witness below needs are built (Multiplicity256, Multiplicity32: extensions/multiplicity.rs).
    The witness is a PADDING-ONLY execution (every row IsPadding = 1, the state the reference pads short programs with): all opcode flags are zero, so
    every gated constraint holds and every column the transcribed chips leave free carries random in-range values (bytes, 5-bit register indices);
    timestamps follow TimestampChip's borrow arithmetic against the preprocessed Reg{1,2,3}TsCur = 3 clk + {1,2,3}.  The CPU checker proves and verifies
    it (tests/), so the kernels are measured on the reference's mask layout, constraint
    shapes (selector x linear combination, degree <= 4) and lookup structure instead of AddMachine's toy AIR."""

    def __init__(self, log_size):
        assert log_size >= 8
        self.log_size = log_size
        air = A.Air()
        # relations in draw order (C::draw_lookup_elements walks the chips: BitOp, LoadStore, ProgramMemCheck, RegisterMemCheck, Range8, 16, 32, 128, 256)
        self.rel_bitop = air.relation("BitOp", 4)            # (op, b nibble, c nibble, a nibble)               bit_op.rs:37
        self.rel_ls = air.relation("LoadStore", 5)           # (addr lo16, addr hi16, byte, ts lo16, ts hi16)   load_store.rs:66-67
        self.rel_prog = air.relation("ProgramCheck", 8)      # (pc lo16, pc hi16, word lo16, word hi16, counter bytes x4)
        self.rel_reg = air.relation("RegisterCheck", 9)
        self.rel8, self.rel16, self.rel32 = air.relation("Range8", 1), air.relation("Range16", 1), air.relation("Range32", 1)
        self.rel128, self.rel256 = air.relation("Range128", 1), air.relation("Range256", 1)
        self.relations = [self.rel_bitop, self.rel_ls, self.rel_prog, self.rel_reg, self.rel8, self.rel16, self.rel32, self.rel128, self.rel256]
        m, _col = record_main_component(air, log_size, {r.name: r for r in self.relations})
        self.n_main = sum(s for _, s in MAIN_COLUMNS)
        # ---------------- extensions: Multiplicity256, Multiplicity32 (extensions/multiplicity.rs) ----------------
        t256 = air.component(8, 1)
        v256 = t256.get_preprocessed_column("Range256Values")
        t256.add_to_relation(self.rel256, -t256.next_trace_mask(), [v256])
        t256.finalize_logup()
        t32 = air.component(5, 1)
        v32 = t32.get_preprocessed_column("Range32Values")
        t32.add_to_relation(self.rel32, -t32.next_trace_mask(), [v32])
        t32.finalize_logup()
        self.air, self.main = air, m
        self.log_sizes = [log_size, 8, 5]
        self.words = air.serialize()

    # ---- columns ----
    def preprocessed_columns(self):
        """Tree 0 in commitment order: one (27, 2^log_size) uint8 block (every preprocessed / program column is a bit or a byte limb here) followed
        by the two table columns.  Built once and cached (the reference's PreprocessedTraces::new is host-side setup, machine.rs:144); a caller
        may replace `self._pre_cache[0]` by a pinned copy."""
        if getattr(self, "_pre_cache", None) is None:
            cols = self._preprocessed_list()
            block = np.stack([c for c in cols[:27]]).astype(np.uint8)
            self._pre_cache = [block] + cols[27:]
        return list(self._pre_cache)

    def _preprocessed_list(self):
        cols = [None] * self.air.n_columns()[0]
        ids = self.air.preprocessed_ids
        for col_id, v in main_preprocessed_columns(self.log_size).items():
            cols[ids[col_id]] = v
        cols[ids["Range256Values"]] = np.arange(256, dtype=np.uint32)
        cols[ids["Range32Values"]] = np.arange(32, dtype=np.uint32)
        return cols

    def fill_main_trace(self, seed=0):
        """The padding-only witness (class docstring).  Returns the tree-1 columns in commitment order: 347 main, then the two multiplicity columns."""
        t = padding_witness(self.log_size, seed)
        cols = [limb for name, _ in MAIN_COLUMNS for limb in t[name]]
        h256, h32 = np.zeros(256, np.int64), np.zeros(32, np.int64)
        for w in R256_WORDS + R256_HALF_WORDS + R256_BYTES:
            for limb in t[w]:
                h256 += np.bincount(limb, minlength=256)
        for w in R32:
            h32 += np.bincount(t[w][0], minlength=32)
        cols.append((h256 % P).astype(np.uint32))
        cols.append((h32 % P).astype(np.uint32))
        assert len(cols) == self.air.n_columns()[1]
        return cols

    # ---- rank-local witness generation (one proof over N GPUs at sizes whose full trace no single host process should build) ----
    def fill_main_trace_shard(self, seed, first, count, out=None):
        """Main columns [first, first + count) of a padding-only witness, generated WITHOUT building the other columns: every word draws from its
        own generator keyed by (seed, word name), so any column range gives the same values whichever rank asks.  Same constraints as
        `fill_main_trace`, a different random stream.  Returns (columns, partial Range256 histogram, partial Range32 histogram): the two
        multiplicity columns are the sums of the partial histograms over a partition of the 347 columns (`multiplicity_columns`)."""
        import zlib
        n = 1 << self.log_size
        sizes = dict(MAIN_COLUMNS)
        index = [(name, k) for name, size in MAIN_COLUMNS for k in range(size)]
        assert 0 <= first and first + count <= len(index)
        ones = {"IsPadding", "ValueAEffectiveFlagAux", "ValueAEffectiveFlagAuxInv"}
        ts_words = {f"{pre}Reg{k}TsPrev": k for k in (1, 2, 3) for pre in ("", "C")}
        ts_words.update({f"CH{k}Minus": k for k in (1, 2, 3)})
        nibbles = {"ValueA4_7": "ValueA", "ValueB4_7": "ValueB", "ValueC4_7": "ValueC"}
        free = set(R256_WORDS + R256_HALF_WORDS + R256_BYTES + ["Reg1ValPrev", "Reg2ValPrev", "Reg3ValPrev", "PcNext"]) - {"ValueAEffective"} - set(ts_words)
        rng_of = lambda tag: np.random.default_rng([int(seed) & 0xFFFFFFFF, zlib.crc32(tag.encode())])
        cache = {}

        def timestamps(k):
            if ("ts", k) not in cache:
                clk = np.arange(1, n + 1, dtype=np.uint64)
                cur = 3 * clk + k
                prev = (rng_of(f"ts{k}").integers(0, 1 << 62, n, dtype=np.uint64) % cur).astype(np.uint64)
                cc = cur - 1 - prev
                b0 = (((cc & 0xFFFF) + (prev & 0xFFFF) + 1) >> 16).astype(np.uint8)
                cache[("ts", k)] = (prev, cc, b0)
            return cache[("ts", k)]

        def word(name):
            """all limbs of one word"""
            if name in cache:
                return cache[name]
            size = sizes[name]
            if name in ones:
                limbs = [np.ones(n, np.uint8) for _ in range(size)]
            elif name in ts_words:
                prev, cc, b0 = timestamps(ts_words[name])
                src = b0 if name.startswith("CH") else (cc if name.startswith("C") else prev)
                if name.startswith("CH"):    # the borrow of the low 16 bits; the second limb (high borrow) is 0 for these values
                    limbs = [b0] + [np.zeros(n, np.uint8) for _ in range(size - 1)]
                else:
                    limbs = [((src >> (8 * i)) & 0xFF).astype(np.uint8) for i in range(4)]
            elif name in nibbles:
                limbs = [v >> 4 for v in word(nibbles[name])]
            elif name in ("OpB", "Reg1Address", "Reg2Address", "Reg3Address"):
                limbs = [rng_of(name).integers(0, 32, n, dtype=np.uint8)]
            elif name in free:
                g = rng_of(name)
                limbs = [g.integers(0, 256, n, dtype=np.uint8) for _ in range(size)]      # every limb is a byte: kept as bytes until it is stored
                if name == "Pc":
                    for limb in limbs:
                        limb[0] = 0
            else:
                limbs = [np.zeros(n, np.uint8) for _ in range(size)]
            cache[name] = limbs
            return limbs

        cols, h256, h32 = [], np.zeros(256, np.int64), np.zeros(32, np.int64)
        r256 = set(R256_WORDS + R256_HALF_WORDS + R256_BYTES)
        for i, (name, k) in enumerate(index[first:first + count]):
            col = word(name)[k]
            if out is not None:                  # a preallocated (count, 2^log_size) block, e.g. pinned host memory
                out[i] = col
            else:
                cols.append(col.astype(np.uint32))
            if name in r256:
                h256 += np.bincount(col, minlength=256)
            if name in R32:
                h32 += np.bincount(col, minlength=32)
        return (out if out is not None else cols), h256, h32

    @staticmethod
    def multiplicity_columns(h256, h32):
        """The two extension multiplicity columns (tree 1's small columns) from the histograms summed over all main columns."""
        return [(np.asarray(h256, np.int64) % P).astype(np.uint32), (np.asarray(h32, np.int64) % P).astype(np.uint32)]

    def preprocessed_shard(self, first, count, out=None):
        """Columns [first, first + count) of the 27 big preprocessed columns (a (count, 2^log_size) uint32 array; `out` = a preallocated one) and
        the two table columns; only the requested columns are generated."""
        n = 1 << self.log_size
        ids = self.air.preprocessed_ids
        tables = [np.arange(256, dtype=np.uint32), np.arange(32, dtype=np.uint32)]
        assert ids["Range256Values"] == 27 and ids["Range32Values"] == 28
        if not count:
            return None, tables
        by_id = {}
        for name in ("IsFirst", "IsLast"):
            by_id[ids[f"{name}_0"]] = (name, 0)
        for name in ("Clk", "Reg1TsCur", "Reg2TsCur", "Reg3TsCur"):
            for k in range(4):
                by_id[ids[f"{name}_{k}"]] = (name, k)
        block = out if out is not None else np.empty((count, n), np.uint32)
        clk = None
        for i in range(count):
            name, k = by_id.get(first + i, (None, 0))
            if name is None:                       # program columns: all zero (empty program)
                block[i] = 0
            elif name == "IsFirst":
                block[i] = 0; block[i, 0] = 1
            elif name == "IsLast":
                block[i] = 0; block[i, n - 1] = 1
            else:
                if clk is None:
                    clk = np.arange(1, n + 1, dtype=np.uint64)
                v = clk if name == "Clk" else 3 * clk + int(name[3])
                block[i] = (v >> (8 * k)) & 0xFF
        return block, tables

    def column_log_sizes(self):
        return self.air.column_log_sizes()
