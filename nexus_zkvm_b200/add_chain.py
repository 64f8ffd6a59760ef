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
   2 BitOpMultiplicity           no bit-op lookup here: zero
   3 RamInitFinal                2^4 zero rows
   4-8 Multiplicity8/16/32/128/256
Relations: BitOp, LoadStore, ProgramCheck, RegisterCheck, Range8, 16, 32, 128, 256 (draw_lookup_elements over BaseComponent).

The step record (`STEP_FIELDS`, one uint32 row per field, one column per step) is what the device fill (nb200_v1_main_trace,
csrc/v1_trace.{cu,cuh}) takes; `fill_main_trace` is its numpy reference, a port of the per-row fills of CpuChip (cpu.rs:36-316), DecodingCheck
R / I (type_r.rs:25-60, type_i.rs:29-69), AddChip (add.rs:64-100), ProgramMemCheck (program_mem_check.rs:44-100), RegisterMemCheck
(register_mem_check.rs:53-117) and Timestamp (timestamp.rs:33-75) for ADD, ADDI and padding rows."""
import numpy as np

from . import air as A
from . import nexus_v1 as V
from . import whole_machine as W

P = (1 << 31) - 1
ELF_TEXT_START = 136                       # PUBLIC_OUTPUT_ADDRESS_LOCATION + 4 (common/src/constants/mod.rs:8-10)
NUM_REGISTERS = 32
OP_ADD, OP_ADDI = 0, 1
# the step record, field by field (nb200_v1_main_trace's `steps`): op_c is rs2 for ADD and the sign-extended immediate for ADDI; the
# three previous timestamps are those of the rs1 read, the rs2 read and the rd write (0 when the access does not happen); pc_ctr_prev is
# how often the instruction at pc was executed before
STEP_FIELDS = ["pc", "word", "opcode", "rd", "rs1", "op_c", "value_b", "value_c", "rd_prev", "ts1_prev", "ts2_prev", "ts3_prev", "pc_ctr_prev"]


def encode_add(rd, rs1, rs2):
    return (rs2 << 20) | (rs1 << 15) | (rd << 7) | 0b0110011


def encode_addi(rd, rs1, imm):
    return ((imm & 0xFFF) << 20) | (rs1 << 15) | (rd << 7) | 0b0010011


def add_chain_program(log_size, n_instructions=None):
    """The ADD chain's first `n_instructions` (default 2^log_size) instructions: (words uint32, [(opcode, rd, rs1, rs2 or imm)])."""
    n = (1 << log_size) if n_instructions is None else int(n_instructions)
    ops, (i, j, k) = [(OP_ADDI, 1, 0, 1)], (0, 1, 2)
    while len(ops) < n:
        ops.append((OP_ADD, k, j, i))
        i, j, k = (i + 1) % NUM_REGISTERS, (j + 1) % NUM_REGISTERS, (k + 1) % NUM_REGISTERS
    ops = ops[:n]
    words = np.array([encode_add(rd, rs1, c) if op == OP_ADD else encode_addi(rd, rs1, c) for op, rd, rs1, c in ops], np.uint32)
    return words, ops


def execute(ops, base=ELF_TEXT_START):
    """Run a straight-line ADD / ADDI program once from the all-zero register file.  Returns (steps, final registers) where steps is
    (len(STEP_FIELDS), n_steps) uint32 in STEP_FIELDS order and final registers = (values, timestamps) of the 32 registers after the last
    step (FinalReg's rows).  Step t (clk = t + 1) reads rs1 at 3 clk + 1, rs2 at 3 clk + 2 and writes rd at 3 clk + 3 (preprocessed.rs:75-100);
    a write to x0 stores 0 (ValueAEffective)."""
    val, ts = [0] * NUM_REGISTERS, [0] * NUM_REGISTERS
    pc_ctr = {}
    cols = [[] for _ in STEP_FIELDS]
    words = [encode_add(rd, rs1, c) if op == OP_ADD else encode_addi(rd, rs1, c) for op, rd, rs1, c in ops]
    for t, ((op, rd, rs1, c), word) in enumerate(zip(ops, words)):
        assert op in (OP_ADD, OP_ADDI) and 0 <= rd < 32 and 0 <= rs1 < 32
        clk = t + 1
        pc = base + 4 * t
        b, ts1 = val[rs1], ts[rs1]
        ts[rs1] = 3 * clk + 1
        if op == OP_ADD:
            assert 0 <= c < 32
            cv, ts2 = val[c], ts[c]
            ts[c] = 3 * clk + 2
            op_c = c
        else:
            op_c = (c & 0xFFF) - ((c & 0x800) << 1) & 0xFFFFFFFF        # the 12-bit immediate, sign-extended
            cv, ts2 = op_c, 0
        a = (b + cv) & 0xFFFFFFFF
        rd_prev, ts3 = val[rd], ts[rd]
        val[rd], ts[rd] = (a if rd else 0), 3 * clk + 3
        ctr = pc_ctr.get(pc, 0)
        pc_ctr[pc] = ctr + 1
        for col, v in zip(cols, (pc, word, op, rd, rs1, op_c, b, cv, rd_prev, ts1, ts2, ts3, ctr)):
            col.append(v)
    steps = np.array(cols, dtype=np.uint32).reshape(len(STEP_FIELDS), len(ops))
    return steps, (np.array(val, np.uint32), np.array(ts, np.uint32))


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

    is_add, is_addi = s["opcode"] == OP_ADD, s["opcode"] == OP_ADDI
    rd, rs1 = s["rd"], s["rs1"]
    a = (s["value_b"] + s["value_c"]) & np.uint64(0xFFFFFFFF)
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
    put("PcNext", _le(s["pc"] + 4))
    put("InstrVal", _le(s["word"]))
    put("IsAdd", [np.ones(m, np.uint32)])
    put("ValueB", _le(s["value_b"]))
    put("ValueC", _le(s["value_c"]))
    put("OpA", [rd])
    put("OpB", [rs1])
    put("OpC", [np.where(is_add, s["op_c"], s["op_c"] & 0xFFF)])
    put("ImmC", [is_addi.astype(np.uint32)])
    put("Reg1Address", [rs1])
    put("Reg2Address", [np.where(is_add, s["op_c"], 0)])
    put("Reg3Address", [rd])
    # DecodingCheck, types R (ADD) and I (ADDI): type_r.rs:43-59, type_i.rs:46-68
    c = s["op_c"]
    put("OpA0", [rd & 1]); put("OpA1_4", [(rd >> 1) & 0xF])
    put("OpB0", [rs1 & 1]); put("OpB1_4", [(rs1 >> 1) & 0xF])
    put("OpC0_3", [c & 0xF])
    put("OpC4", [np.where(is_add, (c >> 4) & 1, 0)])
    put("OpC4_7", [np.where(is_addi, (c >> 4) & 0xF, 0)])
    put("OpC8_10", [np.where(is_addi, (c >> 8) & 0x7, 0)])
    put("OpC11", [np.where(is_addi, (c >> 11) & 1, 0)])
    # AddChip (add.rs:64-100)
    put("ValueA", _le(a))
    put("CarryFlag", _carries16(s["value_b"], s["value_c"]))
    # ProgramMemCheck (program_mem_check.rs:44-100): the counters of this access; FinalPrgMemoryCtr on the program's rows
    put("ProgCtrPrev", _le(s["pc_ctr_prev"]))
    put("ProgCtrCur", _le(s["pc_ctr_prev"] + 1))
    put("ProgCtrCarry", _carries16(s["pc_ctr_prev"], 1))
    put("FinalPrgMemoryCtr", _le(final_ctr), slice(0, len(final_ctr)))
    # RegisterMemCheck (register_mem_check.rs:53-117): ValueAEffective and the previous values / timestamps of the accessed registers
    put("ValueAEffective", _le(a * flag))
    put("Reg1ValPrev", _le(s["value_b"]))
    put("Reg2ValPrev", _le(np.where(is_add, s["value_c"], 0)))
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


def _count(hist, values):
    hist += np.bincount(np.asarray(values, np.int64), minlength=hist.size)


def table_counts(t, ram_cols):
    """The multiplicities of Range8, 16, 32, 128, 256 as the main component's lookups (nexus_v1.record_main_component's range checks, their
    numerators on ADD, ADDI and padding rows) and RamInitFinal's nine Range256 lookups per row count them."""
    h = {r: np.zeros(length, np.int64) for r, length, _ls in W.MULTIPLICITY_TABLES}
    is_add = (t["IsAdd"][0] == 1) & (t["ImmC"][0] == 0)
    is_addi = (t["IsAdd"][0] == 1) & (t["ImmC"][0] == 1)
    for w in V.R256_WORDS + V.R256_HALF_WORDS + V.R256_BYTES:
        for limb in t[w]:
            _count(h["Range256"], limb)
    for v in ram_cols[[0, 1, 2, 3, 5, 6, 7, 8, 9]]:
        _count(h["Range256"], v)
    for w in V.R32:
        _count(h["Range32"], t[w][0])
    vtype = {"R": is_add, "INoShift": is_addi}
    for ty, names in V.R16:
        for nm in names:
            if ty in vtype:
                _count(h["Range16"], t[nm][0][vtype[ty]])
    for ty, names in V.R8:
        for nm in names:
            if ty in vtype:
                _count(h["Range8"], t[nm][0][vtype[ty]])
    return h


class AddChainMachine:
    """The ADD chain of the module docstring at 2^log_size rows, `n_steps` executed steps (default 2^log_size); `ops` = [(opcode, rd, rs1,
    rs2 or imm)] runs another straight-line ADD / ADDI program instead.  Same interface as the other
    machines: `air`, `words`, `relations`, `log_sizes`, `preprocessed_columns()`, `fill_main_trace()` (tree 1 in commitment order, the
    multiplicity columns counted on the host), `column_log_sizes()`, and `device_trees(ctx)` (the main trace filled on the device by
    nb200_v1_main_trace, the multiplicities counted there)."""

    def __init__(self, log_size, n_steps=None, ops=None):
        assert log_size >= 8
        self.log_size = self.log_size_main = log_size
        if ops is None:
            self.n_steps = (1 << log_size) if n_steps is None else int(n_steps)
            self.program, ops = add_chain_program(log_size, self.n_steps)
        else:                                                                 # another straight-line ADD / ADDI program
            self.n_steps = len(ops)
        assert 1 <= self.n_steps <= 1 << log_size
        self.steps, (self.final_values, self.final_timestamps) = execute(ops)
        self.program = self.steps[STEP_FIELDS.index("word")].copy()
        # every instruction runs once: the final counter of each program row (program_mem_check.rs:88-99)
        self.final_ctr = np.ones(self.program.size, np.uint32)
        self.ram_log_size = W.ram_log_size(0)
        air = A.Air()
        names = [("BitOp", 4), ("LoadStore", 5), ("ProgramCheck", 8), ("RegisterCheck", 9), ("Range8", 1), ("Range16", 1), ("Range32", 1),
                 ("Range128", 1), ("Range256", 1)]
        self.relations = [air.relation(n, s) for n, s in names]
        rel = {r.name: r for r in self.relations}
        self.main, _col = V.record_main_component(air, log_size, rel, decoding=True)
        self.final_reg = W._final_reg_component(air, rel["RegisterCheck"])
        self.bit_op = W._bit_op_component(air, rel["BitOp"])
        self.ram = W._ram_init_final_component(air, self.ram_log_size, rel["LoadStore"], rel["Range256"])
        self.tables = [W._multiplicity_component(air, rel[r], length, ls) for r, length, ls in W.MULTIPLICITY_TABLES]
        self.air = air
        self.log_sizes = [log_size, W.FINAL_REG_LOG_SIZE, W.BIT_OP_LOG_SIZE, self.ram_log_size] + [ls for _r, _l, ls in W.MULTIPLICITY_TABLES]
        self.words = air.serialize()
        self._main = None

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
            cols += [np.zeros(1 << W.BIT_OP_LOG_SIZE, np.uint32) for _ in range(3)]
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
        columns uploaded, the main component filled on the device from the step record (nb200_v1_main_trace; `out` = a batch of 347 columns
        of 2^log_size rows to reuse), RamInitFinal and BitOpMultiplicity zero, and every table column counted on the device from the filled
        trace (nb200_table_multiplicities_first_row)."""
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
        tree1 = [ctx.v1_main_trace(self.steps, self.final_ctr, self.log_size, out=out)]
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
