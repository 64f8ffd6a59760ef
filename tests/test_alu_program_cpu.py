"""A straight-line program of every RV32I register-register and register-immediate instruction but LUI / AUIPC, proven as an executing v1
trace (add_chain.AluMachine), without a GPU: the encoders and the emulator against an independent numpy restatement of RV32I and known
answers, oracle proofs whose verifier accepts and whose claimed sums cancel with BitOpMultiplicity counted, no constraint failing on the
executing witness, every constraint SltuChip, SltChip, SllChip, SrlChip and SraChip add broken by some single-cell corruption, their degrees,
the device fill's per-row code (csrc/v1_trace.cuh, compiled as host C++) equal to the numpy columns on ALU programs and on edge step records
of all 19 opcodes, and the fill kernel and the machine's generated kernels compiled for sm_90a."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from nexus_zkvm_b200 import add_chain as AC
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200 import nexus_v1 as V
from tests.keccak_side_notes import finalized_src_rows
from tests.oracle_backend import OracleBackend, verify
from tests.test_add_chain_cpu import CSRC, DRIVER, NVCC, OFFSETS, _decode, _failures
from tests.test_add_chain_random_witness_cpu import edgy_u32
from tests.test_d2_high_degree_cpu import _walk_degrees

u32p = C.POINTER(C.c_uint32)
F = {n: i for i, n in enumerate(AC.STEP_FIELDS)}
# the constraints each new chip adds, read from the sources' add_constraint sites with the loops expanded
CHIP_CONSTRAINTS = {"SltuChip": 6, "SltChip": 8, "SllChip": 10, "SrlChip": 14, "SraChip": 21}


# ---- encoders and emulator

def test_every_encoding_decodes_back():
    rng = np.random.default_rng(1)
    for op, (name, ty, f3, f7, _flag) in enumerate(AC.OPCODES):
        enc = getattr(AC, f"encode_{name.lower()}")
        for _ in range(50):
            rd, rs1 = int(rng.integers(0, 32)), int(rng.integers(0, 32))
            c = int(rng.integers(0, 32)) if ty != "I" else int(rng.choice([-2048, -1, 0, 2047, int(rng.integers(-2048, 2048))]))
            w = enc(rd, rs1, c)
            assert w == AC.encode(op, rd, rs1, c)
            d = _decode(w)
            assert (d["rd"], d["rs1"], d["funct3"]) == (rd, rs1, f3), name
            if ty == "R":
                assert (d["opcode"], d["rs2"], d["funct7"]) == (0b0110011, c, f7), name
            elif ty == "I":
                assert (d["opcode"], d["imm"]) == (0b0010011, c), name
            else:
                assert (d["opcode"], d["rs2"], d["funct7"]) == (0b0010011, c, f7), name


def _numpy_rv32i(ops):
    """RV32I restated on numpy int32 / uint32 registers: [(rs1 value, operand c, result)] per step and the final registers."""
    x = np.zeros(32, np.uint32)
    out = []
    with np.errstate(over="ignore"):
        for op, rd, rs1, c in ops:
            name, ty = AC.OPCODES[op][:2]
            b = x[rs1]
            if ty == "R":
                cv = x[c]
            elif ty == "I":
                cv = np.int32(c).astype(np.uint32)
            else:
                cv = np.uint32(c)
            sh = np.uint32(cv & np.uint32(31))
            sb, sc = b.astype(np.int32), cv.astype(np.int32)
            r = {"ADD": lambda: b + cv, "SUB": lambda: b - cv, "SLL": lambda: b << sh, "SLT": lambda: np.uint32(sb < sc),
                 "SLTU": lambda: np.uint32(b < cv), "XOR": lambda: b ^ cv, "SRL": lambda: b >> sh,
                 "SRA": lambda: (sb >> sh.astype(np.int32)).astype(np.uint32), "OR": lambda: b | cv, "AND": lambda: b & cv}
            key = "SLTU" if name == "SLTIU" else name if ty == "R" else name[:-1]
            res = np.uint32(r[key]())
            out.append((int(b), int(cv), int(res)))
            if rd:
                x[rd] = res
    return out, x


@pytest.mark.parametrize("seed", [0, 7])
def test_emulator_matches_a_numpy_restatement(seed):
    words, ops = AC.alu_program(12, seed=seed)
    steps, (final, _ts) = AC.execute(ops)
    want, x = _numpy_rv32i(ops)
    assert np.array_equal(steps[F["value_b"]], [w[0] for w in want]) and np.array_equal(steps[F["value_c"]], [w[1] for w in want])
    assert np.array_equal(AC.alu_np(steps[F["opcode"]], steps[F["value_b"]], steps[F["value_c"]]), [w[2] for w in want])
    assert np.array_equal(final, x) and np.array_equal(steps[F["word"]], words)
    assert set(int(o) for o in steps[F["opcode"]]) == set(range(19))
    # the prefix's edge cases are there: 0, 1, -1, 0x7FFFFFFF, 0x80000000 as operands, shifts by 0 and 31, an R shift with rs2 above 31,
    # the immediate -2048 and a write to x0
    assert {0, 1, 0xFFFFFFFF, 0x7FFFFFFF, 0x80000000} <= set(int(v) for v in steps[F["value_b"]])
    shifts = np.isin(steps[F["opcode"]], [AC.OP_SLL, AC.OP_SRL, AC.OP_SRA, AC.OP_SLLI, AC.OP_SRLI, AC.OP_SRAI])
    assert {0, 31} <= set(int(v) & 31 for v in steps[F["value_c"]][shifts])
    r_shift = np.isin(steps[F["opcode"]], [AC.OP_SLL, AC.OP_SRL, AC.OP_SRA])
    assert np.any(steps[F["value_c"]][r_shift] > 31)
    assert 0xFFFFF800 in set(int(v) for v in steps[F["op_c"]]) and np.any(steps[F["rd"]] == 0)


def _run(ops, reg=None):
    _steps, (final, _ts) = AC.execute(ops)
    return [int(v) for v in final] if reg is None else int(final[reg])


def test_known_answers():
    li = [(AC.OP_ADDI, 1, 0, 1), (AC.OP_SLLI, 2, 1, 31)]                          # x2 = 0x80000000
    assert _run(li + [(AC.OP_SRAI, 3, 2, 31)], 3) == 0xFFFFFFFF
    for v in (0, 1, 5):
        pre = [(AC.OP_ADDI, 4, 0, v)]
        assert _run(pre + [(AC.OP_SLTIU, 5, 4, 1)], 5) == int(v == 0)
        assert _run(pre + [(AC.OP_SLTU, 5, 0, 4)], 5) == int(v != 0)
    for v in (0, -1, 1234, -2048):
        assert _run([(AC.OP_ADDI, 4, 0, v), (AC.OP_XORI, 5, 4, -1)], 5) == ~v & 0xFFFFFFFF
    base = [(AC.OP_ADDI, 6, 0, 1234), (AC.OP_ADDI, 7, 0, 33), (AC.OP_ADDI, 8, 0, 1)]
    assert _run(base + [(AC.OP_SLL, 9, 6, 7)], 9) == _run(base + [(AC.OP_SLL, 9, 6, 8)], 9) == 2468
    assert _run([(AC.OP_ADDI, 0, 0, 5), (AC.OP_ADD, 1, 0, 0)]) == [0] * 32           # x0 stays 0


# ---- oracle proofs and the constraints

@pytest.fixture(scope="module", params=[(9, None), (10, 700)], ids=["2^9", "700-in-2^10"])
def machine(request):
    m = AC.AluMachine(*request.param)
    return m, m.fill_main_trace()


def test_oracle_proves_verifies_and_sums_cancel(machine):
    m, t1 = machine
    assert m.log_sizes == [m.log_size, 5, 8, 4, 4, 4, 5, 7, 8]
    assert all(np.any(c) for c in t1[347 + 8:347 + 11])                            # BitOpMultiplicity's And, Or, Xor columns
    proof, claimed, aux = M.prove(m, OracleBackend(), t1, None, associated_data=b"alu program")
    verify(m, proof, aux)
    assert len(claimed) == 9 and M.verify_claimed_sums(claimed)
    assert claimed[0] != (0, 0, 0, 0) and claimed[2] != (0, 0, 0, 0)


def test_no_constraint_fails_on_the_executing_witness(machine):
    m, t1 = machine
    assert all(not v for v in _failures(m, t1).values())


def chip_ranges(log_size=9, **kw):
    """(AluMachine, {chip name: range of its constraints in the main component})."""
    seen = {}

    def wrap(name, record):
        def wrapped(comp, *a):
            first = len(comp.constraints)
            record(comp, *a)
            seen[name] = range(first, len(comp.constraints))
        return wrapped

    before, after = V.ALU_CHIPS_BEFORE_BIT_OP, V.ALU_CHIPS_AFTER_BIT_OP
    V.ALU_CHIPS_BEFORE_BIT_OP = [(n, wrap(n, r)) for n, r in before]
    V.ALU_CHIPS_AFTER_BIT_OP = [(n, wrap(n, r)) for n, r in after]
    try:
        m = AC.AluMachine(log_size, **kw)
    finally:
        V.ALU_CHIPS_BEFORE_BIT_OP, V.ALU_CHIPS_AFTER_BIT_OP = before, after
    return m, seen


def test_chip_constraint_counts_and_degrees():
    """Each chip adds its pinned number of constraints, 59 in all after the ADD chain's 486; every one is a selector times at most three
    factors (degree <= 4), so the ones of degree 3 and 4 go to the half-coset D2 kernel (air.h:constraint_degrees counts as _walk_degrees)."""
    m, seen = chip_ranges()
    assert {k: len(v) for k, v in seen.items()} == CHIP_CONSTRAINTS
    deg = _walk_degrees(m.air.components[0])
    assert len(deg) == 486 + 59
    new = [deg[i] for r in seen.values() for i in r]
    assert max(new) == 4 and min(new) == 2
    assert sum(d > 2 for d in new) == 34


def _corruptions(m, t1):
    """Single-cell corruptions, one per row: every column the chips read, +1 on a row of each opcode that the chip holds."""
    ops = m.steps[F["opcode"]]
    chip_ops = {"IsSltu": [AC.OP_SLTU, AC.OP_SLTIU], "IsSlt": [AC.OP_SLT, AC.OP_SLTI], "IsSll": [AC.OP_SLL, AC.OP_SLLI],
                "IsSrl": [AC.OP_SRL, AC.OP_SRLI], "IsSra": [AC.OP_SRA, AC.OP_SRAI]}
    cols = [("ValueA", k) for k in range(4)] + [("ValueB", k) for k in range(4)] + [("ValueC", k) for k in range(4)]
    cols += [(n, k) for n in ("CarryFlag",) for k in range(2)] + [(n, k) for n in ("Helper1", "Helper2", "Helper3", "Rem", "Qt", "RemDiff")
                                                                     for k in range(4)]
    cols += [(n, 0) for n in ("SgnB", "SgnC", "ShiftBit1", "ShiftBit2", "ShiftBit3", "ShiftBit4", "ShiftBit5", "Exp1_3", "Exp", "SraDegreeAux")]
    used = set()
    bad = [c.copy() for c in t1]
    for flag, which in chip_ops.items():
        rows = [r for r in range(1, m.n_steps) if ops[r] in which]
        rows = [r for r in rows if r not in used]
        for (name, limb), row in zip(cols, rows):
            used.add(row)
            c = bad[OFFSETS[name] + limb]
            c[row] = (int(c[row]) + 1) % ((1 << 31) - 1)
        assert len(rows) >= len(cols), flag
    return bad


def test_every_new_chip_constraint_is_broken_by_some_corruption():
    m, seen = chip_ranges(10)
    t1 = m.fill_main_trace()
    fails = {i for i, _a, _r in _failures(m, _corruptions(m, t1), comps=[0])[0]}
    missing = {k: [i for i in r if i not in fails] for k, r in seen.items()}
    assert not any(missing.values()), missing


# ---- the device fill's row code

@pytest.fixture(scope="module")
def host_fill(tmp_path_factory):
    d = tmp_path_factory.mktemp("v1_fill")
    src, so = d / "fill.cc", d / "fill.so"
    src.write_text(DRIVER)
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-w", "-I", CSRC, str(src), "-o", str(so)], check=True)
    lib = C.CDLL(str(so))

    def run(steps, final_ctr, log_size):
        st = np.ascontiguousarray(steps, np.uint32)
        ctr = np.ascontiguousarray(final_ctr, np.uint32)
        out = np.zeros((347, 1 << log_size), np.uint32)                       # the device clears the batch first
        lib.v1_fill_host(C.c_uint32(st.shape[1]), st.ctypes.data_as(u32p), C.c_uint32(ctr.size), ctr.ctypes.data_as(u32p), C.c_uint32(log_size),
                         out.ctypes.data_as(u32p))
        return out
    return run


def _want(steps, final_ctr, log_size):
    t = AC.main_columns(steps, final_ctr, log_size)
    return np.stack([limb for name, _ in V.MAIN_COLUMNS for limb in t[name]])[:, finalized_src_rows(log_size)]


@pytest.mark.parametrize("ls,n,seed", [(8, None, 0), (10, 700, 1), (12, None, 2), (9, 40, 3)])
def test_host_fill_equals_the_numpy_columns(host_fill, ls, n, seed):
    m = AC.AluMachine(ls, n, seed=seed)
    want = np.stack(m.fill_main_trace()[:347])[:, finalized_src_rows(ls)]
    bad = np.argwhere(host_fill(m.steps, m.final_ctr, ls) != want)
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"


def alu_edge_steps(log_size, n_steps, seed):
    """A step record of n_steps steps over all 19 opcodes that nb200_v1_alu_trace's host check accepts (valid_alu_steps), its operands
    from the edges of u32 (edgy_u32) rather than from an execution, with shift amounts 0 and 31 and immediates -2048 and 2047 among them."""
    rng = np.random.default_rng(seed)
    s = np.zeros((len(AC.STEP_FIELDS), n_steps), np.uint64)
    op = rng.integers(0, 19, n_steps)
    op[:19] = np.arange(19)
    ty = np.array(AC.OP_TYPE)[op]
    s[F["opcode"]] = op
    for f in ("pc", "word", "value_b", "rd_prev"):
        s[F[f]] = edgy_u32(rng, n_steps)
    s[F["rd"]], s[F["rs1"]] = rng.integers(0, 32, n_steps), rng.integers(0, 32, n_steps)
    imm = np.where(rng.integers(0, 3, n_steps) == 0, rng.choice([-2048, 2047, -1, 0], n_steps), rng.integers(-2048, 2048, n_steps))
    shamt = np.where(rng.integers(0, 3, n_steps) == 0, rng.choice([0, 31], n_steps), rng.integers(0, 32, n_steps))
    s[F["op_c"]] = np.select([ty == "R", ty == "I"], [rng.integers(0, 32, n_steps), imm.astype(np.int64) & 0xFFFFFFFF], shamt)
    s[F["value_c"]] = np.where(ty == "R", edgy_u32(rng, n_steps), s[F["op_c"]])
    clk = np.arange(1, n_steps + 1, dtype=np.uint64)
    for k in (1, 2, 3):
        s[F[f"ts{k}_prev"]] = (rng.random(n_steps) * (3 * clk + k)).astype(np.uint64)
    s[F["pc_ctr_prev"]] = np.minimum(edgy_u32(rng, n_steps), 0xFFFFFFFE)
    steps = s.astype(np.uint32)
    final_ctr = rng.integers(0, 1 << 32, min(n_steps, 1 << log_size), dtype=np.uint64).astype(np.uint32)
    assert valid_alu_steps(steps, final_ctr, log_size)
    return steps, final_ctr


def valid_alu_steps(steps, final_ctr, log_size):
    """nb200_v1_alu_trace's host check (csrc/v1_trace.cu), restated."""
    n_steps = steps.shape[1]
    s = {f: steps[i].astype(np.uint64) for i, f in enumerate(AC.STEP_FIELDS)}
    if not (n_steps <= 1 << log_size and final_ctr.size <= 1 << log_size and np.all(s["opcode"] < 19)):
        return False
    ty = np.array(AC.OP_TYPE)[s["opcode"].astype(np.int64)]
    imm = steps[F["op_c"]].view(np.int32)
    clk = np.arange(1, n_steps + 1, dtype=np.uint64)
    return bool(np.all(s["rd"] < 32) and np.all(s["rs1"] < 32) and np.all((ty == "I") | (s["op_c"] < 32))
                and np.all((ty != "I") | ((imm >= -2048) & (imm < 2048))) and np.all(s["pc_ctr_prev"] != 0xFFFFFFFF)
                and all(np.all(s[f"ts{k}_prev"] < 3 * clk + k) for k in (1, 2, 3)))


@pytest.mark.parametrize("ls,n_steps", [(8, 256), (10, 900), (12, 4096), (16, 40000)])
def test_host_fill_on_edge_step_records(host_fill, ls, n_steps):
    """(16, 40000): from the 21845th step on the timestamps pass 2^16, and the CH*Minus borrow is taken."""
    steps, final_ctr = alu_edge_steps(ls, n_steps, seed=ls)
    want = _want(steps, final_ctr, ls)
    bad = np.argwhere(host_fill(steps, final_ctr, ls) != want)
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"
    for name in ("SgnB", "SgnC", "ShiftBit5", "SraDegreeAux", "Exp"):                # the edges show in the chips' helpers
        assert want[OFFSETS[name]].any(), name


# ---- sm_90a builds

def _ptxas_blocks(src_path, out_path, cubin=False):
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++", "-Xcudafe",
                        "--diag_suppress=177", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-x", "cu", "-cubin" if cubin else "-c",
                        str(src_path), "-o", str(out_path)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    return {b.split("'")[0]: b for b in re.split(r"Compiling entry function '", r.stderr)[1:]}


def _spills(block):
    return max(int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", block))


def test_fill_kernel_compiles_for_sm90a_without_spills(tmp_path):
    blocks = _ptxas_blocks(os.path.join(CSRC, "v1_trace.cu"), tmp_path / "v1_trace.o")
    (name,) = [n for n in blocks if "v1_main_trace_kernel" in n]
    assert _spills(blocks[name]) == 0, blocks[name]


def test_generated_kernels_compile_for_sm90a(tmp_path):
    """The kernels generated for AluMachine's main component (the only component whose AIR differs from the ADD chain's): constraints
    (D1), LogUp, D2, check and table count build for sm_90a.  Their spill bytes are printed (pytest -s) beside the ADD chain's."""
    import nexus_zkvm_b200 as nb
    from tests import test_constraint_check_cpu as chk
    from tests.test_d2_high_degree_cpu import _load, _source
    from tests.test_table_multiplicities_cpu import count_source
    report = {}
    for label, m in (("add_chain", AC.AddChainMachine(8)), ("alu", AC.AluMachine(8))):
        h = _load(m.words)
        try:
            srcs = {"d1": _source(h, 0, 0), "logup": _source(h, 0, 1), "d2": _source(h, 0, 2), "check": chk.kernel_source(m.words, 0)[1],
                    "count": count_source(h, 0)[1]}
        finally:
            nb.lib().nb200_air_free(h)
        for kind, src in srcs.items():
            assert src, (label, kind)
            path = tmp_path / f"{label}_{kind}.cu"
            path.write_bytes(src if isinstance(src, bytes) else src.encode())
            blocks = _ptxas_blocks(path, tmp_path / f"{label}_{kind}.cubin", cubin=True)
            assert blocks, (label, kind)
            report[(label, kind)] = max(_spills(b) for b in blocks.values())
    print("spill bytes of the main component's generated kernels, sm_90a:", report)
