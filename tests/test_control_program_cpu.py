"""Looping RV32I programs with branches, JAL, JALR, LUI and AUIPC proven as executing v1 traces (add_chain.ControlMachine), without a GPU:
the new encoders, the pc-driven emulator (`run`) against a numpy restatement of RV32I, known answers and `execute`, its refusal of a pc
outside the program, oracle proofs whose verifier accepts and whose claimed sums cancel, no constraint failing on the executing witness,
every constraint of DecodingCheck B / U / J and of the ten new chips broken by some single-cell corruption, their counts and degrees, the
device fill's per-row code (csrc/v1_trace.cuh, compiled as host C++) equal to the numpy columns on programs and on edge step records of all
29 opcodes, and the fill kernel and the machine's generated kernels compiled for sm_90a."""
import os

import numpy as np
import pytest

from nexus_zkvm_b200 import add_chain as AC
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200 import nexus_v1 as V
from tests.keccak_side_notes import finalized_src_rows
from tests.oracle_backend import OracleBackend, verify
from tests.test_add_chain_cpu import CSRC, OFFSETS, _decode, _failures
from tests.test_add_chain_random_witness_cpu import edgy_u32
from tests.test_alu_program_cpu import _ptxas_blocks, _spills, _want, host_fill  # noqa: F401  (host_fill is a fixture)
from tests.test_d2_high_degree_cpu import _walk_degrees

F = {n: i for i, n in enumerate(AC.STEP_FIELDS)}
# the constraints each decoding type and chip adds, read from the sources' add_constraint sites with the loops expanded
CHIP_CONSTRAINTS = {"TypeBChip": 16, "TypeUChip": 16, "TypeJChip": 15, "BneChip": 9, "BeqChip": 9, "BltuChip": 4, "BltChip": 7,
                    "BgeuChip": 4, "BgeChip": 7, "JalChip": 4, "LuiChip": 4, "AuipcChip": 2, "JalrChip": 9}
N_NEW = sum(CHIP_CONSTRAINTS.values())                                          # 106, after the ALU program's 545


def _sext(x, bits):
    x &= (1 << bits) - 1
    return x - ((x >> (bits - 1)) << bits)


# ---- encoders and emulator

def test_every_new_encoding_decodes_back():
    rng = np.random.default_rng(2)
    for k, (name, ty, f3, _flag) in enumerate(AC.CONTROL_OPCODES):
        op = AC.OP_BEQ + k
        for j in range(60):
            a, b = int(rng.integers(0, 32)), int(rng.integers(0, 32))
            if ty == "B":
                c = [-4096, 4094, -2, 0][j] if j < 4 else 2 * int(rng.integers(-2048, 2048))
                w = getattr(AC, f"encode_{name.lower()}")(a, b, c)
                d = _decode(w)
                imm = _sext(((w >> 31) << 12) | (((w >> 7) & 1) << 11) | (((w >> 25) & 0x3F) << 5) | (((w >> 8) & 0xF) << 1), 13)
                assert (d["opcode"], d["funct3"], d["rs1"], d["rs2"], imm) == (0b1100011, f3, a, b, c), name
            elif ty == "J":
                c = [-(1 << 20), (1 << 20) - 2, -4, 0][j] if j < 4 else 2 * int(rng.integers(-(1 << 19), 1 << 19))
                w = AC.encode_jal(a, c)
                imm = _sext(((w >> 31) << 20) | (((w >> 12) & 0xFF) << 12) | (((w >> 20) & 1) << 11) | (((w >> 21) & 0x3FF) << 1), 21)
                assert (w & 0x7F, (w >> 7) & 31, imm) == (0b1101111, a, c)
            elif ty == "I":
                c = [-2048, 2047, -1, 0][j] if j < 4 else int(rng.integers(-2048, 2048))
                d = _decode(AC.encode_jalr(a, b, c))
                assert (d["opcode"], d["funct3"], d["rd"], d["rs1"], d["imm"]) == (0b1100111, 0, a, b, c)
            else:
                c = [0, (1 << 20) - 1, 1, 0x80000][j] if j < 4 else int(rng.integers(0, 1 << 20))
                w = getattr(AC, f"encode_{name.lower()}")(a, c)
                assert (w & 0x7F, (w >> 7) & 31, w >> 12) == (0b0110111 if name == "LUI" else 0b0010111, a, c)
            assert AC.encode(op, a, b if ty in ("B", "I") else 0, c) == w if ty != "I" else True


def _numpy_rv32i(ops, n_steps, base=AC.ELF_TEXT_START):
    """RV32I restated on numpy uint32 registers, decoding each instruction from its word: the final registers, the pc sequence and the
    execution count of every row."""
    words = np.array([AC.encode(*o) for o in ops], np.uint32)
    x = np.zeros(32, np.uint32)
    pcs, counts = [], np.zeros(len(ops), np.int64)
    pc = np.uint32(base)
    with np.errstate(over="ignore"):
        for _ in range(n_steps):
            row = (int(pc) - base) // 4
            w = int(words[row])
            pcs.append(int(pc))
            counts[row] += 1
            d = _decode(w)
            rd, rs1, rs2, f3 = d["rd"], d["rs1"], d["rs2"], d["funct3"]
            nxt, res = pc + np.uint32(4), None
            opc = w & 0x7F
            if opc == 0b1100011:
                imm = _sext(((w >> 31) << 12) | (((w >> 7) & 1) << 11) | (((w >> 25) & 0x3F) << 5) | (((w >> 8) & 0xF) << 1), 13)
                u1, u2 = x[rs1], x[rs2]
                s1, s2 = u1.astype(np.int32), u2.astype(np.int32)
                if {0: u1 == u2, 1: u1 != u2, 4: s1 < s2, 5: s1 >= s2, 6: u1 < u2, 7: u1 >= u2}[f3]:
                    nxt = pc + np.uint32(imm & 0xFFFFFFFF)
            elif opc == 0b1101111:
                imm = _sext(((w >> 31) << 20) | (((w >> 12) & 0xFF) << 12) | (((w >> 20) & 1) << 11) | (((w >> 21) & 0x3FF) << 1), 21)
                res, nxt = pc + np.uint32(4), pc + np.uint32(imm & 0xFFFFFFFF)
            elif opc == 0b1100111:
                res, nxt = pc + np.uint32(4), (x[rs1] + np.uint32(d["imm"] & 0xFFFFFFFF)) & np.uint32(0xFFFFFFFE)
            elif opc == 0b0110111:
                res = np.uint32(w & 0xFFFFF000)
            elif opc == 0b0010111:
                res = pc + np.uint32(w & 0xFFFFF000)
            else:
                b = x[rs1]
                cv = x[rs2] if opc == 0b0110011 else np.uint32(d["imm"] & 0xFFFFFFFF)
                sh = np.uint32(cv & np.uint32(31))
                alt = (w >> 30) & 1 if (opc == 0b0110011 or f3 == 0b101) else 0
                res = {(0, 0): b + cv, (0, 1): b - cv, (1, 0): b << sh, (2, 0): np.uint32(b.astype(np.int32) < cv.astype(np.int32)),
                       (3, 0): np.uint32(b < cv), (4, 0): b ^ cv, (5, 0): b >> sh, (5, 1): (b.astype(np.int32) >> sh.astype(np.int32)).astype(np.uint32),
                       (6, 0): b | cv, (7, 0): b & cv}[(f3, alt if opc == 0b0110011 or f3 in (1, 5) else 0)]
            if res is not None and rd:
                x[rd] = np.uint32(res)
            pc = np.uint32(nxt)
    return x, pcs, counts


@pytest.mark.parametrize("ls,n,seed", [(8, None, 0), (10, 5000, 1), (12, None, 2)])
def test_emulator_matches_a_numpy_restatement(ls, n, seed):
    words, ops, n_steps = AC.control_program(ls, n, seed)
    steps, (final, ts), final_ctr = AC.run(ops, n_steps)
    x, pcs, counts = _numpy_rv32i(ops, n_steps)
    assert np.array_equal(final, x) and np.array_equal(steps[F["pc"]], pcs) and np.array_equal(final_ctr, counts)
    assert np.array_equal(steps[F["word"]], words[(steps[F["pc"]] - AC.ELF_TEXT_START) // 4])
    assert set(int(o) for o in steps[F["opcode"]]) == set(range(29))
    assert final_ctr.max() > 1 and (final_ctr == 0).any()                       # rows that run many times and rows that never run
    # pc_ctr_prev counts the earlier runs of the row
    rows = (steps[F["pc"]] - AC.ELF_TEXT_START) // 4
    seen = np.zeros(len(ops), np.int64)
    for t, r in enumerate(rows):
        assert steps[F["pc_ctr_prev"], t] == seen[r]
        seen[r] += 1


def _run(ops, reg=None, n=None):
    _steps, (final, _ts), _ctr = AC.run(ops, len(ops) if n is None else n)
    return [int(v) for v in final] if reg is None else int(final[reg])


def test_known_answers():
    pc0 = AC.ELF_TEXT_START
    assert _run([(AC.OP_LUI, 1, 0, 0xFFFFF)], 1) == 0xFFFFF000
    assert _run([(AC.OP_LUI, 1, 0, 0)], 1) == 0
    assert _run([(AC.OP_ADDI, 0, 0, 0), (AC.OP_AUIPC, 1, 0, 0xFFFFF)], 1) == (pc0 + 4 - 4096) & 0xFFFFFFFF
    assert _run([(AC.OP_JAL, 1, 0, 8), (AC.OP_ADDI, 2, 0, 5), (AC.OP_ADDI, 3, 0, 7)], n=2) == [0, pc0 + 4, 0, 7] + [0] * 28
    # JALR to an odd target clears bit 0; rd == rs1 links after reading
    assert _run([(AC.OP_AUIPC, 5, 0, 0), (AC.OP_JALR, 5, 5, 13), (AC.OP_ADDI, 6, 0, 1), (AC.OP_ADDI, 7, 0, 2)], n=3) \
        == [0] * 5 + [pc0 + 8, 0, 2] + [0] * 24
    # BLT and BLTU disagree on 0x7FFFFFFF vs 0x80000000
    pre = [(AC.OP_ADDI, 1, 0, -1), (AC.OP_SRLI, 1, 1, 1), (AC.OP_ADDI, 2, 1, 1)]            # x1 = max, x2 = min
    for op, taken in ((AC.OP_BLT, False), (AC.OP_BLTU, True), (AC.OP_BGE, True), (AC.OP_BGEU, False)):
        got = _run(pre + [(op, 1, 2, 8), (AC.OP_ADDI, 3, 0, 1), (AC.OP_ADDI, 4, 0, 1)], n=5 if taken else 6)
        assert (got[3], got[4]) == ((0, 1) if taken else (1, 1)), AC.ALL_OPCODES[op][0]
    # a counted loop: x1 = 5 iterations of x2 += 3
    loop = [(AC.OP_ADDI, 1, 0, 5), (AC.OP_ADDI, 2, 2, 3), (AC.OP_ADDI, 1, 1, -1), (AC.OP_BNE, 1, 0, -8), (AC.OP_ADDI, 3, 0, 9)]
    steps, (final, _ts), ctr = AC.run(loop, 1 + 3 * 5 + 1)
    assert (int(final[2]), int(final[3])) == (15, 9) and list(ctr) == [1, 5, 5, 5, 1]


@pytest.mark.parametrize("seed", [0, 3])
def test_run_equals_execute_on_straight_line_programs(seed):
    _words, ops = AC.alu_program(10, 700, seed)
    s1, (v1, t1) = AC.execute(ops)
    s2, (v2, t2), ctr = AC.run(ops, len(ops))
    assert np.array_equal(s1, s2) and np.array_equal(v1, v2) and np.array_equal(t1, t2) and np.all(ctr == 1)


def test_run_refuses_a_pc_outside_the_program_or_misaligned():
    with pytest.raises(ValueError):
        AC.run([(AC.OP_ADDI, 1, 0, 1)], 2)                                       # falls off the end
    with pytest.raises(ValueError):
        AC.run([(AC.OP_JAL, 0, 0, -4)], 1 + 1)                                   # jumps before the program
    with pytest.raises(ValueError):
        AC.run([(AC.OP_BEQ, 0, 0, 6), (AC.OP_ADDI, 1, 0, 1), (AC.OP_ADDI, 1, 0, 1)], 2)   # a taken branch to pc + 6
    with pytest.raises(ValueError):                                              # JALR to base + 2 (bit 0 cleared, not bit 1)
        AC.run([(AC.OP_ADDI, 1, 0, AC.ELF_TEXT_START + 3), (AC.OP_JALR, 0, 1, 0), (AC.OP_ADDI, 1, 0, 1)], 3)
    assert AC.run([(AC.OP_BNE, 0, 1, 6), (AC.OP_ADDI, 1, 0, 1)], 2)[1][0][1] == 1        # not taken: the offset is never used


# ---- oracle proofs and the constraints

@pytest.fixture(scope="module", params=[(8, None), (9, 1500)], ids=["2^8", "1500-steps"])
def machine(request):
    m = AC.ControlMachine(*request.param)
    return m, m.fill_main_trace()


def test_oracle_proves_verifies_and_sums_cancel(machine):
    m, t1 = machine
    assert m.log_sizes == [m.log_size, 5, 8, 4, 4, 4, 5, 7, 8]
    assert m.final_ctr.max() > 1 and (m.final_ctr == 0).any()
    proof, claimed, aux = M.prove(m, OracleBackend(), t1, None, associated_data=b"control program")
    verify(m, proof, aux)
    assert len(claimed) == 9 and M.verify_claimed_sums(claimed)


def test_no_constraint_fails_on_the_executing_witness(machine):
    m, t1 = machine
    assert all(not v for v in _failures(m, t1).values())


def chip_ranges(log_size=9, **kw):
    """(ControlMachine, {decoding type or chip name: range of its constraints in the main component})."""
    seen = {}

    def wrap(name, record):
        def wrapped(comp, *a):
            first = len(comp.constraints)
            record(comp, *a)
            seen[name] = range(first, len(comp.constraints))
        return wrapped

    dec, chips = V.CONTROL_DECODING, V.CONTROL_CHIPS
    V.CONTROL_DECODING = [(n, wrap(n, r)) for n, r in dec]
    V.CONTROL_CHIPS = [(n, wrap(n, r)) for n, r in chips]
    try:
        m = AC.ControlMachine(log_size, **kw)
    finally:
        V.CONTROL_DECODING, V.CONTROL_CHIPS = dec, chips
    return m, seen


def test_chip_constraint_counts_and_degrees():
    """Each decoding type and chip adds its pinned number of constraints, 106 in all after the ALU program's 545; each has degree at most
    4, and the 30 of degree 3 or 4 (every one of BEQ's and BNE's, BLTU's and BGEU's next-pc pair, five of BLT's, three of BGE's; none of the
    decoding types' or of JAL, LUI, AUIPC and JALR's) go to the half-coset D2 kernel."""
    m, seen = chip_ranges()
    assert {k: len(v) for k, v in seen.items()} == CHIP_CONSTRAINTS
    deg = _walk_degrees(m.air.components[0])
    assert len(deg) == 545 + N_NEW == 651
    new = [deg[i] for r in seen.values() for i in r]
    assert max(new) == 4 and min(new) == 2
    assert sum(d > 2 for d in new) == 30
    by_chip = {k: sum(deg[i] > 2 for i in r) for k, r in seen.items()}
    assert by_chip == {"TypeBChip": 0, "TypeUChip": 0, "TypeJChip": 0, "BneChip": 9, "BeqChip": 9, "BltuChip": 2, "BltChip": 5,
                       "BgeuChip": 2, "BgeChip": 3, "JalChip": 0, "LuiChip": 0, "AuipcChip": 0, "JalrChip": 0}, by_chip
    # the order: decoding B, U, J right after types R / I, the chips between SltChip's and SllChip's
    lo = min(r.start for r in seen.values())
    assert [k for k, _r in sorted(seen.items(), key=lambda kv: kv[1].start)] == list(CHIP_CONSTRAINTS)
    assert seen["TypeJChip"].stop < seen["BneChip"].start and lo > 0


# CpuChip's next-row Pc constraints: PcNext's 16-bit halves equal the next row's Pc (cpu.rs:520-534)
NEXT_ROW_PC = (18, 19)


def broken_chain(log_size=9, n_steps=400):
    """(ControlMachine whose step record has one broken pc chain, the row it breaks at): step row + 1 claims another pc (with its own
    instruction word), so row's PcNext no longer equals the next row's Pc."""
    m = AC.ControlMachine(log_size, n_steps)
    row = 150
    s = m.steps.copy()
    s[F["pc"], row + 1] += 8
    m.steps, m._main = s, None
    return m, row


def test_a_broken_pc_chain_fails_only_the_next_row_pc_constraint():
    m, row = broken_chain()
    fails = _failures(m, m.fill_main_trace(), comps=[0])[0]
    assert {i for i, _n, _first in fails} == {NEXT_ROW_PC[0]} and all(first == row for _i, _n, first in fails), fails   # the low half


def _corruptions(m, t1):
    """Single-cell corruptions, one per row: every column the new decoding types and chips read, +1 on a row of each opcode."""
    ops = m.steps[F["opcode"]]
    words = [("ValueA", k) for k in range(4)] + [("ValueB", k) for k in range(4)] + [("ValueC", k) for k in range(4)]
    words += [("Pc", k) for k in range(4)] + [("PcNext", k) for k in range(4)] + [("InstrVal", k) for k in range(4)]
    words += [(n, k) for n in ("CarryFlag", "BorrowFlag") for k in range(2)] + [(n, k) for n in ("Helper1", "PcNextAux") for k in range(4)]
    words += [("Helper2", 3), ("Helper3", 3)]
    words += [(n, 0) for n in ("OpA", "OpB", "OpC", "OpA0", "OpA1_4", "OpB0_3", "OpB4", "OpC1_3", "OpC1_4", "OpC4_7", "OpC5_7", "OpC8_10",
                               "OpC11", "OpC12", "OpC12_15", "OpC16_19", "OpC16_23", "OpC20", "OpC24_31", "SgnA", "SgnB", "LtFlag", "Neq",
                               "Neq12", "Neq34", "Neq12Aux", "Neq34Aux", "Neq12AuxInv", "Neq34AuxInv", "RemAux", "QtAux")]
    bad = [c.copy() for c in t1]
    used = set()
    for op in range(AC.OP_BEQ, AC.N_OPCODES):
        rows = [r for r in range(1, m.n_steps - 1) if ops[r] == op and r not in used]
        assert len(rows) >= len(words), (AC.ALL_OPCODES[op][0], len(rows))
        for (name, limb), row in zip(words, rows):
            used.add(row)
            c = bad[OFFSETS[name] + limb]
            c[row] = (int(c[row]) + 1) % ((1 << 31) - 1)
    return bad


def test_every_new_constraint_is_broken_by_some_corruption():
    """On the edge-case prefix of control_program run 40 times over (then a JAL to itself), so that every new opcode has a row per
    corrupted column."""
    m, seen = chip_ranges(13, n_steps=1 << 13, ops=AC._control_prefix() * 40 + [(AC.OP_JAL, 0, 0, 0)])
    t1 = m.fill_main_trace()
    fails = {i for i, _a, _r in _failures(m, _corruptions(m, t1), comps=[0])[0]}
    missing = {k: [i for i in r if i not in fails] for k, r in seen.items()}
    assert not any(missing.values()), missing


def test_identically_zero_constraints_on_the_executing_trace():
    """Trees 0 and 1 of the executing control program make 96 of the 651 constraints identically zero (the ALU program: 121 of 545), 32
    of the 174 of degree > 2 among them.  Of the new ones only JalrChip's last two are: PcNextAux[2..3] = PcNext[2..3], whose bytes are zero
    while every pc stays below 2^16.  No other constraint of the ten chips or of DecodingCheck B / U / J is."""
    from tests import random_witness as rw
    from tests.test_v1_random_witness_cpu import committed, high_flags
    m, seen = chip_ranges(8)
    high = high_flags(m)
    _p, _params, trees = committed(m, "padding")
    z = np.array(rw.identically_zero(m.words, 0, trees[:2]))
    assert (len(z), int(z.sum()), int((z & high).sum()), int(high.sum())) == (651, 96, 32, 174)
    zero_new = {k: [i - r.start for i in r if z[i]] for k, r in seen.items() if any(z[i] for i in r)}
    assert zero_new == {"JalrChip": [7, 8]}, zero_new


# ---- the device fill's row code

@pytest.mark.parametrize("ls,n,seed", [(8, None, 0), (10, 3000, 1), (12, None, 2)])
def test_host_fill_equals_the_numpy_columns(host_fill, ls, n, seed):  # noqa: F811
    m = AC.ControlMachine(ls, n, seed=seed)
    want = np.stack(m.fill_main_trace()[:347])[:, finalized_src_rows(m.log_size)]
    bad = np.argwhere(host_fill(m.steps, m.final_ctr, m.log_size) != want)
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"


def control_edge_steps(log_size, n_steps, seed):
    """A step record of n_steps steps over all 29 opcodes that nb200_v1_control_trace's host check accepts (valid_control_steps), its
    operands and pcs from the edges of u32 (edgy_u32) rather than from an execution: branch offsets -4096 and 4094, JAL offsets -2^20 and
    2^20 - 2, U immediates 0 and 0xFFFFF, operands equal in one 16-bit half only, pc_ctr_prev 0xFFFF and 0xFFFFFFFE among them."""
    rng = np.random.default_rng(seed)
    s = np.zeros((len(AC.STEP_FIELDS), n_steps), np.uint64)
    op = rng.integers(0, 29, n_steps)
    op[:29] = np.arange(29)
    op[29:29 + 40] = rng.choice([AC.OP_BEQ, AC.OP_BNE], 40)
    ty = np.array(AC.ALL_OP_TYPE)[op]
    s[F["opcode"]] = op
    for f in ("pc", "word", "value_b", "rd_prev"):
        s[F[f]] = edgy_u32(rng, n_steps)
    half = rng.integers(0, 3, n_steps)                                            # op_a and op_b equal in a half, or equal
    eq_rows = np.isin(op, [AC.OP_BEQ, AC.OP_BNE]) & (rng.integers(0, 2, n_steps) == 0)
    va, vb = s[F["rd_prev"]], s[F["value_b"]]
    s[F["value_b"]] = np.where(eq_rows, np.select([half == 0, half == 1], [(vb & 0xFFFF0000) | (va & 0xFFFF), (vb & 0xFFFF) | (va & 0xFFFF0000)], va), vb)
    s[F["pc"]][29:29 + 40:2] &= np.uint64(0xFFFF00FF)                            # pc halves that read 0 big-endian: the fallback 1
    s[F["pc"]][30:29 + 40:2] &= np.uint64(0x00FFFF00)
    s[F["rd"]], s[F["rs1"]] = rng.integers(0, 32, n_steps), rng.integers(0, 32, n_steps)
    imm = np.where(rng.integers(0, 3, n_steps) == 0, rng.choice([-2048, 2047, -1, 0], n_steps), rng.integers(-2048, 2048, n_steps))
    boff = np.where(rng.integers(0, 3, n_steps) == 0, rng.choice([-4096, 4094, -2, 0], n_steps), 2 * rng.integers(-2048, 2048, n_steps))
    joff = np.where(rng.integers(0, 3, n_steps) == 0, rng.choice([-(1 << 20), (1 << 20) - 2, 0], n_steps), 2 * rng.integers(-(1 << 19), 1 << 19, n_steps))
    uimm = np.where(rng.integers(0, 3, n_steps) == 0, rng.choice([0, 0xFFFFF, 0x80000], n_steps), rng.integers(0, 1 << 20, n_steps))
    shamt = np.where(rng.integers(0, 3, n_steps) == 0, rng.choice([0, 31], n_steps), rng.integers(0, 32, n_steps))
    m32 = 0xFFFFFFFF
    s[F["op_c"]] = np.select([ty == "R", ty == "I", ty == "IShift", ty == "B", ty == "J"],
                             [rng.integers(0, 32, n_steps), imm.astype(np.int64) & m32, shamt, boff.astype(np.int64) & m32, joff.astype(np.int64) & m32],
                             uimm)
    s[F["value_c"]] = np.select([ty == "R", ty == "U"], [edgy_u32(rng, n_steps), (s[F["op_c"]] << np.uint64(12)) & m32], s[F["op_c"]])
    no_b = np.isin(ty, ["J", "U"])
    s[F["rs1"]] = np.where(no_b, 0, s[F["rs1"]])
    s[F["value_b"]] = np.where(no_b, 0, s[F["value_b"]])
    clk = np.arange(1, n_steps + 1, dtype=np.uint64)
    for k in (1, 2, 3):
        s[F[f"ts{k}_prev"]] = (rng.random(n_steps) * (3 * clk + k)).astype(np.uint64)
    s[F["pc_ctr_prev"]] = np.minimum(edgy_u32(rng, n_steps), 0xFFFFFFFE)
    s[F["pc_ctr_prev"]][:4] = [0xFFFF, 0xFFFFFFFE, 0xFFFF, 0x1FFFF]
    steps = s.astype(np.uint32)
    final_ctr = rng.integers(0, 1 << 32, min(n_steps, 1 << log_size), dtype=np.uint64).astype(np.uint32)
    assert valid_control_steps(steps, final_ctr, log_size)
    return steps, final_ctr


def valid_control_steps(steps, final_ctr, log_size):
    """nb200_v1_control_trace's host check (csrc/v1_trace.cu), restated."""
    n_steps = steps.shape[1]
    s = {f: steps[i].astype(np.uint64) for i, f in enumerate(AC.STEP_FIELDS)}
    if not (n_steps <= 1 << log_size and final_ctr.size <= 1 << log_size and np.all(s["opcode"] < 29)):
        return False
    ty = np.array(AC.ALL_OP_TYPE)[s["opcode"].astype(np.int64)]
    imm = steps[F["op_c"]].view(np.int32).astype(np.int64)
    oc = s["op_c"]
    clk = np.arange(1, n_steps + 1, dtype=np.uint64)
    return bool(np.all(s["rd"] < 32) and np.all(s["rs1"] < 32) and np.all((ty != "R") | (oc < 32)) and np.all((ty != "IShift") | (oc < 32))
                and np.all((ty != "I") | ((imm >= -2048) & (imm < 2048)))
                and np.all((ty != "B") | ((imm >= -4096) & (imm < 4096) & (imm % 2 == 0)))
                and np.all((ty != "J") | ((imm >= -(1 << 20)) & (imm < 1 << 20) & (imm % 2 == 0)))
                and np.all((ty != "U") | (oc < 1 << 20)) and np.all(s["pc_ctr_prev"] != 0xFFFFFFFF)
                and all(np.all(s[f"ts{k}_prev"] < 3 * clk + k) for k in (1, 2, 3)))


@pytest.mark.parametrize("ls,n_steps", [(8, 256), (10, 900), (12, 4096)])
def test_host_fill_on_edge_step_records(host_fill, ls, n_steps):  # noqa: F811
    steps, final_ctr = control_edge_steps(ls, n_steps, seed=ls)
    want = _want(steps, final_ctr, ls)
    bad = np.argwhere(host_fill(steps, final_ctr, ls) != want)
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"
    for name in ("Neq", "Neq12", "Neq34", "SgnA", "LtFlag", "RemAux", "QtAux", "OpC12", "OpC20", "OpB4", "OpC24_31", "PcNextAux"):
        assert want[OFFSETS[name]].any(), name
    # the big-endian fallback of BEQ / BNE's aux pair: some equal half whose pc half reads 0 takes 1, others take the pc half
    eq = np.isin(steps[F["opcode"]], [AC.OP_BEQ, AC.OP_BNE])
    t = AC.main_columns(steps, final_ctr, ls)
    lo_eq = eq & ((steps[F["rd_prev"]] & 0xFFFF) == (steps[F["value_b"]] & 0xFFFF))
    inv = t["Neq12AuxInv"][0][:n_steps][lo_eq]
    pc = steps[F["pc"]][lo_eq].astype(np.int64)
    be = ((pc & 0xFF) << 8) | ((pc >> 8) & 0xFF)
    assert np.array_equal(inv, np.maximum(be, 1)) and (be == 0).any() and (be != (pc & 0xFFFF)).any()
    assert (t["ProgCtrCarry"][0][:n_steps] == 1).any()


# ---- sm_90a builds

def test_fill_kernel_compiles_for_sm90a_without_spills(tmp_path):
    """One entry function, the fill kernel the three entries share; its register count is printed (pytest -s)."""
    import re
    blocks = _ptxas_blocks(os.path.join(CSRC, "v1_trace.cu"), tmp_path / "v1_trace.o")
    (name,) = [n for n in blocks if "v1_main_trace_kernel" in n]
    assert _spills(blocks[name]) == 0, blocks[name]
    print("v1_main_trace_kernel on sm_90a:", re.search(r"Used (\d+) registers", blocks[name]).group(0))


def test_generated_kernels_compile_for_sm90a(tmp_path):
    """The kernels generated for ControlMachine's main component: constraints (D1), LogUp, D2, check and table count build for sm_90a.
    Their spill bytes are printed (pytest -s) beside the ALU program's."""
    import nexus_zkvm_b200 as nb
    from tests import test_constraint_check_cpu as chk
    from tests.test_d2_high_degree_cpu import _load, _source
    from tests.test_table_multiplicities_cpu import count_source
    report = {}
    for label, m in (("alu", AC.AluMachine(8)), ("control", AC.ControlMachine(8))):
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
