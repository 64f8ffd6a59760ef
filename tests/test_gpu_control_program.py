"""Looping RV32I programs with branches, JAL, JALR, LUI and AUIPC as executing v1 traces on the GPU (add_chain.ControlMachine; run on an
H100: `pytest -m gpu`): the main trace filled on the device from the step record (nb200_v1_control_trace) equals the numpy columns over a
batch pre-filled with garbage, full and padded, on programs and on edge step records of all 29 opcodes; bad step records are refused with
the context left usable, and the older entries still refuse the new opcodes; proofs from device trees equal the host-column proof and the
oracle's; the GPU constraint check names the corrupted constraint and row of each new chip and a broken pc chain; a two-instruction loop
whose execution counters carry past 2^16 is checked and proven; and a 2^20-step proof from device trees is accepted."""
import gc

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import add_chain as AC
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.prover import CudaBackend
from tests.keccak_side_notes import finalized_src_rows
from tests.oracle_backend import OracleBackend, verify, verify_with_replayed_transcript
from tests.test_add_chain_cpu import OFFSETS
from tests.test_alu_program_cpu import _want
from tests.test_control_program_cpu import NEXT_ROW_PC, broken_chain, chip_ranges, control_edge_steps

pytestmark = pytest.mark.gpu
F = {n: i for i, n in enumerate(AC.STEP_FIELDS)}


@pytest.fixture(scope="module")
def backend():
    b = CudaBackend(nb.Context(0))
    yield b
    gc.collect()
    b.ctx.close()


def _garbage(ctx, log_size, seed=3):
    return ctx.upload(np.random.default_rng(seed).integers(0, 1 << 32, (347, 1 << log_size), dtype=np.uint64).astype(np.uint32))


@pytest.mark.parametrize("ls,n", [(8, None), (8, 100), (10, None), (12, None), (12, 3001), (16, None), (16, 40000)])
def test_device_fill_equals_numpy(backend, ls, n):
    m = AC.ControlMachine(ls, n, seed=ls)
    assert m.log_size == ls
    out = _garbage(backend.ctx, ls)
    assert backend.ctx.v1_control_trace(m.steps, m.final_ctr, ls, out=out) is out
    want = np.stack(m.fill_main_trace()[:347])[:, finalized_src_rows(ls)]
    bad = np.argwhere(out.download() != want)
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"


@pytest.mark.parametrize("ls,n_steps", [(8, 256), (12, 4000), (16, 40000)])
def test_device_fill_on_edge_step_records(backend, ls, n_steps):
    steps, final_ctr = control_edge_steps(ls, n_steps, seed=ls + 100)
    out = backend.ctx.v1_control_trace(steps, final_ctr, ls, out=_garbage(backend.ctx, ls))
    bad = np.argwhere(out.download() != _want(steps, final_ctr, ls))
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"


def test_bad_step_records_are_refused_and_the_context_stays_usable(backend):
    ctx = backend.ctx
    m = AC.ControlMachine(8, 250)
    out = ctx.alloc(347, 8)
    ops = m.steps[F["opcode"]]
    row = {op: int(np.nonzero(ops == op)[0][0]) for op in (AC.OP_SUB, AC.OP_SRAI, AC.OP_XORI, AC.OP_JALR, AC.OP_BGE, AC.OP_JAL, AC.OP_LUI)}

    def refused(steps, ctr=m.final_ctr, log=8, batch=out, entry=ctx.v1_control_trace):
        with pytest.raises(nb.Nb200Error, match="status 2"):
            entry(steps, ctr, log, out=batch)

    for field, op, value in (("opcode", AC.OP_SUB, 29), ("opcode", AC.OP_SUB, 0xFFFFFFFF), ("rd", AC.OP_SUB, 32), ("rs1", AC.OP_BGE, 40),
                             ("op_c", AC.OP_SUB, 32), ("op_c", AC.OP_SRAI, 32), ("op_c", AC.OP_XORI, 2048), ("op_c", AC.OP_JALR, 0xFFFFF7FF),
                             ("op_c", AC.OP_BGE, 4096), ("op_c", AC.OP_BGE, 3), ("op_c", AC.OP_BGE, 0xFFFFEFFE), ("op_c", AC.OP_JAL, 1 << 20),
                             ("op_c", AC.OP_JAL, 5), ("op_c", AC.OP_LUI, 1 << 20), ("ts3_prev", AC.OP_SUB, None),
                             ("pc_ctr_prev", AC.OP_SUB, 0xFFFFFFFF)):
        s = m.steps.copy()
        s[F[field], row[op]] = 3 * (row[op] + 1) + 3 if value is None else value                 # a timestamp not below the current one
        refused(s)
    refused(AC.ControlMachine(9).steps)                                          # more steps than rows
    refused(m.steps, ctr=np.ones(257, np.uint32))                                # more program rows than rows
    refused(m.steps, batch=ctx.alloc(347, 9))                                     # a batch of another shape
    # nb200_v1_alu_trace keeps refusing opcodes 19-28, nb200_v1_main_trace everything but ADD / ADDI
    for op in range(AC.OP_BEQ, AC.N_OPCODES):
        s = m.steps.copy()
        s[F["opcode"], :] = AC.OP_ADD
        s[F["op_c"], :] = 0
        s[F["opcode"], 7] = op
        refused(s, entry=ctx.v1_alu_trace)
        refused(s, entry=ctx.v1_main_trace)
    ctx.v1_control_trace(m.steps, m.final_ctr, 8, out=out)
    assert np.array_equal(out.download(), np.stack(m.fill_main_trace()[:347])[:, finalized_src_rows(8)])


def test_proofs_equal_the_oracle_and_each_other(backend):
    m = AC.ControlMachine(10, 900, seed=4)
    t1 = m.fill_main_trace()
    h_proof, h_claimed, h_aux = M.prove(m, backend, t1, None, associated_data=b"control program")
    d_proof, d_claimed, d_aux = M.prove(m, backend, None, None, associated_data=b"control program", resident=m.device_trees(backend.ctx))
    o_proof, o_claimed, o_aux = M.prove(m, OracleBackend(), t1, None, associated_data=b"control program")
    assert h_aux["roots"] == d_aux["roots"] == o_aux["roots"]
    assert h_claimed == d_claimed == o_claimed
    assert h_proof == d_proof == o_proof
    assert M.verify_claimed_sums(h_claimed)
    verify(m, h_proof, o_aux)


def test_check_constraints_names_each_chips_corrupted_constraint(backend):
    m, seen = chip_ranges(10, n_steps=3000)
    t1 = m.fill_main_trace()
    report, sums_ok = M.check_constraints(m, backend, t1, None)
    assert sums_ok and all(not v for v in report.values())
    ops = m.steps[F["opcode"]]
    # one corrupted cell per chip, each on a row of its own opcode: the chip's first constraint reads it
    for chip, op, (name, limb) in (("TypeBChip", AC.OP_BLTU, ("OpC1_4", 0)), ("TypeUChip", AC.OP_AUIPC, ("OpC12_15", 0)),
                                   ("TypeJChip", AC.OP_JAL, ("OpC1_3", 0)), ("BneChip", AC.OP_BNE, ("Neq12Aux", 0)),
                                   ("BeqChip", AC.OP_BEQ, ("Neq34Aux", 0)), ("BltuChip", AC.OP_BLTU, ("Helper1", 0)),
                                   ("BltChip", AC.OP_BLT, ("Helper1", 1)), ("BgeuChip", AC.OP_BGEU, ("Helper1", 2)),
                                   ("BgeChip", AC.OP_BGE, ("Helper1", 3)), ("JalChip", AC.OP_JAL, ("ValueA", 0)),
                                   ("LuiChip", AC.OP_LUI, ("ValueA", 0)), ("AuipcChip", AC.OP_AUIPC, ("ValueA", 1)),
                                   ("JalrChip", AC.OP_JALR, ("ValueA", 0))):
        row = int(np.nonzero(ops == op)[0][-1])
        bad = list(t1)
        c = bad[OFFSETS[name] + limb].copy()
        c[row] += 1
        bad[OFFSETS[name] + limb] = c
        report, _ = M.check_constraints(m, backend, bad, None)
        failing = {k: first for k, _deg, _n, first in report[0]}
        mine = [k for k in seen[chip] if k in failing]
        assert mine and all(failing[k] == row for k in mine), (chip, report[0])


def test_check_constraints_reports_a_broken_pc_chain(backend):
    m, row = broken_chain()
    report, _ = M.check_constraints(m, backend, m.fill_main_trace(), None)
    failing = {k: first for k, _deg, _n, first in report[0]}
    assert failing and set(failing) <= set(NEXT_ROW_PC) and all(first == row for first in failing.values()), report[0]


def test_two_instruction_loop_carries_the_execution_counters(backend):
    """2^17 steps of a two-instruction loop: each row runs 2^16 times, so ProgCtrCarry is set on the rows whose previous count is 0xFFFF."""
    m = AC.ControlMachine(17, ops=[(AC.OP_ADDI, 1, 1, 1), (AC.OP_JAL, 0, 0, -4)])
    assert m.log_size == 17 and list(m.final_ctr) == [1 << 16, 1 << 16]
    t1 = m.fill_main_trace()
    assert t1[OFFSETS["ProgCtrCarry"]].any()
    report, sums_ok = M.check_constraints(m, backend, t1, None)
    assert sums_ok and all(not v for v in report.values())
    proof, claimed, aux = M.prove(m, backend, None, None, resident=m.device_trees(backend.ctx))
    assert M.verify_claimed_sums(claimed)
    verify_with_replayed_transcript(m, proof, claimed, aux)


def test_largest_size_proof_is_accepted(backend):
    """2^20 steps of a control program, every tree built on the device."""
    m = AC.ControlMachine(20)
    assert m.log_size == 20
    proof, claimed, aux = M.prove(m, backend, None, None, resident=m.device_trees(backend.ctx))
    assert M.verify_claimed_sums(claimed)
    verify_with_replayed_transcript(m, proof, claimed, aux)
