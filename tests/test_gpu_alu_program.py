"""A program of RV32I's ALU instructions as an executing v1 trace on the GPU (add_chain.AluMachine; run on an H100: `pytest -m gpu`): the
main trace filled on the device from the step record (nb200_v1_alu_trace) equals the numpy columns over a batch pre-filled with garbage,
full and padded, on programs and on edge step records of all 19 opcodes; bad step records are refused with the context left usable; proofs
from device trees equal the host-column proof and the oracle's; the GPU constraint check passes the executing witness and names the
corrupted constraint and row of each new chip; and a 2^20-step proof from device trees is accepted."""
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
from tests.test_alu_program_cpu import _want, alu_edge_steps, chip_ranges

pytestmark = pytest.mark.gpu


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
    m = AC.AluMachine(ls, n, seed=ls)
    out = _garbage(backend.ctx, ls)
    assert backend.ctx.v1_alu_trace(m.steps, m.final_ctr, ls, out=out) is out
    want = np.stack(m.fill_main_trace()[:347])[:, finalized_src_rows(ls)]
    bad = np.argwhere(out.download() != want)
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"


@pytest.mark.parametrize("ls,n_steps", [(8, 256), (12, 4000)])
def test_device_fill_on_edge_step_records(backend, ls, n_steps):
    steps, final_ctr = alu_edge_steps(ls, n_steps, seed=ls + 100)
    out = backend.ctx.v1_alu_trace(steps, final_ctr, ls, out=_garbage(backend.ctx, ls))
    bad = np.argwhere(out.download() != _want(steps, final_ctr, ls))
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"


def test_bad_step_records_are_refused_and_the_context_stays_usable(backend):
    ctx = backend.ctx
    m = AC.AluMachine(8, 200)
    out = ctx.alloc(347, 8)
    f = {n: i for i, n in enumerate(AC.STEP_FIELDS)}
    ops = m.steps[f["opcode"]]
    r_row, i_row, shift_row = (int(np.nonzero(np.isin(ops, which))[0][0])
                               for which in ([AC.OP_SUB], [AC.OP_XORI], [AC.OP_SRAI]))

    def refused(steps, ctr=m.final_ctr, log=8, batch=out):
        with pytest.raises(nb.Nb200Error, match="status 2"):
            ctx.v1_alu_trace(steps, ctr, log, out=batch)

    for field, row, value in (("opcode", 9, 19), ("opcode", 9, 0xFFFFFFFF), ("rd", 9, 32), ("rs1", 9, 40), ("op_c", r_row, 32),
                              ("op_c", shift_row, 32), ("op_c", i_row, 2048), ("op_c", i_row, 0xFFFFF7FF), ("ts1_prev", 9, 3 * 10 + 1),
                              ("pc_ctr_prev", 9, 0xFFFFFFFF)):
        s = m.steps.copy()
        s[f[field], row] = value
        refused(s)
    refused(AC.AluMachine(9).steps)                                              # more steps than rows
    refused(m.steps, ctr=np.ones(257, np.uint32))                                # more program rows than rows
    refused(m.steps, batch=ctx.alloc(347, 9))                                     # a batch of another shape
    # nb200_v1_main_trace keeps ADD / ADDI only
    with pytest.raises(nb.Nb200Error, match="status 2"):
        ctx.v1_main_trace(m.steps, m.final_ctr, 8, out=out)
    ctx.v1_alu_trace(m.steps, m.final_ctr, 8, out=out)
    assert np.array_equal(out.download(), np.stack(m.fill_main_trace()[:347])[:, finalized_src_rows(8)])


def test_proofs_equal_the_oracle_and_each_other(backend):
    m = AC.AluMachine(10, 900, seed=4)
    t1 = m.fill_main_trace()
    h_proof, h_claimed, h_aux = M.prove(m, backend, t1, None, associated_data=b"alu program")
    d_proof, d_claimed, d_aux = M.prove(m, backend, None, None, associated_data=b"alu program", resident=m.device_trees(backend.ctx))
    o_proof, o_claimed, o_aux = M.prove(m, OracleBackend(), t1, None, associated_data=b"alu program")
    assert h_aux["roots"] == d_aux["roots"] == o_aux["roots"]
    assert h_claimed == d_claimed == o_claimed
    assert h_proof == d_proof == o_proof
    assert M.verify_claimed_sums(h_claimed)
    verify(m, h_proof, o_aux)


def test_check_constraints_names_each_chips_corrupted_constraint(backend):
    m, seen = chip_ranges(10, n_steps=700)
    t1 = m.fill_main_trace()
    report, sums_ok = M.check_constraints(m, backend, t1, None)
    assert sums_ok and all(not v for v in report.values())
    ops = m.steps[AC.STEP_FIELDS.index("opcode")]
    # one corrupted cell per chip, each on a row of its own opcode: the chip's first constraint reads it
    for chip, op, (name, limb) in (("SltuChip", AC.OP_SLTU, ("ValueA", 1)), ("SltChip", AC.OP_SLT, ("Helper1", 0)),
                                   ("SllChip", AC.OP_SLLI, ("ShiftBit1", 0)), ("SrlChip", AC.OP_SRL, ("ShiftBit2", 0)),
                                   ("SraChip", AC.OP_SRAI, ("Helper1", 0))):
        row = int(np.nonzero(ops == op)[0][-1])
        bad = list(t1)
        c = bad[OFFSETS[name] + limb].copy()
        c[row] += 1
        bad[OFFSETS[name] + limb] = c
        report, _ = M.check_constraints(m, backend, bad, None)
        failing = {k: first for k, _deg, _n, first in report[0]}
        mine = [k for k in seen[chip] if k in failing]
        assert mine and all(failing[k] == row for k in mine), (chip, report[0])


def test_largest_size_proof_is_accepted(backend):
    """2^20 steps of an ALU program, every tree built on the device."""
    m = AC.AluMachine(20)
    proof, claimed, aux = M.prove(m, backend, None, None, resident=m.device_trees(backend.ctx))
    assert M.verify_claimed_sums(claimed)
    verify_with_replayed_transcript(m, proof, claimed, aux)
