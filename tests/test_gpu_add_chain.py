"""The reference's ADD-chain benchmark as an executing v1 trace on the GPU (add_chain.py; run on an H100: `pytest -m gpu`): the main trace
filled on the device from the step record (nb200_v1_main_trace) equals the numpy columns over a batch pre-filled with garbage, full and
padded; the device-counted multiplicities equal the host counts; proofs from host columns and from device trees are byte-identical and equal
the oracle's; the GPU constraint check passes the executing witness and names the constraint a corrupted row breaks; bad step records are
refused with the context left usable; and a 2^20-step proof from device trees is accepted with sums that cancel."""
import gc

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import add_chain as AC
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.prover import CudaBackend
from tests.keccak_side_notes import finalized_src_rows
from tests.oracle_backend import OracleBackend, verify, verify_with_replayed_transcript
from tests.test_add_chain_cpu import OFFSETS, mixed_program

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def backend():
    b = CudaBackend(nb.Context(0))
    yield b
    gc.collect()
    b.ctx.close()


def _garbage(ctx, log_size, seed=3):
    return ctx.upload(np.random.default_rng(seed).integers(0, 1 << 32, (347, 1 << log_size), dtype=np.uint64).astype(np.uint32))


@pytest.mark.parametrize("ls,n", [(8, None), (8, 100), (12, None), (12, 3001), (16, None), (16, 40000), (9, "mixed")])
def test_device_fill_equals_numpy(backend, ls, n):
    m = AC.AddChainMachine(ls, ops=mixed_program()) if n == "mixed" else AC.AddChainMachine(ls, n)
    out = _garbage(backend.ctx, ls)
    got = backend.ctx.v1_main_trace(m.steps, m.final_ctr, ls, out=out)
    assert got is out
    want = np.stack(m.fill_main_trace()[:347])[:, finalized_src_rows(ls)]
    bad = np.argwhere(out.download() != want)
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"


@pytest.mark.parametrize("ls,n", [(10, None), (10, 700)])
def test_device_counts_equal_host_counts(backend, ls, n):
    m = AC.AddChainMachine(ls, n)
    _tree0, tree1 = m.device_trees(backend.ctx)
    host = m.fill_main_trace()[347:]
    dev = [c for b in tree1[1:] for c in b.download()]
    assert len(dev) == len(host)
    for k, (d, h) in enumerate(zip(dev, host)):
        log = int(len(h)).bit_length() - 1
        assert np.array_equal(d, np.asarray(h, np.uint32)[finalized_src_rows(log)]), k


@pytest.mark.parametrize("ls,n", [(10, None), (10, 700), (12, None)])
def test_proofs_equal_the_oracle_and_each_other(backend, ls, n):
    m = AC.AddChainMachine(ls, n)
    t1 = m.fill_main_trace()
    h_proof, h_claimed, h_aux = M.prove(m, backend, t1, None, associated_data=b"add chain")
    d_proof, d_claimed, d_aux = M.prove(m, backend, None, None, associated_data=b"add chain", resident=m.device_trees(backend.ctx))
    o_proof, o_claimed, o_aux = M.prove(m, OracleBackend(), t1, None, associated_data=b"add chain")
    assert h_aux["roots"] == d_aux["roots"] == o_aux["roots"]
    assert h_claimed == d_claimed == o_claimed
    assert h_proof == d_proof == o_proof
    assert M.verify_claimed_sums(h_claimed)
    verify(m, h_proof, o_aux)


def test_check_constraints_passes_and_names_a_corrupted_constraint(backend):
    m = AC.AddChainMachine(10, 700)
    t1 = m.fill_main_trace()
    report, sums_ok = M.check_constraints(m, backend, t1, None)
    assert sums_ok and all(not v for v in report.values())
    # CarryFlag's low limb raised on trace row 5: AddChip's two carry constraints and CarryFlag's booleanity fail there
    bad = list(t1)
    c = bad[OFFSETS["CarryFlag"]].copy()
    c[5] += 2
    bad[OFFSETS["CarryFlag"]] = c
    report, _ = M.check_constraints(m, backend, bad, None)
    failing = report[0]
    assert failing and all(first == 5 for _k, _deg, _n, first in failing)
    add_lo = _constraint_index(m, "add_lo")
    assert add_lo in [k for k, _deg, _n, _first in failing]


def _constraint_index(m, which):
    """Index of AddChip's low 16-bit constraint in the main component: recorded right after CpuChip's and DecodingCheck's."""
    from nexus_zkvm_b200 import air as A
    from nexus_zkvm_b200 import nexus_v1 as V
    air = A.Air()
    rel = {r.name: r for r in [air.relation(nm, s) for nm, s in [("BitOp", 4), ("LoadStore", 5), ("ProgramCheck", 8), ("RegisterCheck", 9),
                                                               ("Range8", 1), ("Range16", 1), ("Range32", 1), ("Range128", 1), ("Range256", 1)]]}
    seen = []
    orig = V._record_decoding_r_i

    def wrapped(comp, *a):
        orig(comp, *a)
        seen.append(len(comp.constraints))
    V._record_decoding_r_i = wrapped
    try:
        V.record_main_component(air, m.log_size, rel, decoding=True)
    finally:
        V._record_decoding_r_i = orig
    assert which == "add_lo"
    return seen[0]


def test_bad_step_records_are_refused_and_the_context_stays_usable(backend):
    ctx = backend.ctx
    m = AC.AddChainMachine(8, 200)
    out = ctx.alloc(347, 8)
    f = {n: i for i, n in enumerate(AC.STEP_FIELDS)}

    def refused(steps, ctr=m.final_ctr, log=8, batch=out):
        with pytest.raises(nb.Nb200Error, match="status 2"):
            ctx.v1_main_trace(steps, ctr, log, out=batch)

    for field, value in (("opcode", 2), ("rd", 32), ("rs1", 40), ("op_c", 32), ("ts1_prev", 3 * 10 + 1), ("pc_ctr_prev", 0xFFFFFFFF)):
        s = m.steps.copy()
        s[f[field], 9] = value
        refused(s)
    refused(AC.AddChainMachine(9).steps)                                         # more steps than rows
    refused(m.steps, ctr=np.ones(257, np.uint32))                                # more program rows than rows
    refused(m.steps, batch=ctx.alloc(347, 9))                                     # a batch of another shape
    refused(m.steps, log=3, batch=ctx.alloc(347, 3))                              # log_size below 4
    ctx.v1_main_trace(m.steps, m.final_ctr, 8, out=out)
    assert np.array_equal(out.download(), np.stack(m.fill_main_trace()[:347])[:, finalized_src_rows(8)])


def test_largest_reference_size_proof_is_accepted(backend):
    """2^20 steps of the ADD chain (the reference bench's largest size), every tree built on the device."""
    m = AC.AddChainMachine(20)
    proof, claimed, aux = M.prove(m, backend, None, None, resident=m.device_trees(backend.ctx))
    assert M.verify_claimed_sums(claimed)
    verify_with_replayed_transcript(m, proof, claimed, aux)
