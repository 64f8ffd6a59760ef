"""The v1 main component, its eight base extensions and the keccak extension proven as one machine on the GPU (whole_machine.py; run on an
H100: `pytest -m gpu`): proof bytes, claimed sums and roots equal the oracle's, the oracle's verifier accepts, RamInitFinal's device fill
(nb200_ram_init_final_trace) equals the numpy columns over a batch pre-filled with garbage, the proof from device-filled trees equals the
host-column proof, the generic table count refuses the machine (Multiplicity8's repeated zero), each bad argument is refused with the
context left usable, and a proof at 2^20 main rows with 2^12 permutations is accepted.

The machines are built once per module: each size's generated kernels (the keccak round components' take minutes of NVRTC on first use)
compile once per run."""
import gc

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200 import whole_machine as W
from nexus_zkvm_b200.prover import CudaBackend
from tests.keccak_side_notes import finalized_src_rows
from tests.oracle_backend import OracleBackend, verify, verify_with_replayed_transcript
from tests.test_whole_machine_cpu import edge_side_notes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def backend():
    b = CudaBackend(nb.Context(0))
    yield b
    gc.collect()
    b.ctx.close()


@pytest.fixture(scope="module")
def machines():
    return {"small": W.NexusV1KeccakMachine(8, 15, seed=1), "mid": W.NexusV1KeccakMachine(16, 1 << 6, seed=2)}


@pytest.mark.parametrize("size", ["small", "mid"])
def test_proof_equals_the_oracle_and_is_accepted(backend, machines, size):
    m = machines[size]
    t1 = m.fill_main_trace()
    g_proof, g_claimed, g_aux = M.prove(m, backend, t1, None, associated_data=b"whole")
    o_proof, o_claimed, o_aux = M.prove(m, OracleBackend(), t1, None, associated_data=b"whole")
    assert g_aux["roots"] == o_aux["roots"]
    assert g_claimed == o_claimed
    assert g_proof == o_proof
    assert M.verify_claimed_sums(g_claimed)
    verify(m, g_proof, o_aux)


def _garbage_batch(ctx, log_size, seed):
    return ctx.upload(np.random.default_rng(seed).integers(0, 1 << 32, (W.RAM_COLS, 1 << log_size), dtype=np.uint64).astype(np.uint32))


@pytest.mark.parametrize("case", edge_side_notes(), ids=lambda c: c[0])
def test_ram_init_final_fill_equals_numpy(backend, case):
    _name, side_note, (ia, iv) = case
    addr, _v, _c = W.last_access(*side_note, ia, iv)
    log_size = W.ram_log_size(addr.size)
    out = _garbage_batch(backend.ctx, log_size, 3)
    got, n_rows = backend.ctx.ram_init_final_trace(*side_note, ia, iv, log_size, out=out)
    assert got is out and n_rows == addr.size
    want = W.ram_init_final_columns(*side_note, ia, iv, log_size)[:, finalized_src_rows(log_size)]
    bad = np.argwhere(out.download() != want)
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"


@pytest.mark.parametrize("size", ["small", "mid"])
def test_machine_fill_and_device_tree_proof(backend, machines, size):
    m = machines[size]
    out = _garbage_batch(backend.ctx, m.ram_log_size, 4)
    backend.ctx.ram_init_final_trace(*m.side_note(), *m.initial_memory(), m.ram_log_size, out=out)
    assert np.array_equal(out.download(), m.ram_init_final_columns()[:, finalized_src_rows(m.ram_log_size)])
    h_proof, h_claimed, h_aux = M.prove(m, backend, m.fill_main_trace(), None)
    d_proof, d_claimed, d_aux = M.prove(m, backend, None, None, resident=m.device_trees(backend.ctx))
    assert d_aux["roots"] == h_aux["roots"]
    assert d_claimed == h_claimed
    assert d_proof == h_proof


def test_generic_table_count_refuses_the_repeated_zero_of_multiplicity8(backend, machines):
    """The known limit of nb200_table_multiplicities: the Range8 table lists the tuple (0) nine times (multiplicity8.rs:48)."""
    m = machines["small"]
    tree0, tree1 = m.device_trees(backend.ctx)
    with pytest.raises(nb.Nb200Error, match="status 2: table_multiplicities: a table lists the same tuple in two rows of one relation"):
        M.fill_table_multiplicities(m, backend.ctx, tree0, tree1)


def test_bad_arguments_are_refused_and_the_context_stays_usable(backend):
    ctx = backend.ctx
    _name, (inputs, addresses, ts), (ia, iv) = edge_side_notes()[1]
    addresses, ts = addresses.astype(np.uint32), ts.astype(np.uint32)
    n_addr = W.last_access(inputs, addresses, ts, ia, iv)[0].size
    log_size = W.ram_log_size(n_addr)
    out = ctx.alloc(W.RAM_COLS, log_size)

    def refused(*args, log=log_size, batch=out):
        with pytest.raises(nb.Nb200Error, match="status 2"):
            ctx.ram_init_final_trace(*args, log, out=batch)

    refused(inputs[:0], addresses[:0], ts[:0], ia, iv)                           # no permutation
    a = addresses.copy()
    a[1] = (1 << 32) - 199                                                      # byte 199 would be at 2^32
    refused(inputs, a, ts, ia, iv)
    t = ts.copy()
    t[2, 7] = (1 << 32) - 1                                                     # a counter that would wrap
    refused(inputs, addresses, t, ia, iv)
    b = ia.copy()
    b[[3, 4]] = b[[4, 3]]                                                       # init addresses not ascending
    refused(inputs, addresses, ts, b, iv)
    b = ia.copy()
    b[4] = b[3]                                                                 # ... nor strictly
    refused(inputs, addresses, ts, b, iv)
    refused(inputs, addresses, ts, ia, iv, batch=ctx.alloc(W.RAM_COLS, log_size + 1))   # a batch of another shape
    small = ctx.alloc(W.RAM_COLS, log_size - 1)                                 # too few rows: refused, the count reported
    with pytest.raises(nb.Nb200Error, match=rf"status 2: .*more distinct addresses \({n_addr}\)"):
        ctx.ram_init_final_trace(inputs, addresses, ts, ia, iv, log_size - 1, out=small)
    got, n_rows = ctx.ram_init_final_trace(inputs, addresses, ts, ia, iv, log_size, out=out)
    assert n_rows == n_addr
    assert np.array_equal(got.download(), W.ram_init_final_columns(inputs, addresses, ts, ia, iv, log_size)[:, finalized_src_rows(log_size)])


def test_large_whole_machine_proof_is_accepted(backend):
    """Main component at 2^20 rows, 2^12 permutations, every extension tree filled on the device."""
    m = W.NexusV1KeccakMachine(20, 1 << 12)
    proof, claimed, aux = M.prove(m, backend, None, None, resident=m.device_trees(backend.ctx))
    assert M.verify_claimed_sums(claimed)
    verify_with_replayed_transcript(m, proof, claimed, aux)
