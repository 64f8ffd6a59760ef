"""The keccak extension's main trace filled on the device from its side note (nb200_keccak_main_trace, csrc/keccak_trace.cu; run on an H100:
`pytest -m gpu`): the five batches equal the numpy columns in finalized order bit for bit, proofs from them equal proofs from the host columns,
a large one is accepted by the verifier, a tampered cell is refused and named, bad side notes are rejected, and the scratch memory goes back to
the pool."""
import gc

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import keccak as K
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.prover import CudaBackend
from tests.keccak_side_notes import edge_machine, finalized_main_trace, finalized_src_rows
from tests.oracle_backend import verify_with_replayed_transcript
from tests.test_gpu_prove_ownership import _settled_pool_bytes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def backend():
    b = CudaBackend(nb.Context(0))
    yield b
    gc.collect()
    b.ctx.close()


def _machine(kind):
    if kind[0] == "edge":
        return edge_machine(kind[1], seed=kind[1])
    if kind[0] == "n":
        return K.KeccakMachine(None, seed=kind[1], n_perms=kind[1])
    return K.KeccakMachine(kind[1], seed=kind[1])


@pytest.mark.parametrize("kind", [("log", 4), ("log", 6), ("n", 37), ("n", 16), ("edge", 1), ("edge", 37), ("edge", 64), ("log", 8), ("log", 14)])
def test_device_batches_equal_the_numpy_columns(backend, kind):
    m = _machine(kind)
    batches = backend.ctx.keccak_main_trace(*m.side_note())
    want = finalized_main_trace(m)
    assert [(b.n_cols, b.log_size) for b in batches] == [(w.shape[0], w.shape[1].bit_length() - 1) for w in want]
    for k, (b, w) in enumerate(zip(batches, want)):
        got = b.download()
        bad = np.argwhere(got != w)
        assert bad.size == 0, f"batch {k}: {len(bad)} cells differ, first (column, position) {tuple(bad[0])}"
        del got
        b.free()


@pytest.mark.parametrize("log_n_perms,n_queries", [(6, 3), (8, 40)])
def test_proof_from_the_device_fill_equals_the_host_columns_proof(backend, log_n_perms, n_queries):
    m = K.KeccakMachine(log_n_perms, seed=log_n_perms)
    cfg = dict(pow_bits=5, log_blowup=1, log_last=0, n_queries=n_queries)
    h_proof, h_claimed, h_aux = M.prove(m, backend, m.fill_main_trace(), None, config=cfg, associated_data=b"keccak")
    d_proof, d_claimed, d_aux = M.prove(m, backend, None, None, config=cfg, associated_data=b"keccak", resident=m.device_trees(backend.ctx))
    assert d_aux["roots"] == h_aux["roots"]
    assert d_claimed == h_claimed
    assert d_proof == h_proof


def test_large_device_filled_proof_is_accepted(backend):
    """2^14 - 1 permutations: KeccakRound 0 at 2^18 rows, filled on the device."""
    m = K.KeccakMachine(14)
    proof, claimed, aux = M.prove(m, backend, None, None, resident=m.device_trees(backend.ctx))
    verify_with_replayed_transcript(m, proof, claimed, aux)


def test_tampered_device_cell_is_refused_and_named(backend):
    """One byte of the first rotation's output lane at trace row 37 of KeccakRound 0, changed in the device batch: the proof stops with
    NB200_ERR_CONSTRAINTS and the constraint check on the resident trees names rotate_left's constraint for that byte at that row."""
    m = K.KeccakMachine(6, seed=1)
    row, out_lane = 37, (25 + 20 + 2) * K.LANE_SIZE
    tree0, tree1 = m.device_trees(backend.ctx)
    rnd = tree1[1].download()
    pos = int(np.flatnonzero(finalized_src_rows(tree1[1].log_size) == row)[0])
    rnd[out_lane + 3, pos] ^= 1
    tree1[1].upload(rnd)
    with pytest.raises(nb.Nb200Error, match="status 5"):
        M.prove(m, backend, None, None, resident=(tree0, tree1))
    report, _ = M.check_constraints(m, backend, None, None, resident=(tree0, tree1))
    assert report[1] == [(3, 1, 1, row)]
    assert not any(report[k] for k in (0, 2, 3, 4, 5))
    report, _ = M.check_constraints(m, backend, None, None, resident=m.device_trees(backend.ctx))
    assert not any(report.values())


def test_bad_side_notes_are_rejected(backend):
    ctx = backend.ctx
    inputs, addresses, timestamps = K.KeccakMachine(4, seed=2).side_note()
    with pytest.raises(nb.Nb200Error, match="status 2"):
        ctx.keccak_main_trace(inputs[:0], addresses[:0], timestamps[:0])
    a = addresses.copy()
    a[7] = (1 << 32) - 199                      # byte 199 would be at 2^32
    with pytest.raises(nb.Nb200Error, match="status 2"):
        ctx.keccak_main_trace(inputs, a, timestamps)
    a[7] = (1 << 32) - 200                      # the last range that fits is accepted
    for b in ctx.keccak_main_trace(inputs, a, timestamps):
        b.free()
    t = timestamps.copy()
    t[3, 11] = (1 << 32) - 1
    with pytest.raises(nb.Nb200Error, match="status 2"):
        ctx.keccak_main_trace(inputs, addresses, t)
    n = (1 << 18) + 1                           # beyond the 32-bit multiplicity counters' bound
    with pytest.raises(nb.Nb200Error, match="status 2"):
        ctx.keccak_main_trace(np.zeros((n, 25), np.uint64), np.zeros(n, np.uint32), np.zeros((n, 200), np.uint32))


def test_fill_and_free_return_the_pool_to_its_baseline(backend):
    ctx = backend.ctx
    side_note = K.KeccakMachine(8, seed=4).side_note()
    for b in ctx.keccak_main_trace(*side_note):  # warm-up: the first fill may leave the pool larger, not more used
        b.free()
    base = _settled_pool_bytes(ctx)
    batches = ctx.keccak_main_trace(*side_note)
    assert _settled_pool_bytes(ctx) > base
    for b in batches:
        b.free()
    assert _settled_pool_bytes(ctx) == base
