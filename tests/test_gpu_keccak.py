"""The keccak precompile extension (nexus_zkvm_b200/keccak.py) proven on the GPU (run on an H100: `pytest -m gpu`): proof bytes equal to the
oracle's at two small sizes, a tampered witness refused and named by the constraint check, and a large proof accepted by the oracle's
verifier."""
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import keccak as K
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.prover import CudaBackend
from tests.oracle_backend import OracleBackend, verify, verify_with_replayed_transcript

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def backend():
    b = CudaBackend(nb.Context(0))
    yield b
    b.ctx.close()


@pytest.mark.parametrize("log_n_perms,n_queries", [(6, 3), (8, 40)])
def test_proof_bytes_match_oracle(backend, log_n_perms, n_queries):
    """KeccakRound 0 at 2^10 / 2^12 rows (the 200-value State relation, 1042 paired fractions per row, 9 preprocessed columns per round
    component, the expanded bitwise tables): the GPU's proof bytes are the oracle's and the oracle's verifier accepts them."""
    import os
    from oracle import pyoracle as orc
    orc.set_num_threads(os.cpu_count() or 1)
    m = K.KeccakMachine(log_n_perms, seed=log_n_perms)
    cols = m.fill_main_trace()
    cfg = dict(pow_bits=5, log_blowup=1, log_last=0, n_queries=n_queries)
    g_proof, g_claimed, g_aux = M.prove(m, backend, cols, None, config=cfg, associated_data=b"keccak")
    o_proof, o_claimed, o_aux = M.prove(m, OracleBackend(), cols, None, config=cfg, associated_data=b"keccak")
    assert g_aux["roots"] == o_aux["roots"]
    assert g_claimed == o_claimed
    assert g_proof == o_proof, f"proof bytes differ (len {len(g_proof)} vs {len(o_proof)})"
    verify(m, g_proof, o_aux)


def test_tampered_witness_is_refused_and_named(backend):
    """One byte of a rotation's output lane in KeccakRound 0: the proof stops with NB200_ERR_CONSTRAINTS and the GPU's constraint check names
    rotate_left's constraint for that byte (degree 1) at that row, in that component only."""
    m = K.KeccakMachine(6, seed=1)
    cols = m.fill_main_trace()
    row, out_lane = 37, (25 + 20 + 2) * K.LANE_SIZE     # the first rotation's output lane (after the input state, C's XORs, low, high)
    bad = [c.copy() for c in cols]
    bad[1][out_lane + 3, row] ^= 1
    with pytest.raises(nb.Nb200Error, match="status 5"):
        M.prove(m, backend, bad, None)
    report, _ = M.check_constraints(m, backend, bad, None)
    assert report[1] == [(3, 1, 1, row)]
    assert not any(report[k] for k in (0, 2, 3, 4, 5))
    report, _ = M.check_constraints(m, backend, cols, None)
    assert not any(report.values())


def test_large_proof_is_accepted(backend):
    """2^14 - 1 permutations: KeccakRound 0 at 2^18 rows (1705 main and 2084 interaction columns), KeccakRound 1 at 2^17."""
    m = K.KeccakMachine(14)
    cols = m.fill_main_trace()
    proof, claimed, aux = M.prove(m, backend, cols, None)
    verify_with_replayed_transcript(m, proof, claimed, aux)
