"""Self-consistency of the oracle's full prover (CPU): a proof of the Nexus-shaped synthetic machine is accepted by
the oracle's independent verifier; tampering and unsatisfied constraints are rejected.  (The reference's own
proving tests are exactly this kind of prove -> verify round trip: prover/src/machine.rs:505-533.)"""
import numpy as np
import pytest

from nexus_zkvm_b200 import machine as M
from oracle import pyoracle as orc
from tests.oracle_backend import OracleBackend, verify

P = (1 << 31) - 1


@pytest.fixture(scope="module")
def proved():
    m = M.AddMachine(log_size=8, n_lanes=2)
    cols, mult = m.fill_main_trace(seed=3, n_padding=5)
    proof, claimed, aux = M.prove(m, OracleBackend(), cols, mult, associated_data=b"\x01\x02")
    return m, proof, claimed, aux


def test_air_shape():
    m = M.AddMachine(log_size=8, n_lanes=21)
    assert m.air.n_columns() == [3, 2 + 16 * 21 + 1, 4 * 12 * 21 + 4]  # 3 / 339 / 1012 columns
    assert len(m.main.constraints) == 3 + 8 * 21 + 12 * 21


def test_oracle_proof_verifies(proved):
    m, proof, claimed, aux = proved
    assert M.verify_claimed_sums(claimed)
    verify(m, proof, aux)
    assert 1000 < len(proof) < 200000


def test_tampered_proof_rejected(proved):
    m, proof, claimed, aux = proved
    rng = np.random.default_rng(0)
    rejected = 0
    for _ in range(12):
        i = int(rng.integers(8, len(proof)))
        bad = bytearray(proof); bad[i] ^= 1 << int(rng.integers(0, 7))
        try:
            verify(m, bytes(bad), aux)
        except orc.OracleError:
            rejected += 1
    assert rejected == 12


@pytest.mark.parametrize("log_last", [0, 1, 2, 3])
def test_proof_with_a_larger_last_fri_layer_verifies(log_last):
    """The last FRI layer is sent as a LinePoly of 2^log_last coefficients.  From four coefficients on, its evaluation at a query depends on
    which doubling of x multiplies which split of the coefficients; with one or two coefficients every order gives the same value."""
    m = M.AddMachine(log_size=9, n_lanes=1)
    cols, mult = m.fill_main_trace(seed=9)
    proof, _claimed, aux = M.prove(m, OracleBackend(), cols, mult, config=dict(pow_bits=5, log_blowup=1, log_last=log_last, n_queries=10))
    verify(m, proof, aux)


def test_unsatisfied_constraint_is_reported():
    m = M.AddMachine(log_size=8, n_lanes=1)
    cols, mult = m.fill_main_trace(seed=4)
    cols[2 + 8][17] = (int(cols[2 + 8][17]) + 1) % 256  # break c[0] of the ADD at row 17 (also breaks the range multiset)
    with pytest.raises(orc.OracleError, match="ConstraintsNotSatisfied"):
        M.prove(m, OracleBackend(), cols, mult)


def test_larger_trace_with_mixed_sizes():
    m = M.AddMachine(log_size=10, n_lanes=1)
    cols, mult = m.fill_main_trace(seed=5)
    proof, claimed, aux = M.prove(m, OracleBackend(), cols, mult)
    assert M.verify_claimed_sums(claimed)
    verify(m, proof, aux)


def test_paired_logup_proof_verifies():
    m = M.AddMachine(log_size=8, n_lanes=2, logup_in_pairs=True)
    cols, mult = m.fill_main_trace(seed=6)
    proof, claimed, aux = M.prove(m, OracleBackend(), cols, mult)
    assert M.verify_claimed_sums(claimed)
    verify(m, proof, aux)


# ---- backend-trait level oracle functions (the checkers of tests/test_gpu_backend_ops.py) ---------------------------
def test_oracle_fold_ops_are_linear_and_grind_is_minimal():
    import hashlib
    rng = np.random.default_rng(42)
    P = (1 << 31) - 1
    a, b = (rng.integers(0, P, size=(4, 64), dtype=np.uint32) for _ in range(2))
    alpha = rng.integers(0, P, size=4, dtype=np.uint32)
    s = ((a.astype(np.uint64) + b) % P).astype(np.uint32)
    add = lambda x, y: ((x.astype(np.uint64) + y) % P).astype(np.uint32)
    assert np.array_equal(orc.fold_line(s, alpha), add(orc.fold_line(a, alpha), orc.fold_line(b, alpha)))
    z = np.zeros((4, 32), np.uint32)
    assert np.array_equal(orc.fold_circle_into_line(z, s, alpha), add(orc.fold_circle_into_line(z, a, alpha), orc.fold_circle_into_line(z, b, alpha)))
    # folding a constant secure column: f0 = f1 = c -> (c + c) + alpha * 0 = 2c
    c = np.tile(np.array([[5], [6], [7], [8]], np.uint32), (1, 16))
    assert np.array_equal(orc.fold_line(c, alpha), np.tile(np.array([[10], [12], [14], [16]], np.uint32), (1, 8)))
    # grind: the nonce satisfies the predicate and no smaller one does (pow_variant 0: Blake2s(digest || nonce_le))
    digest = bytes(range(32))
    def tz(nonce):
        h = hashlib.blake2s(digest + nonce.to_bytes(8, "little")).digest()
        v = int.from_bytes(h[:16], "little")
        return 128 if v == 0 else (v & -v).bit_length() - 1
    n = orc.grind(digest, 9)
    assert tz(n) >= 9 and all(tz(k) < 9 for k in range(n))


def test_half_domain_decomposition_used_by_the_quotient_step():
    """DESIGN §4a: in the circle-FFT basis a polynomial with coefficients [lo | hi] (2^(m+1) of them) equals lo on
    CanonicCoset(m).circle_domain() (the top basis element pi^(m-1)(x) vanishes there) and lo + t * hi on the first half of
    CanonicCoset(m+1).circle_domain() with ONE constant t.  Checked here with the oracle's evaluate / eval_at_point."""
    P = (1 << 31) - 1
    rng = np.random.default_rng(0)
    for m in (3, 6):
        c = rng.integers(0, P, size=1 << (m + 1), dtype=np.uint32)
        lo, hi = c[:1 << m].copy(), c[1 << m:].copy()
        ev_lo = orc.evaluate(lo, m)                           # bit-reversed evaluations of lo on canonic(m)
        for i in range(1 << m):
            x, y = orc.circle_domain_at(m, i)
            v = orc.eval_at_point(c, (x, 0, 0, 0), (y, 0, 0, 0))
            assert tuple(int(t) for t in v) == (int(ev_lo[orc.bit_reverse_index(i, m)]), 0, 0, 0)
        z = np.zeros(1 << m, np.uint32)
        full = orc.evaluate(c, m + 1)
        e_lo = orc.evaluate(np.concatenate([lo, z]), m + 1)
        e_hi = orc.evaluate(np.concatenate([hi, z]), m + 1)
        h = 1 << m
        ts = {(int(full[i]) - int(e_lo[i])) % P * orc.m31_inv(int(e_hi[i])) % P for i in range(h) if int(e_hi[i])}
        assert len(ts) == 1
        t = ts.pop()
        assert all((int(e_lo[i]) + t * int(e_hi[i])) % P == int(full[i]) for i in range(h))


def test_nexus_v1_main_component_oracle_prove_and_verify():
    """The recorded v1 main component (nexus_zkvm_b200/nexus_v1.py) with its padding-only witness: the oracle proves it, its verifier accepts,
    the LogUp sums of the three components cancel, the column counts are the reference's 27 / 347 / 1012 (+ the two tables' columns), and a row
    that is not padding (without a matching opcode flag) is rejected."""
    from nexus_zkvm_b200 import machine as M
    from nexus_zkvm_b200.nexus_v1 import NexusV1Machine, MAIN_COLUMNS
    from tests.oracle_backend import OracleBackend, verify
    m = NexusV1Machine(8)
    assert m.air.n_columns() == [27 + 2, 347 + 2, 1012 + 8]
    assert [len(c.fracs) for c in m.air.components] == [253, 1, 1]
    cols = m.fill_main_trace(seed=3)
    proof, claimed, aux = M.prove(m, OracleBackend(), cols, None)
    assert M.verify_claimed_sums(claimed)
    verify(m, proof, aux)
    off = sum(s for n, s in MAIN_COLUMNS[:[n for n, _ in MAIN_COLUMNS].index("IsPadding")])
    cols[off] = cols[off].copy(); cols[off][7] = 0
    with pytest.raises(Exception, match="ConstraintsNotSatisfied"):
        M.prove(m, OracleBackend(), cols, None)


def test_nexus_v1_rank_local_witness_is_partition_independent_and_satisfies_the_air():
    """NexusV1Machine.fill_main_trace_shard / preprocessed_shard (the generators the multi-GPU proofs use so that no rank builds the whole trace):
    any partition of the columns yields the same values and histograms, the preprocessed shard equals the full list, and the oracle proves and
    verifies the assembled witness (the AIR's constraints and LogUp sums hold)."""
    import numpy as np
    from nexus_zkvm_b200 import machine as M
    from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
    m = NexusV1Machine(8)
    full, h256, h32 = m.fill_main_trace_shard(3, 0, m.n_main)
    parts, g256, g32 = [], 0, 0
    for first, count in [(0, 48), (48, 160), (208, 139)]:
        out = np.empty((count, 256), np.uint32)
        block, a, b = m.fill_main_trace_shard(3, first, count, out=out)
        assert block is out
        parts += list(out); g256 = g256 + a; g32 = g32 + b
    assert all(np.array_equal(x, y) for x, y in zip(full, parts))
    assert np.array_equal(h256, g256) and np.array_equal(h32, g32)
    ref = m._preprocessed_list()
    for first, count in [(0, 16), (16, 11), (3, 20)]:
        block, tables = m.preprocessed_shard(first, count)
        assert np.array_equal(block, np.stack(ref[first:first + count]))
        assert np.array_equal(tables[0], ref[27]) and np.array_equal(tables[1], ref[28])
    assert m.preprocessed_shard(27, 0)[0] is None
    cols = full + m.multiplicity_columns(h256, h32)
    proof, claimed, aux = M.prove(m, OracleBackend(), cols, None, associated_data=b"sh")
    assert M.verify_claimed_sums(claimed)
    verify(m, proof, aux)
