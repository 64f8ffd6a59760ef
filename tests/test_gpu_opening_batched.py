"""The opening stages without a host round trip per step (run on an H100: `pytest -m gpu`):

  1. the channel run by one device thread between FRI's inner layers (csrc/device_channel.cuh) draws what the host channel draws, over
     many random roots, under both draw flavours, and through a rejected draw (a digest whose first draw has a word >= 2P, found on the
     host by brute force and checked here);
  2. the decommitment planned on the host and fetched with one gather equals the oracle's MerkleProver::decommit on a multi-size tree and
     on FRI-layer shaped trees;
  3. OODS evaluation as one launch over many (column, point) pairs equals the oracle's eval_at_point, for columns of 2^0 .. 2^21
     coefficients at 1 or 2 points;
  4. whole proofs, whose FRI commit, OODS sampling and decommitment run through all three, equal the oracle's proof bytes."""
import ctypes as C
import gc

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.prover import Channel, CudaBackend
from oracle import pyoracle as orc
from tests import opening_ref as R
from tests.oracle_backend import OracleBackend

pytestmark = pytest.mark.gpu
P = (1 << 31) - 1
u32p, u64p, u8p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_uint8)
# digest words whose draw at n_sent = 0 (no domain separator) has word 4 >= 2P: the first draw after this state is rejected
REJECTING_DIGEST = np.array([40084852, 0, 0x6E657875, 0, 0, 0, 0, 0], dtype="<u4").tobytes()


@pytest.fixture(scope="module")
def ctx():
    c = nb.Context(0)
    yield c
    gc.collect()
    c.close()


class PyChannel:
    """HostChannel restated on the oracle's RFC Blake2s-256: mix_root and draw_felt only."""

    def __init__(self, digest=bytes(32), n_sent=0, domain_sep=0):
        self.digest, self.n_sent, self.sep = digest, n_sent, domain_sep

    def mix_root(self, root):
        self.digest, self.n_sent = orc.blake2s(self.digest + root), 0

    def draw_words(self):
        data = self.digest + self.n_sent.to_bytes(8, "little") + bytes(24) + (b"\0" if self.sep else b"")
        self.n_sent += 1
        return np.frombuffer(orc.blake2s(data), dtype="<u4")

    def draw_felt(self):
        while True:
            w = self.draw_words()
            if (w < 2 * P).all():
                return [int(x) - P if x >= P else int(x) for x in w[:4]]


def device_draw(ctx, digest, n_sent, roots, n):
    felts = np.zeros(4 * n, np.uint32)
    dout = (C.c_uint8 * 32)()
    nout = C.c_uint64()
    rb = b"".join(roots) if roots is not None else None
    rbuf = (C.c_uint8 * len(rb)).from_buffer_copy(rb) if rb else None
    ctx._chk(nb.lib().nb200_device_channel_draw(ctx._h, (C.c_uint8 * 32).from_buffer_copy(digest), C.c_uint64(n_sent), rbuf, C.c_size_t(n),
                                                 felts.ctypes.data_as(u32p), dout, C.byref(nout)))
    return [list(map(int, felts[4 * i:4 * i + 4])) for i in range(n)], bytes(dout), nout.value


@pytest.mark.parametrize("domain_sep", [0, 1])
def test_device_channel_draws_what_the_host_channel_draws(ctx, domain_sep):
    ctx.set_flavor(draw_domain_sep=domain_sep)
    try:
        rng = np.random.default_rng(40 + domain_sep)
        roots = [rng.integers(0, 256, 32, dtype=np.uint8).tobytes() for _ in range(200)]
        got, digest, n_sent = device_draw(ctx, bytes(32), 0, roots, len(roots))
        host = Channel(ctx)            # the prover's own host channel
        ref = PyChannel(domain_sep=domain_sep)
        for i, r in enumerate(roots):
            host.mix_root(r)
            ref.mix_root(r)
            want = [int(x) for x in np.asarray(host.draw_felt(), dtype=np.uint32).reshape(-1)[:4]]
            assert got[i] == want == ref.draw_felt(), f"draw {i}"
        assert digest == host.digest() == ref.digest and n_sent == ref.n_sent
    finally:
        ctx.set_flavor()


def test_device_channel_retries_a_rejected_draw(ctx):
    ref = PyChannel(REJECTING_DIGEST, 0)
    assert not (ref.draw_words() < 2 * P).all(), "the fixture digest no longer gives a rejected first draw"
    ref = PyChannel(REJECTING_DIGEST, 0)
    want = ref.draw_felt()
    assert ref.n_sent == 2
    got, digest, n_sent = device_draw(ctx, REJECTING_DIGEST, 0, None, 1)
    assert got[0] == want and n_sent == 2 and digest == REJECTING_DIGEST
    # and from a state in the middle of a transcript: draws without a mix continue the count
    got, _d, n_sent = device_draw(ctx, REJECTING_DIGEST, 0, None, 3)
    assert got[0] == want and got[1:] == [ref.draw_felt(), ref.draw_felt()] and n_sent == ref.n_sent


def _queries(rng, log, n):
    size = 1 << log
    q = {0, size - 1} | {int(r) for r in rng.integers(0, size, n)}
    return sorted(q)


def _check(tree, flat, queries, what):
    g_vals, g_hash, g_cols = tree.decommit(queries)
    o_vals, o_hash, o_cols = orc.merkle_decommit(flat, queries)
    assert np.array_equal(g_vals, o_vals), f"{what}: queried values"
    assert g_hash == o_hash, f"{what}: hash witness"
    assert np.array_equal(g_cols, o_cols), f"{what}: column witness"


def test_one_gather_decommitment_of_a_multi_size_tree(ctx):
    rng = np.random.default_rng(7)
    host = [rng.integers(0, P, (n, 1 << l), dtype=np.uint32) for n, l in ((19, 14), (3, 11), (5, 8), (2, 3))]
    flat = [c for h in host for c in h]
    tree = ctx.merkle_commit([ctx.upload(h) for h in host])
    assert tree.root == orc.merkle_commit(flat)
    for queries in ({14: _queries(rng, 14, 40)}, {14: _queries(rng, 14, 20), 11: _queries(rng, 11, 9), 8: _queries(rng, 8, 5), 3: [0, 5, 7]},
                    {8: _queries(rng, 8, 30)}):
        _check(tree, flat, queries, f"queries at {sorted(queries)}")


@pytest.mark.parametrize("log", [1, 4, 10, 17, 20])
def test_one_gather_decommitment_of_a_fri_layer(ctx, log):
    """A FRI layer: one secure column (4 coordinate columns) queried at sibling pairs."""
    rng = np.random.default_rng(log)
    host = rng.integers(0, P, (4, 1 << log), dtype=np.uint32)
    tree = ctx.merkle_commit([ctx.upload(host)])
    q = sorted({p ^ b for p in _queries(rng, log, 3) for b in (0, 1)})
    _check(tree, list(host), {log: q}, f"layer 2^{log}")


def test_one_launch_oods_of_mixed_sizes(ctx):
    """Batches of 2^0 .. 2^21 coefficients at 1 or 2 points (one launch per batch, many (column, point) pairs per launch)."""
    rng = np.random.default_rng(11)
    base = R.oods_point(tuple(int(v) for v in rng.integers(0, P, 4)))
    for log, n_cols, n_pts in ((0, 2, 1), (1, 3, 2), (5, 4, 2), (9, 7, 1), (15, 3, 2), (16, 2, 1), (21, 2, 2)):
        host = rng.integers(0, P, (n_cols, 1 << log), dtype=np.uint32)
        pw = np.array([R.point_words(R.shifted(base, max(log, 1), k)) for k in range(n_pts)], dtype=np.uint32)
        got = ctx.eval_at_points(ctx.upload(host), pw)
        for c in range(n_cols):
            for k in range(n_pts):
                want = orc.eval_at_point(host[c], pw[k, :4], pw[k, 4:])
                assert np.array_equal(got[c, k], want), f"log {log} column {c} point {k}"


@pytest.mark.parametrize("config", [None, dict(pow_bits=5, log_blowup=1, log_last=0, n_queries=20)], ids=["default", "20 queries"])
def test_whole_proof_bytes_equal_the_oracle(ctx, config):
    from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
    m = NexusV1Machine(12)
    cols = m.fill_main_trace(seed=3)
    g_proof, g_claimed, _ = M.prove(m, CudaBackend(ctx), cols, None, config=config)
    o_proof, o_claimed, _ = M.prove(m, OracleBackend(), cols, None, config=config)
    assert g_proof == o_proof and g_claimed == o_claimed
