"""The DEEP quotients of a proof's non-sharded column groups (csrc/prove.cu quotients_from_coeffs): every sample batch's columns combined
on their coefficients (deep_combine_kernel), the combinations extended, then quotients_combined_kernel.  Run on an H100: `pytest -m gpu`.

The route must give, word for word, the quotient accumulate_quotients computes over the committed LDEs (nb200_fri_quotients, itself
checked against the oracle in tests/test_gpu_opening_at_scale.py).  Here the LDEs are the GPU's own evaluations of the same coefficients.
Inputs are full-entropy and edge columns (all P - 1: the largest sums of the lazily reduced accumulators, zero, zero but the last word),
from 2^5 to the benchmarked proof's 2^21-row LDE, with batches whose columns repeat across points and batches of one column.  A whole
v1 proof at 2^16 rows, whose main column group goes through the route, must equal the oracle's."""
import gc
import os

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200 import prover as NP
from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
from oracle import pyoracle as orc
from tests import opening_ref as R
from tests import random_witness as rw
from tests.oracle_backend import OracleBackend, verify
from tests.test_gpu_opening_at_scale import _edge_columns, _qm31, _same

pytestmark = pytest.mark.gpu
P = (1 << 31) - 1


@pytest.fixture(scope="module", autouse=True)
def _oracle_threads():
    before = orc.num_threads()
    orc.set_num_threads(os.cpu_count())
    yield
    orc.set_num_threads(before)


@pytest.fixture(scope="module")
def ctx():
    c = nb.Context(0)
    yield c
    gc.collect()
    c.close()


def _values(rng, k):
    return [rw.mixed(rng, 4) for _ in range(k)]


def _both_routes(ctx, host_coeffs, blow, batches, rc, what, oracle=False):
    """The quotient from the coefficients and from their LDEs (evaluated on the GPU); equal word for word, and, when `oracle`, equal to
    the oracle's quotient over the downloaded LDEs."""
    n_log = int(np.log2(host_coeffs[0].shape[1]))
    log = n_log + blow
    coeffs = [ctx.upload(h) for h in host_coeffs]
    ldes = [ctx.evaluate(c, blow) for c in coeffs]
    want = NP.fri_quotients(ctx, ldes, log, batches, rc).download()
    got = NP.fri_quotients_from_coeffs(ctx, coeffs, log, blow, batches, rc)
    assert got.n_cols == 4 and got.log_size == log
    _same(got.download(), want, what)
    if oracle:
        host_ldes = np.concatenate([l.download() for l in ldes])
        _same(want, orc.accumulate_quotients(list(host_ldes), np.array(rc, np.uint32), batches), what + " (oracle)")


def _shifted_batches(rng, log, n_cols, counts):
    """One sample batch per count at its own point (shifts of one OODS point), over a shuffled choice of columns: a column appears in
    several batches."""
    oods = R.oods_point(_qm31(rng))
    return [(R.point_words(R.shifted(oods, max(log - 1, 1), k)), [(int(c), v) for c, v in zip(rng.permutation(n_cols)[:cnt], _values(rng, cnt))])
            for k, cnt in enumerate(counts)]


@pytest.mark.parametrize("blow", [1, 2, 3])
@pytest.mark.parametrize("n_log", [2, 3, 5, 8, 11, 16])
def test_every_batch_size(ctx, n_log, blow):
    """Batches of 1..17 columns (every residue of the 8- and 4-column loops and every tail below 4), at every size from the smallest the
    route takes (4 coefficients, one thread) up, against the LDE route and the oracle."""
    rng = np.random.default_rng(1000 * blow + n_log)
    host = _edge_columns(20, n_log, seed=n_log + 7 * blow, n_max=8)
    batches = _shifted_batches(rng, n_log + blow, 20, list(range(1, 18)))
    _both_routes(ctx, [host], blow, batches, _qm31(rng), f"combined DEEP quotients 2^{n_log} x blow-up {blow}", oracle=n_log <= 11)


@pytest.mark.parametrize("n_log", [5, 12])
def test_one_column_and_repeated_columns(ctx, n_log):
    """A lone batch of one column; then a column in every batch and every column at one point, over two device batches."""
    rng = np.random.default_rng(77 + n_log)
    host = [rng.integers(0, P, (7, 1 << n_log), dtype=np.uint32), _edge_columns(5, n_log, seed=n_log)]
    oods = R.oods_point(_qm31(rng))
    one = [(R.point_words(oods), [(9, rw.mixed(rng, 4))])]
    _both_routes(ctx, host, 1, one, _qm31(rng), f"one column 2^{n_log}", oracle=True)
    pts = [R.point_words(R.shifted(oods, n_log, k)) for k in (0, 1, -1, 2)]
    rep = [(pts[0], [(c, v) for c, v in zip(range(12), _values(rng, 12))])] + [(p, [(3, rw.mixed(rng, 4)), (10, rw.mixed(rng, 4))]) for p in pts[1:]]
    _both_routes(ctx, host, 1, rep, _qm31(rng), f"repeated columns 2^{n_log}", oracle=True)


@pytest.mark.parametrize("rc", [(1, 0, 0, 0), (P - 1, 0, 0, 0), None])
def test_proof_shape_at_2p20(ctx, rc):
    """The benchmarked proof's shape: 2^20 coefficients per column, a 2^21-row LDE, 205 columns in three device batches (the first 24 all
    P - 1) at the OODS point, three columns again at the mask-shifted point and a 4-column composition-like block at a third point."""
    n_log, blow = 20, 1
    rng = np.random.default_rng(2020)
    host = [_edge_columns(195, n_log, seed=3, n_max=24), _edge_columns(6, n_log, seed=4), rw.mixed(rng, 4 << n_log).reshape(4, -1)]
    oods = R.oods_point(_qm31(rng))
    vals = _values(rng, 212)
    batches = [(R.point_words(oods), [(c, vals[c]) for c in range(205)]),
               (R.point_words(R.shifted(oods, n_log, 1)), [(c, vals[205 + k]) for k, c in enumerate((0, 100, 194))]),
               (R.point_words(R.shifted(oods, n_log, -1)), [(201 + k, vals[208 + k]) for k in range(4)])]
    _both_routes(ctx, host, blow, batches, rc or _qm31(rng), f"combined DEEP quotients 205 x 2^20, random_coeff {rc}")


def test_rejects_what_the_route_cannot_take(ctx):
    rng = np.random.default_rng(5)
    co = ctx.upload(rng.integers(0, P, (2, 2), dtype=np.uint32))
    with pytest.raises(RuntimeError):   # 2 coefficients: below the 4-coefficient group of the kernels
        NP.fri_quotients_from_coeffs(ctx, [co], 2, 1, [(R.point_words(R.oods_point(_qm31(rng))), [(0, _qm31(rng))])], _qm31(rng))
    co = ctx.upload(rng.integers(0, P, (2, 16), dtype=np.uint32))
    with pytest.raises(RuntimeError):   # no sample batch
        NP.fri_quotients_from_coeffs(ctx, [co], 5, 1, [], _qm31(rng))


def test_v1_proof_at_2p16_equals_the_oracle(ctx):
    """A whole proof of bench.py's machine at 2^16 rows: its main size group (columns of trees 0, 1 and 2, some at two points) takes the
    combined route, the composition's few columns the LDE route; proof bytes and claimed sums equal the oracle's and the verifier accepts."""
    m = NexusV1Machine(16)
    cols = m.fill_main_trace(seed=16)
    g_proof, g_claimed, _ = M.prove(m, NP.CudaBackend(ctx), cols, None)
    o_proof, o_claimed, o_aux = M.prove(m, OracleBackend(), cols, None)
    assert g_claimed == o_claimed
    assert g_proof == o_proof, "proof bytes differ from the oracle's"
    verify(m, g_proof, o_aux)
