"""The kernels that run after the trace commits, at the sizes of the benchmarked proof (2^20 trace rows, 2^21-row LDE, blow-up 2), against
the oracle, bit-exact (run on an H100: `pytest -m gpu`):

  1. OODS sampling (csrc/evalpoint.cu): one CTA and 2..128 CTAs per column, 1 to 347 columns, 1, 2 and 64 points per call, at points drawn
     the way sample_oods draws them; and, independently of the oracle, at points of the LDE domain, where the value is an LDE word;
  2. DEEP quotients (csrc/pcs_kernels.cu): about 200 columns of 2^21 rows in three device batches, every batch size mod 8, the one- and
     two-thread launches of quotients_kernel_x4, and the scalar quotients_kernel on columns at a 4-byte offset; a plain Python restatement
     of the formula (tests/opening_ref.py) referees a few dozen rows of the largest case as well;
  3. FRI folds on the smallest twiddle bank each fold accepts and on a bank prepared for 2^24;
  4. Merkle decommitment of a mixed-size tree shaped like the v1 tree-1 LDE, the single-CTA tail of the last ten layers, and the chunked
     leaf hashing of nb200_commit_host, under both node-hash flavours;
  5. the LogUp finalisation (column sum, coset gather, recursive prefix scan) at 2^16..2^22 rows, where the scan recurses once or twice;
  6. whole proofs of bench.py's machine (NexusV1Machine) at 2^16 rows under the default and a many-query configuration.

Inputs reach the field's edges: columns that are all P - 1 (the largest sums of the lazily reduced 64-bit accumulators), zero, zero but the
last word (the last thread, the largest block weight), and random_witness.mixed.  A mismatch names the first differing column and row."""
import gc
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200 import prover as NP
from nexus_zkvm_b200.prover import CudaBackend
from oracle import pyoracle as orc
from tests import opening_ref as R
from tests import random_witness as rw
from tests.oracle_backend import OracleBackend, verify
from tests.test_gpu_commit_shapes import _Unaligned

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


@pytest.fixture(scope="module")
def big_bank_ctx():
    c = nb.Context(0)
    c.precompute_twiddles(24)
    yield c
    gc.collect()
    c.close()


def _edge_columns(n_cols, log, seed, n_max=0):
    """n_cols x 2^log words: the first n_max columns all P - 1, then in turn all P - 1, random_witness.mixed, zero but a non-zero last word,
    zero, uniform in [0, P)."""
    rng = np.random.default_rng(seed)
    n = 1 << log
    out = np.empty((n_cols, n), np.uint32)
    for c in range(n_cols):
        kind = 0 if c < n_max else (c - n_max) % 5
        if kind == 0:
            out[c] = P - 1
        elif kind == 1:
            out[c] = rw.mixed(rng, n)
        elif kind in (2, 3):
            out[c] = 0
            if kind == 2:
                out[c, n - 1] = rng.integers(1, P)
        else:
            out[c] = rng.integers(0, P, n, dtype=np.uint32)
    return out


def _same(got, exp, what, inner="row"):
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.shape == exp.shape, f"{what}: shape {got.shape} != {exp.shape}"
    g, e = got.reshape(got.shape[0], -1), exp.reshape(exp.shape[0], -1)
    bad = np.nonzero(g != e)
    if bad[0].size:
        c, r = int(bad[0][0]), int(bad[1][0])
        pytest.fail(f"{what}: {bad[0].size} words differ, the first in column {c} {inner} {r}: {g[c, r]} != {e[c, r]}")


def _qm31(rng):
    return tuple(int(v) for v in rng.integers(0, P, 4))


# ---- 1. OODS sampling --------------------------------------------------------------------------------------------------------------

def _oods_points(rng, log, n_points):
    """Points as sample_oods builds them: the circle point of a drawn t, then that point moved by one step of the trace domain (the point of a
    mask at row offset 1), then further drawn points and their shifts by -1.  Returns (n_points, 2, 4)."""
    out = []
    while len(out) < n_points:
        p = R.oods_point(_qm31(rng))
        out.append(p)
        out.append(R.shifted(p, max(log, 1), 1 if len(out) == 1 else -1))
    return np.array([[list(x), list(y)] for x, y in out[:n_points]], np.uint32)


def _oracle_eval(coeffs, points):
    jobs = [(c, k) for c in range(coeffs.shape[0]) for k in range(points.shape[0])]
    with ThreadPoolExecutor(os.cpu_count()) as ex:
        vals = list(ex.map(lambda ck: orc.eval_at_point(coeffs[ck[0]], points[ck[1], 0], points[ck[1], 1]), jobs))
    return np.array(vals, np.uint32).reshape(coeffs.shape[0], points.shape[0], 4)


# (log size, columns, points per call): sizes <= 15 are one CTA (EP_QMAX = 15) with LB < 8, LB = 8 and the largest block; from 2^16 on,
# 2..128 CTAs per column whose partials eval_points_sum_kernel adds
OODS = [(0, 5, 2), (3, 1, 64), (8, 5, 2), (9, 1, 64), (9, 5, 1), (14, 5, 64), (15, 5, 2), (15, 1, 64),
        (16, 5, 64), (16, 1, 1), (20, 1, 64), (20, 5, 2), (21, 5, 1), (21, 1, 2), (22, 5, 2), (22, 1, 64)]


@pytest.mark.parametrize("log,n_cols,n_points", OODS)
def test_eval_at_points_matches_oracle(ctx, log, n_cols, n_points):
    rng = np.random.default_rng(100 * log + n_cols + n_points)
    coeffs = _edge_columns(n_cols, log, seed=log + n_points)
    pts = _oods_points(rng, log, n_points)
    _same(ctx.eval_at_points(ctx.upload(coeffs), pts), _oracle_eval(coeffs, pts), f"eval_at_points 2^{log}", inner="point x coordinate")


@pytest.mark.parametrize("log,n_cols,n_points,n_max", [(20, 67, 2, 16), (16, 347, 1, 16), (16, 347, 2, 0)])
def test_eval_at_points_on_a_proof_sized_column_group(ctx, log, n_cols, n_points, n_max):
    """One eval_at_points launch per group of consecutive columns with the same mask offsets: 67 columns of 2^20 coefficients at the OODS
    point and its mask-shifted point, the 347 main columns of the v1 tree 1 at 2^16."""
    rng = np.random.default_rng(7 * n_cols + log)
    coeffs = _edge_columns(n_cols, log, seed=n_cols, n_max=n_max)
    pts = _oods_points(rng, log, n_points)
    _same(ctx.eval_at_points(ctx.upload(coeffs), pts), _oracle_eval(coeffs, pts), f"eval_at_points {n_cols} x 2^{log}", inner="point x coordinate")


@pytest.mark.parametrize("log", [0, 1, 8, 9, 15, 16, 20, 21])
def test_eval_at_points_on_the_lde_domain_equals_the_lde(ctx, log):
    """Independent of the oracle's eval_at_point: at the points of CanonicCoset(log + 1).circle_domain(), embedded in QM31, the sampled value
    is the LDE word at that position (the LDE from the oracle's FFT, the points from tests/opening_ref.py)."""
    rng = np.random.default_rng(300 + log)
    coeffs = _edge_columns(3, log, seed=300 + log)
    n = 2 << log
    rows = sorted({0, n - 1, n // 2 - 1, n // 2} | {int(r) for r in rng.integers(0, n, 12)})
    pts = np.array([[list(R.embed(x)), list(R.embed(y))] for x, y in (R.domain_point(log + 1, r) for r in rows)], np.uint32)
    got = ctx.eval_at_points(ctx.upload(coeffs), pts)
    for c in range(3):
        lde = orc.evaluate(coeffs[c], log + 1)
        want = np.array([[lde[r], 0, 0, 0] for r in rows], np.uint32)
        _same(got[c][None], want[None], f"column {c} on the LDE domain (rows {rows})", inner="point x coordinate")


# ---- 2. DEEP quotients -------------------------------------------------------------------------------------------------------------

RC_KINDS = ["one", "minus_one", "random"]


def _random_coeff(kind, rng):
    return {"one": (1, 0, 0, 0), "minus_one": (P - 1, 0, 0, 0)}.get(kind) or _qm31(rng)


def _values(rng, k):
    return [rw.mixed(rng, 4) for _ in range(k)]


def _check_quotients(ctx, batches_dev, host_cols, log, sample_batches, rc, what):
    got = NP.fri_quotients(ctx, batches_dev, log, sample_batches, rc)
    assert got.n_cols == 4 and got.log_size == log
    got = got.download()
    _same(got, orc.accumulate_quotients(list(host_cols), np.array(rc, np.uint32), sample_batches), what)
    return got


@pytest.fixture(scope="module")
def proof_sized_quotient_case(ctx):
    """205 columns of 2^21 rows in three device batches (195 trace-like columns, the first 24 all P - 1; 6 more; a 4-column composition-like
    block) and the proof's sample structure: every column at the OODS point (205 = 5 mod 8 entries), three columns at the mask-shifted
    point, the composition block at a third point."""
    log = 21
    rng = np.random.default_rng(2100)
    host = np.concatenate([_edge_columns(195, log, seed=1, n_max=24), _edge_columns(6, log, seed=2), rw.mixed(rng, 4 << log).reshape(4, -1)])
    dev = [ctx.upload(host[:195]), ctx.upload(host[195:201]), ctx.upload(host[201:])]
    oods = R.oods_point(_qm31(rng))
    vals = _values(rng, host.shape[0] + 7)
    batches = [(R.point_words(oods), [(c, vals[c]) for c in range(host.shape[0])]),
               (R.point_words(R.shifted(oods, log - 1, 1)), [(c, vals[205 + k]) for k, c in enumerate((0, 100, 194))]),
               (R.point_words(R.shifted(oods, log - 1, -1)), [(201 + k, vals[208 + k]) for k in range(4)])]
    yield log, host, dev, batches, rng
    del dev
    gc.collect()


@pytest.mark.parametrize("rc_kind", RC_KINDS)
def test_deep_quotients_at_2p21(ctx, proof_sized_quotient_case, rc_kind):
    log, host, dev, batches, rng = proof_sized_quotient_case
    rc = _random_coeff(rc_kind, rng)
    got = _check_quotients(ctx, dev, host, log, batches, rc, f"DEEP quotients 205 x 2^21, random_coeff {rc_kind}")
    # the plain restatement, on rows 0 and N - 1, both sides of several 4-row groups (one thread of quotients_kernel_x4 each) and random rows
    n = 1 << log
    rows = sorted({0, 1, 3, 4, 7, 8, 511, 512, n // 2 - 1, n // 2, n - 8, n - 5, n - 4, n - 1} | {int(r) for r in rng.integers(0, n, 50)})
    ref = R.deep_quotient_rows(lambda c, r: host[c, r], log, batches, rc, rows)
    for r in rows:
        assert tuple(int(v) for v in got[:, r]) == ref[r], f"row {r}: GPU {got[:, r]} != plain restatement {ref[r]}"


def _count_batches(rng, log, n_cols, counts):
    """One sample batch per count, each at its own point (shifts of one OODS point), over columns in a shuffled order."""
    oods = R.oods_point(_qm31(rng))
    return [(R.point_words(R.shifted(oods, max(log - 1, 1), k)), [(int(c), v) for c, v in zip(rng.permutation(n_cols)[:cnt], _values(rng, cnt))])
            for k, cnt in enumerate(counts)]


# log 1: the scalar kernel (no 4-row group); log 2 / 3: one / two threads of quotients_kernel_x4
@pytest.mark.parametrize("rc_kind", RC_KINDS)
@pytest.mark.parametrize("log", [1, 2, 3, 10, 16])
def test_deep_quotients_every_batch_size(ctx, log, rc_kind):
    """Sample batches of 1..17 entries: every residue mod 8 (the 8-column loop, the 4-column loop and the tail of quotients_kernel_x4) and
    every count below 4."""
    rng = np.random.default_rng(40 * log + len(rc_kind))
    host = _edge_columns(20, log, seed=log, n_max=8)
    batches = _count_batches(rng, log, 20, list(range(1, 18)))
    _check_quotients(ctx, [ctx.upload(host)], host, log, batches, _random_coeff(rc_kind, rng), f"DEEP quotients 2^{log}, random_coeff {rc_kind}")


@pytest.mark.parametrize("log", [10, 21])
def test_scalar_quotients_kernel_on_unaligned_columns(ctx, log):
    """Columns at a 4-byte offset cannot be read with 128-bit loads: quotients_launch falls back to the scalar quotients_kernel, which must
    give the words of quotients_kernel_x4 (itself compared with the oracle here)."""
    rng = np.random.default_rng(500 + log)
    host = _edge_columns(12, log, seed=500 + log, n_max=8)
    batches = _count_batches(rng, log, 12, [12, 8, 5, 3, 1])
    rc = _random_coeff("random", rng)
    aligned = _check_quotients(ctx, [ctx.upload(host)], host, log, batches, rc, f"DEEP quotients 2^{log} (aligned)")
    u = _Unaligned(ctx, 12, log)
    u.cols.upload(host)
    _same(NP.fri_quotients(ctx, [u.cols], log, batches, rc).download(), aligned, f"DEEP quotients 2^{log} (columns at a 4-byte offset)")


# ---- 3. FRI folds ------------------------------------------------------------------------------------------------------------------

def _alphas(rng):
    return [("0", (0, 0, 0, 0)), ("1", (1, 0, 0, 0)), ("random", _qm31(rng))]


@pytest.fixture
def fresh_ctx():
    c = nb.Context(0)
    yield c
    gc.collect()
    c.close()


def _fold_contexts(big_bank_ctx, fresh_ctx):
    """The fold on a bank prepared for 2^24 (entries far from the bank's end, as in a proof), then on a fresh context, whose bank the entry
    point prepares for the fold alone (the smallest bank it accepts: the fold reads its last entries)."""
    return [("a 2^24 twiddle bank", big_bank_ctx), ("a fresh context", fresh_ctx)]


@pytest.mark.parametrize("src_log", [3, 16, 21, 22])
def test_fold_circle_into_line_matches_oracle(big_bank_ctx, fresh_ctx, src_log):
    rng = np.random.default_rng(600 + src_log)
    src, dst = _edge_columns(4, src_log, 600 + src_log, n_max=1), rw.mixed(rng, 4 << (src_log - 1)).reshape(4, -1)
    want = {name: orc.fold_circle_into_line(dst, src, np.array(a, np.uint32)) for name, a in _alphas(np.random.default_rng(src_log))}
    for where, c in _fold_contexts(big_bank_ctx, fresh_ctx):
        g_src = c.upload(src)
        for name, a in _alphas(np.random.default_rng(src_log)):
            g = c.upload(dst)
            NP.fold_circle_into_line(c, g, g_src, a)
            _same(g.download(), want[name], f"fold_circle_into_line 2^{src_log}, alpha {name}, on {where}")
    assert nb.lib().nb200_twiddles_domain_log(fresh_ctx._h) == src_log
    assert nb.lib().nb200_twiddles_domain_log(big_bank_ctx._h) == 24


@pytest.mark.parametrize("src_log", [1, 20, 21])
def test_fold_line_matches_oracle(big_bank_ctx, fresh_ctx, src_log):
    src = _edge_columns(4, src_log, 700 + src_log, n_max=1)
    want = {name: orc.fold_line(src, np.array(a, np.uint32)) for name, a in _alphas(np.random.default_rng(src_log))}
    for where, c in _fold_contexts(big_bank_ctx, fresh_ctx):
        g_src = c.upload(src)
        for name, a in _alphas(np.random.default_rng(src_log)):
            _same(NP.fold_line(c, g_src, a).download(), want[name], f"fold_line 2^{src_log}, alpha {name}, on {where}")
    assert nb.lib().nb200_twiddles_domain_log(fresh_ctx._h) == src_log + 1
    assert nb.lib().nb200_twiddles_domain_log(big_bank_ctx._h) == 24


# ---- 4. Merkle decommitment --------------------------------------------------------------------------------------------------------

@pytest.fixture(params=[0, 1], ids=["chained-compressions", "blake2s-256"])
def merkle_hash(request, ctx):
    ctx.set_flavor(merkle_hash=request.param)
    orc.set_flavor(merkle_hash=request.param)
    yield request.param
    ctx.set_flavor()
    orc.set_flavor()


def _queries(rng, log, n_random):
    """0, the last leaf, sibling pairs (2k, 2k + 1), pairs that share only their grandparent (4k + 1, 4k + 2) and random leaves."""
    n = 1 << log
    q = {0, n - 1}
    for k in rng.integers(0, n // 4, 6):
        k = int(k)
        q |= {4 * k, 4 * k + 1} if k % 2 else {4 * k + 1, 4 * k + 2}
    q |= {int(r) for r in rng.integers(0, n, n_random)}
    return sorted(q)


def _check_decommit(tree, flat, queries, what):
    g_vals, g_hash, g_cols = tree.decommit(queries)
    o_vals, o_hash, o_cols = orc.merkle_decommit(flat, queries)
    _same(g_vals[None], o_vals[None], f"{what}: queried values", inner="word")
    assert len(g_hash) == len(o_hash), f"{what}: {len(g_hash)} witness hashes != {len(o_hash)}"
    bad = [i for i, (a, b) in enumerate(zip(g_hash, o_hash)) if a != b]
    assert not bad, f"{what}: {len(bad)} witness hashes differ, the first at {bad[0]}"
    _same(g_cols[None], o_cols[None], f"{what}: column witness", inner="word")


@pytest.fixture(scope="module")
def lde_shaped_tree(ctx):
    """Like the v1 tree-1 LDE at 2^20 trace rows: 70 columns of 2^21 (not a multiple of the 16-word message block), and smaller columns of
    2^9 and 2^6 injected into the inner layers."""
    host = [_edge_columns(70, 21, seed=21, n_max=16), _edge_columns(3, 9, seed=9), _edge_columns(2, 6, seed=6)]
    yield host, [ctx.upload(h) for h in host]
    gc.collect()


def test_merkle_decommit_of_an_lde_shaped_tree(ctx, merkle_hash, lde_shaped_tree):
    host, dev = lde_shaped_tree
    flat = [c for h in host for c in h]
    tree = ctx.merkle_commit(dev)
    assert tree.root == orc.merkle_commit(flat)
    rng = np.random.default_rng(800 + merkle_hash)
    big = _queries(rng, 21, 300)
    for queries in ({21: big}, {21: big, 9: _queries(rng, 9, 20), 6: _queries(rng, 6, 8)}, {9: _queries(rng, 9, 30), 6: _queries(rng, 6, 5)},
                    {6: [0, 63]}):
        _check_decommit(tree, flat, queries, f"queries at log sizes {sorted(queries)}")


def test_merkle_tail_of_the_last_ten_layers(ctx, merkle_hash):
    """The smallest column has 2^10 rows, so layers 2^9 .. 2^0 hold no columns: merkle_tail_kernel builds all ten in one CTA."""
    host = [_edge_columns(20, 12, seed=12, n_max=3), _edge_columns(3, 10, seed=10)]
    flat = [c for h in host for c in h]
    tree = ctx.merkle_commit([ctx.upload(h) for h in host])
    assert tree.root == orc.merkle_commit(flat)
    rng = np.random.default_rng(900)
    _check_decommit(tree, flat, {12: _queries(rng, 12, 40), 10: _queries(rng, 10, 10)}, "tail tree")


def test_commit_host_chunked_leaf_hashing_with_blake2s_256(ctx):
    """nb200_commit_host hashes the leaf layer chunk by chunk (64 columns of 2^20 rows per chunk) while the next chunk is copied; under the
    RFC Blake2s-256 node hash the byte counter of every compression carries across chunks.  71 columns: a full chunk and a partial one,
    whose last message block is partly filled."""
    ctx.set_flavor(merkle_hash=1)
    orc.set_flavor(merkle_hash=1)
    try:
        host = ctx.host_alloc(71, 20)
        host[:] = _edge_columns(71, 20, seed=71, n_max=16)
        small = _edge_columns(3, 8, seed=8)
        _evals, coeffs, ldes, tree = ctx.commit_host([host, small], 1)
        flat = []
        for k, h in enumerate((host, small)):
            oco, olde = orc.interpolate_evaluate_batch(h, 1, want_coeffs=True)
            _same(coeffs[k].download(), oco, "coefficients")
            _same(ldes[k].download(), olde, "LDE")
            flat += list(olde)
        assert tree.root == orc.merkle_commit(flat)
        _check_decommit(tree, flat, {21: _queries(np.random.default_rng(71), 21, 20)}, "chunked tree")
    finally:
        ctx.set_flavor()
        orc.set_flavor()


# ---- 5. LogUp finalisation at scale ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("log_size", [16, 20, pytest.param(21, marks=pytest.mark.slow), pytest.param(22, marks=pytest.mark.slow)])
def test_interaction_trace_at_scale(ctx, log_size):
    """nb200_gen_interaction_trace of AddMachine(n_lanes=1) on a full-entropy witness: the claimed sums do not cancel, so every row's shift
    matters.  2^20 rows are exactly 1024 scan blocks (one recursion of inclusive_scan); 2^21 and 2^22 recurse a second time."""
    m = M.AddMachine(log_size=log_size, n_lanes=1)
    w = rw.random_trees(m, 1000 + log_size, "full")
    sides = []
    for be in (CudaBackend(ctx), OracleBackend()):
        ch = be.channel()
        p = be.prover(m.words, rw.CONFIG)
        p.commit(w.tree0, ch, coset_order=True)
        p.commit(w.tree1, ch, coset_order=True)
        sides.append([p.gen_interaction(k, comp.log_size, max(comp.batching) + 1, w.params) for k, comp in enumerate(m.air.components)])
        del p
    for k, ((g_cols, g_sum), (o_cols, o_sum)) in enumerate(zip(*sides)):
        assert g_sum == o_sum, f"component {k}: claimed sum"
        _same(g_cols.download(), o_cols, f"component {k}: interaction trace")
    assert not M.verify_claimed_sums([s for _c, s in sides[0]])


# ---- 6. whole proofs of bench.py's machine -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("log_size,config", [
    (16, None),
    (16, dict(pow_bits=10, log_blowup=1, log_last=2, n_queries=40)),     # many merged decommitment paths, a last FRI layer of 4 points
    pytest.param(18, None, marks=pytest.mark.slow),
], ids=["2p16-default", "2p16-40-queries", "2p18-default"])
def test_proof_of_the_bench_machine(ctx, log_size, config):
    from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
    m = NexusV1Machine(log_size)
    cols = m.fill_main_trace(seed=log_size)
    g_proof, g_claimed, g_aux = M.prove(m, CudaBackend(ctx), cols, None, config=config, associated_data=b"bench")
    o_proof, o_claimed, o_aux = M.prove(m, OracleBackend(), cols, None, config=config, associated_data=b"bench")
    assert g_aux["roots"] == o_aux["roots"]
    assert g_claimed == o_claimed and M.verify_claimed_sums(g_claimed)
    assert g_proof == o_proof, f"proof bytes differ (len {len(g_proof)} vs {len(o_proof)})"
    verify(m, g_proof, o_aux)
