"""The first-row table count (nb200_table_multiplicities_first_row) on the GPU (run on an H100: `pytest -m gpu`):
  * the whole machine (whole_machine.py), whose Range8 table lists 0 nine times: every table column pre-filled with garbage and counted on
    the device equals the host fill, n_repeated is 8, and the proof from device_trees equals the oracle's proof bytes; at 2^20 main rows
    with 2^12 permutations the oracle's verifier accepts it;
  * a stress machine recorded here: a 2^16-row table listing each of 256 values on 256 rows (many threads race for one hash slot), a second
    table repeating some of them and a lookup component.  Each value's count lands on its first (component, trace row), every other row is
    0, three calls agree, and an unmatched lookup is reported as nb200_table_multiplicities reports it;
  * nb200_table_multiplicities itself still refuses both machines."""
import gc

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import air as A
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200 import whole_machine as W
from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
from nexus_zkvm_b200.prover import Air, CudaBackend
from oracle import pyoracle as orc
from tests import table_mult_ref as ref
from tests.keccak_side_notes import finalized_src_rows
from tests.oracle_backend import OracleBackend, verify_with_replayed_transcript
from tests.random_witness import mixed

pytestmark = pytest.mark.gpu
P = (1 << 31) - 1
REFUSAL = "status 2: table_multiplicities: a table lists the same tuple in two rows of one relation"


@pytest.fixture(scope="module")
def backend():
    b = CudaBackend(nb.Context(0))
    yield b
    gc.collect()
    b.ctx.close()


@pytest.fixture(scope="module")
def machines():
    return {"small": W.NexusV1KeccakMachine(8, 15, seed=1), "mid": W.NexusV1KeccakMachine(16, 1 << 6, seed=2)}


def _where(batches):
    """Flat column index -> (batch, index in batch)."""
    return [(b, k) for b, x in enumerate(batches) for k in range(x.n_cols)]


def _table_cols(m):
    return sorted({col for row in ref.classify(m.air) for (kind, _r, col) in row if kind == "table"})


def _garble(tree1, cols, seed):
    """Overwrite the given flat columns of tree 1 with random words."""
    where = _where(tree1)
    rng = np.random.default_rng(seed)
    for b in sorted({where[c][0] for c in cols}):
        x = tree1[b].download()
        for c in cols:
            if where[c][0] == b:
                x[where[c][1]] = rng.integers(0, 1 << 32, x.shape[1], dtype=np.uint64).astype(np.uint32)
        tree1[b].upload(x)


def _download(tree1, cols):
    where = _where(tree1)
    down = {b: tree1[b].download() for b in {where[c][0] for c in cols}}
    return {c: down[where[c][0]][where[c][1]] for c in cols}


@pytest.mark.parametrize("size", ["small", "mid"])
def test_whole_machine_counted_on_the_device(backend, machines, size):
    m = machines[size]
    ctx = backend.ctx
    tree0, tree1 = m.device_trees(ctx)
    cols = _table_cols(m)
    _garble(tree1, cols, 5)
    assert M.fill_table_multiplicities(m, ctx, tree0, tree1, first_row=True) == 8
    host = ref.flat(m.fill_main_trace())
    for c, got in _download(tree1, cols).items():
        assert np.array_equal(got, orc.finalize_column(host[c])), c
    d_proof, d_claimed, d_aux = M.prove(m, backend, None, None, resident=(tree0, tree1), associated_data=b"first row")
    o_proof, o_claimed, o_aux = M.prove(m, OracleBackend(), m.fill_main_trace(), None, associated_data=b"first row")
    assert d_aux["roots"] == o_aux["roots"] and d_claimed == o_claimed and d_proof == o_proof


def test_large_whole_machine_counted_on_the_device_is_accepted(backend):
    m = W.NexusV1KeccakMachine(20, 1 << 12)
    ctx = backend.ctx
    tree0, tree1 = m.device_trees(ctx)
    cols = _table_cols(m)
    host = ref.flat(m.fill_main_trace())
    for c, got in _download(tree1, cols).items():
        assert np.array_equal(got, orc.finalize_column(host[c])), c
    del host
    proof, claimed, aux = M.prove(m, backend, None, None, resident=(tree0, tree1))
    assert M.verify_claimed_sums(claimed)
    verify_with_replayed_transcript(m, proof, claimed, aux)


def test_plain_count_still_refuses_the_whole_machine(backend, machines):
    m = machines["small"]
    tree0, tree1 = m.device_trees(backend.ctx)
    with pytest.raises(nb.Nb200Error, match=REFUSAL):
        M.fill_table_multiplicities(m, backend.ctx, tree0, tree1)


# ---- the stress machine
LOG_A, LOG_B, LOG_C = 16, 8, 16
B_OWN = 64          # B's rows 128..191 list 256..319, which A does not; its rows 0..127 list A's even values, its rows 192..255 repeat its own


def stress_air():
    air = A.Air()
    rel = air.relation("Stress", 1)
    for log_size, name in ((LOG_A, "stress_values_a"), (LOG_B, "stress_values_b")):
        c = air.component(log_size)
        v = c.get_preprocessed_column(name)
        c.add_to_relation(rel, -c.next_trace_mask(), [v])
        c.finalize_logup()
    c = air.component(LOG_C)
    x, n = c.next_trace_mask(), c.next_trace_mask()
    c.add_to_relation(rel, n, [x])
    c.finalize_logup()
    return air


def stress_tables():
    """Trace-order values of tables A (each of 0..255 on 256 rows, scattered) and B."""
    r = np.arange(1 << LOG_A, dtype=np.uint64)
    a = (((r * 40503 + 12345) & 0xFFFF) >> 8).astype(np.uint32)
    rb = np.arange(1 << LOG_B, dtype=np.uint32)
    b = np.where(rb < 128, 2 * rb, 256 + rb % B_OWN).astype(np.uint32)
    return a, b


def stress_lookups(seed):
    rng = np.random.default_rng(seed)
    x = rng.integers(0, 256 + B_OWN, 1 << LOG_C).astype(np.uint32)
    n = rng.integers(0, 1 << 20, 1 << LOG_C).astype(np.uint32)
    n[rng.random(1 << LOG_C) < 0.1] = 0
    x[np.flatnonzero(n == 0)[::7]] = 5000                 # a tuple in no table under a zero numerator: neither counted nor unmatched
    x[:16], n[:16] = 7, P - 1                             # numerators near P: value 7's counter exceeds 2^32
    return x, n


def stress_expected(a, b, x, n):
    """Trace-order columns: each value's count on its first row (A before B), 0 elsewhere."""
    count = np.zeros(1 << 13, np.int64)
    np.add.at(count, x, n.astype(np.int64))
    ca, cb = np.zeros(len(a), np.int64), np.zeros(len(b), np.int64)
    seen = set()
    for col, vals in ((ca, a), (cb, b)):
        _u, first = np.unique(vals, return_index=True)
        for r in first:
            if int(vals[r]) not in seen:
                seen.add(int(vals[r]))
                col[r] = count[vals[r]]
    return (ca % P).astype(np.uint32), (cb % P).astype(np.uint32)


def stress_trees(ctx, a, b, x, n, garbage_seed):
    rng = np.random.default_rng(garbage_seed)
    tree0 = [ctx.upload(a, coset_order=True), ctx.upload(b, coset_order=True)]
    tree1 = [ctx.upload(rng.integers(0, P, 1 << LOG_A).astype(np.uint32)), ctx.upload(rng.integers(0, P, 1 << LOG_B).astype(np.uint32)),
             ctx.upload(np.stack([x, n]), coset_order=True)]
    return tree0, tree1


def test_stress_machine_credits_every_value_to_its_first_row(backend):
    ctx = backend.ctx
    air = stress_air()
    assert [[k for k, _r, _c in row] for row in ref.classify(air)] == [["table"], ["table"], ["lookup"]]
    a, b = stress_tables()
    # the race matters: for most values the row at the smallest finalized position is not the first trace row
    pos = np.argsort(finalized_src_rows(LOG_A))           # trace row -> finalized position
    first_row = {int(v): int(np.flatnonzero(a == v)[0]) for v in range(256)}
    first_pos = {int(v): int(np.flatnonzero(a == v)[np.argmin(pos[a == v])]) for v in range(256)}
    assert sum(first_row[v] != first_pos[v] for v in range(256)) > 200
    x, n = stress_lookups(1)
    want_a, want_b = stress_expected(a, b, x, n)
    assert want_a.any() and want_b.any()
    loaded = Air(ctx, air.serialize())
    runs = []
    for seed in range(3):
        tree0, tree1 = stress_trees(ctx, a, b, x, n, seed)
        got = ctx.table_multiplicities(loaded, tree0, tree1, first_row=True)
        assert got == (0, None, (1 << LOG_A) + (1 << LOG_B) - (256 + B_OWN))
        runs.append((tree1[0].download()[0], tree1[1].download()[0]))
    assert np.array_equal(runs[0][0], orc.finalize_column(want_a)) and np.array_equal(runs[0][1], orc.finalize_column(want_b))
    for r in runs[1:]:
        assert np.array_equal(r[0], runs[0][0]) and np.array_equal(r[1], runs[0][1])
    # one unmatched lookup: counted and named, the other values still counted
    x2, n2 = x.copy(), n.copy()
    x2[777], n2[777] = 4000, 5
    tree0, tree1 = stress_trees(ctx, a, b, x2, n2, 9)
    assert ctx.table_multiplicities(loaded, tree0, tree1, first_row=True)[:2] == (1, (2, 0, 777))
    n2[777] = 0
    want_a2, want_b2 = stress_expected(a, b, x2, n2)
    assert np.array_equal(tree1[0].download()[0], orc.finalize_column(want_a2))
    assert np.array_equal(tree1[1].download()[0], orc.finalize_column(want_b2))
    # the plain count refuses the machine
    with pytest.raises(nb.Nb200Error, match=REFUSAL):
        ctx.table_multiplicities(loaded, *stress_trees(ctx, a, b, x, n, 10))


def test_without_repeats_both_entries_agree(backend):
    """A full-entropy v1 witness (unmatched lookups, no repeated table tuple): same columns, same unmatched report, nothing repeated."""
    m = NexusV1Machine(12)
    ctx = backend.ctx
    rng = np.random.default_rng(12)
    t1 = [mixed(rng, len(c)) for c in ref.flat(m.fill_main_trace(seed=12))]
    loaded = Air(ctx, m.words)
    tree0 = [ctx.upload(np.stack(c), coset_order=True) for c in _runs(ref.flat(m.preprocessed_columns()))]
    out = []
    for first_row in (False, True):
        tree1 = [ctx.upload(np.stack(c), coset_order=True) for c in _runs(t1)]
        res = ctx.table_multiplicities(loaded, tree0, tree1, first_row=first_row)
        out.append((res, _download(tree1, _table_cols(m))))
    (plain, cols_plain), (first, cols_first) = out
    assert plain[0] > 0 and first == plain + (0,)
    for c in cols_plain:
        assert np.array_equal(cols_plain[c], cols_first[c]), c


def _runs(cols):
    out, i = [], 0
    while i < len(cols):
        j = i
        while j < len(cols) and len(cols[j]) == len(cols[i]):
            j += 1
        out.append(cols[i:j])
        i = j
    return out
