"""Table multiplicities counted on the GPU from the recorded AIR (nb200_table_multiplicities; run on an H100: `pytest -m gpu`).  The tree-1
multiplicity columns are filled with garbage first; after the count they must equal the machines' own host columns bit for bit (finalized
order), proofs from them must equal the host-column proofs and pass the oracle's verifier, unmatched lookups are counted and the first one is
named, and a table that lists one tuple twice is refused."""
import gc

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import keccak as K
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
from nexus_zkvm_b200.prover import Air, CudaBackend
from oracle import pyoracle as orc
from tests import table_mult_ref as ref
from tests.keccak_side_notes import edge_machine, finalized_main_trace
from tests.oracle_backend import verify_with_replayed_transcript
from tests.random_witness import mixed

pytestmark = pytest.mark.gpu
P = (1 << 31) - 1


@pytest.fixture(scope="module")
def backend():
    b = CudaBackend(nb.Context(0))
    yield b
    gc.collect()
    b.ctx.close()


def _batches(ctx, cols):
    """Trace-order host columns -> device batches of equal-length runs (finalized order), and column index -> (batch, index)."""
    out, where, i = [], [], 0
    while i < len(cols):
        j = i
        while j < len(cols) and len(cols[j]) == len(cols[i]):
            j += 1
        out.append(ctx.upload(np.stack([np.asarray(c, dtype=np.uint32) for c in cols[i:j]]), coset_order=True))
        where += [(len(out) - 1, k) for k in range(j - i)]
        i = j
    return out, where


def _table_cols(m):
    return sorted({col for row in ref.classify(m.air) for (kind, _r, col) in row if kind == "table"})


def _device(ctx, m, t1, seed=7):
    """(tree0, tree1, where1): tree 1 uploaded with every multiplicity column replaced by garbage."""
    t1 = [np.array(c, dtype=np.uint32) for c in ref.flat(t1)]
    rng = np.random.default_rng(seed)
    for c in _table_cols(m):
        t1[c] = rng.integers(0, P, len(t1[c]), dtype=np.uint32)
    tree0, _ = _batches(ctx, ref.flat(m.preprocessed_columns()))
    tree1, where1 = _batches(ctx, t1)
    return tree0, tree1, where1


def _columns(tree1, where1, cols):
    down = {}
    out = {}
    for c in cols:
        b, k = where1[c]
        if b not in down:
            down[b] = tree1[b].download()
        out[c] = down[b][k]
    return out


def _machine(kind):
    if kind == "add":
        m = M.AddMachine(log_size=16, n_lanes=2)
        cols, mult = m.fill_main_trace(seed=3, n_padding=5)
        return m, list(cols) + [mult]
    if kind == "multi":
        m = M.MultiMachine([4, 5, 8, 12, 16])
        return m, m.fill_main_trace(seed=4)
    m = NexusV1Machine(kind)
    return m, m.fill_main_trace(seed=kind)


@pytest.mark.parametrize("kind", ["add", "multi", 16, 20])
def test_device_columns_equal_the_host_columns(backend, kind):
    m, t1 = _machine(kind)
    tree0, tree1, where1 = _device(backend.ctx, m, t1)
    M.fill_table_multiplicities(m, backend.ctx, tree0, tree1)
    air = m._count_air[id(backend.ctx)]
    M.fill_table_multiplicities(m, backend.ctx, tree0, tree1)   # a second call reuses the loaded AIR (and its count kernels)
    assert m._count_air[id(backend.ctx)] is air
    host = ref.flat(t1)
    for c, got in _columns(tree1, where1, _table_cols(m)).items():
        assert np.array_equal(got, orc.finalize_column(host[c])), c


@pytest.mark.parametrize("kind", [("log", 6), ("log", 14), ("edge", 37)])
def test_keccak_columns_equal_numpy_and_the_fill_kernel(backend, kind):
    """From device_trees (the side-note fill), out[3] / out[4] overwritten with garbage: the count restores numpy's columns and the fill's."""
    m = K.KeccakMachine(kind[1], seed=kind[1]) if kind[0] == "log" else edge_machine(kind[1], seed=kind[1])
    ctx = backend.ctx
    tree0, tree1 = m.device_trees(ctx)
    fill = [tree1[3].download(), tree1[4].download()]
    rng = np.random.default_rng(1)
    for b in (3, 4):
        tree1[b].upload(rng.integers(0, P, (tree1[b].n_cols, 1 << tree1[b].log_size), dtype=np.uint32))
    M.fill_table_multiplicities(m, ctx, tree0, tree1)
    want = finalized_main_trace(m)
    for b, f in zip((3, 4), fill):
        got = tree1[b].download()
        assert np.array_equal(got, f) and np.array_equal(got, want[b]), b


def test_v1_proof_from_device_columns_equals_the_host_proof(backend):
    m, t1 = _machine(16)
    h_proof, h_claimed, h_aux = M.prove(m, backend, t1, None)
    tree0, tree1, _w = _device(backend.ctx, m, t1)
    M.fill_table_multiplicities(m, backend.ctx, tree0, tree1)
    d_proof, d_claimed, d_aux = M.prove(m, backend, None, None, resident=(tree0, tree1))
    assert d_aux["roots"] == h_aux["roots"] and d_claimed == h_claimed and d_proof == h_proof
    verify_with_replayed_transcript(m, d_proof, d_claimed, d_aux)


def test_keccak_proof_from_device_columns_equals_the_host_proof(backend):
    m = K.KeccakMachine(6, seed=6)
    h_proof, h_claimed, h_aux = M.prove(m, backend, m.fill_main_trace(), None)
    tree0, tree1 = m.device_trees(backend.ctx)
    for b in (3, 4):
        tree1[b].upload(np.zeros((tree1[b].n_cols, 1 << tree1[b].log_size), np.uint32))
    M.fill_table_multiplicities(m, backend.ctx, tree0, tree1)
    d_proof, d_claimed, d_aux = M.prove(m, backend, None, None, resident=(tree0, tree1))
    assert d_aux["roots"] == h_aux["roots"] and d_claimed == h_claimed and d_proof == h_proof
    verify_with_replayed_transcript(m, d_proof, d_claimed, d_aux)


def _range256_lookup(m, gated):
    """(fraction index, tree-1 column) of a Range256 lookup of the v1 main component with a constant (or, gated: a column) numerator."""
    comp = m.air.components[0]
    for i, (kind, rel, _x) in enumerate(ref.classify(m.air)[0]):
        if kind != "lookup" or rel.name != "Range256":
            continue
        if (comp.nodes[comp.lookups[i][1].id][0] == "const") != gated:
            (t, col, _o), = ref._leaves(comp, comp.lookups[i][2][0])
            return i, col
    raise AssertionError("no such lookup")


def test_one_unmatched_lookup_is_named_and_a_gated_one_is_not_counted(backend):
    m = NexusV1Machine(16)
    t1 = [np.array(c, dtype=np.uint32) for c in ref.flat(m.fill_main_trace(seed=16))]
    i, col = _range256_lookup(m, gated=False)
    row = 12345
    bad = [c.copy() for c in t1]
    bad[col][row] = 256
    tree0, tree1, _w = _device(backend.ctx, m, bad)
    n, first = backend.ctx.table_multiplicities(Air(backend.ctx, m.words), tree0, tree1)
    assert (n, first) == (1, (0, i, row))
    with pytest.raises(nb.Nb200Error, match=f"component 0, fraction {i}, trace row {row}"):
        M.fill_table_multiplicities(m, backend.ctx, tree0, tree1)
    # under a zero numerator (is_type_u = 0 on the padding witness) the same value is neither counted nor unmatched
    g, gcol = _range256_lookup(m, gated=True)
    gated = [c.copy() for c in t1]
    gated[gcol][row] = 256
    assert ref.multiplicities(m.air, m.preprocessed_columns(), gated)[1] == 0
    tree0, tree1, where1 = _device(backend.ctx, m, gated)
    assert backend.ctx.table_multiplicities(Air(backend.ctx, m.words), tree0, tree1) == (0, None)
    for c, got in _columns(tree1, where1, _table_cols(m)).items():
        assert np.array_equal(got, orc.finalize_column(t1[c])), c


def test_full_entropy_witness_unmatched_count_matches_the_reference(backend):
    m = NexusV1Machine(12)
    rng = np.random.default_rng(12)
    t1 = [mixed(rng, len(c)) for c in ref.flat(m.fill_main_trace(seed=12))]
    cols, n_want, first_want = ref.multiplicities(m.air, m.preprocessed_columns(), t1)
    assert n_want > 0
    tree0, tree1, where1 = _device(backend.ctx, m, t1)
    assert backend.ctx.table_multiplicities(Air(backend.ctx, m.words), tree0, tree1) == (n_want, first_want)
    for c, got in _columns(tree1, where1, list(cols)).items():
        assert np.array_equal(got, orc.finalize_column(cols[c])), c


def test_a_table_listing_one_value_twice_is_refused(backend):
    m, t1 = _machine("add")
    pre = [np.array(c, dtype=np.uint32) for c in ref.flat(m.preprocessed_columns())]
    k = m.air.preprocessed_ids["Range256Values"]
    pre[k][200] = pre[k][100]
    ctx = backend.ctx
    tree0, _ = _batches(ctx, pre)
    tree1, _w = _batches(ctx, ref.flat(t1))
    with pytest.raises(nb.Nb200Error, match="status 2: table_multiplicities: a table lists the same tuple in two rows of one relation"):
        ctx.table_multiplicities(Air(ctx, m.words), tree0, tree1)
