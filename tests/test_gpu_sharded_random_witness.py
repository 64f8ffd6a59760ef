"""The sharded prover's constraint quotients and interaction trace on the GPU against the oracle, on witnesses where every constraint matters
(tests/random_witness.py: `full`, `main_random`), bit-exact.

A proof over N GPUs (machine.prove_sharded) evaluates the main component with code of its own: the constraint quotients read D1 from the LDE row
slices and D2 from the half-coset extension the sharded commit computes (the fused mid kernel's two extra forward heads from 2^16 rows on, the
half-domain transform below), the masks at a row offset from the full copies of the replicated columns, and the interaction trace runs on the
kept trace rows.  The proof-byte tests pin that route only on AddMachine and on the v1 padding witness, which makes 42 of the 45 constraints of
the v1 D2 kernel identically zero.  Here the trees are committed on a one-rank communicator exactly as prove_sharded commits them, and
nb200_constraint_quotients_half, which takes the sharded route for such a component, is compared with the oracle on the same trees.

Not covered on one GPU: rows with row0() != 0, the peer-heap row scatter and the all-gathers of more than one rank (tests/test_gpu_multi.py)."""
import functools
import gc

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.prover import CudaBackend
from tests import random_witness as rw
from tests.oracle_backend import OracleBackend
from tests.test_gpu_backend_ops import component_headers
from tests.test_gpu_v1_random_witness import check_full_route, check_half_route, machine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = nb.Context(0)
    c.comm_init(0, 1, nb.Context.comm_unique_id())
    yield c
    gc.collect()
    c.close()


def log_sizes(m):
    return list(getattr(m, "log_sizes", None) or [m.log_size, 8])


def shard_trees(m, prover, w):
    """Trees 0 and 1 of the witness as shard_host_tree uploads them on rank 0 of 1."""
    return [M.shard_host_tree(m, prover, cols, 0, 1) for cols in (w.tree0, w.tree1)]


def commit_sharded(ctx, m, w):
    """The witness committed as prove_sharded commits it: (GPU prover, params, roots).  `full`: trees 0 to 2 from the witness, each through
    commit_sharded_tree; `main_random`: the whole sequence of prove_sharded up to tree 2, with the witness's trees 0 and 1."""
    be = CudaBackend(ctx)
    if w.tree2 is None:
        _ch, gpu, params, _claimed, roots = M._commit_trees_sharded(m, be, None, None, 0, 1, rw.CONFIG, b"", shard_trees(m, be.prover(m.words, rw.CONFIG), w))
        return gpu, params, roots
    ch, gpu = be.channel(), be.prover(m.words, rw.CONFIG)
    parts = shard_trees(m, gpu, w) + [M.shard_host_tree(m, gpu, w.tree2, 0, 1, coset_order=False)]
    roots = [M.commit_sharded_tree(m, gpu, t, parts[t], t < 2, ch) for t in range(3)]
    return gpu, list(w.params), roots


def replicated_components(m, w):
    """The components that read no sharded column: none of the leading 2^log_size-row columns of trees 0 and 1, none of the main component's
    interaction columns."""
    lead = lambda cols: next((i for i, c in enumerate(cols) if len(c) != 1 << m.log_size), len(cols))
    big = [lead(w.tree0), lead(w.tree1), 4 * (max(m.air.components[0].batching) + 1)]
    return [k for k, comp in enumerate(m.air.components) if not any(c < big[t] for (t, c, _o) in comp.masks)]


def compare(ctx, m, kind, seed):
    w = rw.random_trees(m, seed, kind)
    gpu, params, roots = commit_sharded(ctx, m, w)
    orc_p, o_params = rw.commit(OracleBackend(), m, w, log_sizes(m) if w.tree2 is None else ())
    assert roots == orc_p.roots
    assert params == o_params
    assert check_half_route(ctx, m, gpu, orc_p, params, seed + 1) == 1
    others = replicated_components(m, w)
    assert others == list(range(1, len(m.air.components)))
    check_full_route(ctx, m, gpu, orc_p, params, seed + 2, components=others)


@pytest.mark.parametrize("kind", ["full", "main_random"])
def test_v1_sharded_quotients(ctx, kind):
    """2^12 rows: the sharded commit's D2 comes from the half-domain transform (the fused pipeline starts at 2^16)."""
    compare(ctx, machine("nexus_v1", 12), kind, 600)


def test_add_machine_sharded_quotients(ctx):
    """AddMachine (log_expand 2, three lanes) at 2^12 rows."""
    compare(ctx, machine("add", 12), "full", 610)


@pytest.mark.slow
def test_v1_sharded_quotients_at_2p16(ctx):
    """2^16 rows: the fused pipeline computes D2 with the mid kernel's two forward heads.  The 347 main columns end on a partly filled group of
    the A/C kernels (four columns per CTA: 3 of 4) and of the mid kernel's D2 heads (two per CTA: 1 of 2); tree 2's interaction columns go
    through the same heads."""
    compare(ctx, machine("nexus_v1", 16), "full", 620)


@pytest.mark.parametrize("name", ["nexus_v1", "add"])
def test_sharded_interaction_trace(ctx, name):
    """nb200_gen_interaction_trace_sharded (at world 1 the shard is every column) for the main component and nb200_gen_interaction_trace on the
    replicated batches for the others, on random trees 0 and 1 with random parameters: every column and claimed sum equal the oracle's."""
    m = machine(name, 12)
    w = rw.random_trees(m, 630, "full")
    be = CudaBackend(ctx)
    ch, gpu = be.channel(), be.prover(m.words, rw.CONFIG)
    parts = shard_trees(m, gpu, w)
    for t in (0, 1):
        M.commit_sharded_tree(m, gpu, t, parts[t], True, ch)
    shard2, small, claimed = M.interaction_traces_sharded(m, gpu, parts, list(w.params))
    orc_p = OracleBackend().prover(m.words, rw.CONFIG)
    och = OracleBackend().channel()
    orc_p.commit(w.tree0, och, coset_order=True)
    orc_p.commit(w.tree1, och, coset_order=True)
    assert len(small) == len(m.air.components) - 1
    for k, comp in enumerate(m.air.components):
        o_cols, o_sum = orc_p.gen_interaction(k, comp.log_size, max(comp.batching) + 1, w.params)
        assert claimed[k] == o_sum, f"component {k}: claimed sum"
        assert np.array_equal((shard2 if k == 0 else small[k - 1]).download(), o_cols), f"component {k}: interaction trace"


# ---- refusals: each leaves the context usable ------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def _oracle_proof():
    m = M.AddMachine(log_size=10, n_lanes=1)
    cols, mult = m.fill_main_trace(seed=10, n_padding=3)
    return M.prove(m, OracleBackend(), cols, mult)[0]


def assert_usable(ctx):
    """A sharded proof on the context afterwards has the oracle's bytes."""
    m = M.AddMachine(log_size=10, n_lanes=1)
    cols, mult = m.fill_main_trace(seed=10, n_padding=3)
    assert M.prove_sharded(m, CudaBackend(ctx), cols, mult, 0, 1)[0] == _oracle_proof()


def _half_accumulators(ctx, m):
    lg, _e, _n = component_headers(m.words)[0]
    return [ctx.upload(np.zeros((4, 1 << (lg + rw.CONFIG["log_blowup"])), np.uint32)) for _ in range(3)]


def test_full_domain_entry_refuses_the_sharded_component(ctx):
    m = machine("add", 12)
    w = rw.random_trees(m, 640, "full")
    gpu, params, _roots = commit_sharded(ctx, m, w)
    lg, expand, n = component_headers(m.words)[0]
    acc = ctx.upload(np.zeros((4, 1 << (lg + expand)), np.uint32))
    with pytest.raises(nb.Nb200Error, match=r"nb200 status 2: .*reads sharded columns"):
        gpu.constraint_quotients(0, params, np.zeros((n, 4), np.uint32), acc)
    assert not acc.download().any()
    orc_p, _p = rw.commit(OracleBackend(), m, w)
    assert check_half_route(ctx, m, gpu, orc_p, params, 641) == 1      # the half-domain entry still works on the same scheme
    assert_usable(ctx)


def test_half_entry_names_an_offset_column_that_was_not_replicated(ctx):
    m = machine("add", 12)
    w = rw.random_trees(m, 650, "full")
    be = CudaBackend(ctx)
    ch, gpu = be.channel(), be.prover(m.words, rw.CONFIG)
    parts = shard_trees(m, gpu, w) + [M.shard_host_tree(m, gpu, w.tree2, 0, 1, coset_order=False)]
    M.commit_sharded_tree(m, gpu, 0, parts[0], True, ch)
    shard, total, small = parts[1]
    gpu.commit_sharded(shard, total, m.log_size, small, [], True, ch)            # tree 1 without its replicated columns
    M.commit_sharded_tree(m, gpu, 2, parts[2], False, ch)
    t, c = next((t, c) for (t, c, off) in m.air.components[0].masks if t == 1 and off != 0)
    _lg, _e, n = component_headers(m.words)[0]
    with pytest.raises(nb.Nb200Error, match=rf"nb200 status 2: .*column {c} of tree {t} is read at a row offset but was not listed for replication"):
        gpu.constraint_quotients_half(0, w.params, np.zeros((n, 4), np.uint32), *_half_accumulators(ctx, m))
    assert_usable(ctx)


def test_sharded_route_needs_the_generated_kernels(ctx, monkeypatch):
    """The kernel cache lives in the loaded AIR: with NB200_JIT=0 a freshly loaded one has none, and the sharded route has no interpreter."""
    m = machine("add", 12)
    w = rw.random_trees(m, 660, "full")
    monkeypatch.setenv("NB200_JIT", "0")
    gpu, params, _roots = commit_sharded(ctx, m, w)
    _lg, _e, n = component_headers(m.words)[0]
    with pytest.raises(nb.Nb200Error, match=r"nb200 status 2: sharded constraint quotients need the specialised kernel"):
        gpu.constraint_quotients_half(0, params, np.zeros((n, 4), np.uint32), *_half_accumulators(ctx, m))
    monkeypatch.delenv("NB200_JIT")
    assert_usable(ctx)


def test_prove_sharded_refuses_a_blowup_without_d2(ctx):
    """With log_blowup 2 the main component's quotients are evaluated on the LDE domain itself (Q_FULL), the sharded commit computes no D2,
    and the sharded route, which only exists in the half-domain form, refuses at the composition step."""
    m = M.AddMachine(log_size=10, n_lanes=1)
    cols, mult = m.fill_main_trace(seed=11, n_padding=3)
    with pytest.raises(nb.Nb200Error, match=r"nb200 status 2: sharded constraint quotients: the component must use the half-domain route"):
        M.prove_sharded(m, CudaBackend(ctx), cols, mult, 0, 1, config=dict(rw.CONFIG, log_blowup=2))
    assert_usable(ctx)
