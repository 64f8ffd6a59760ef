"""The ADD chain's kernels on the GPU against the oracle, on witnesses where every constraint matters (tests/random_witness.py: `full`,
`main_random`, `sparse`), bit-exact; run on an H100 with `pytest -m gpu`.

Its main component (add_chain.AddChainMachine: the v1 main component with DecodingCheck types R and I, 486 constraints, 110 of degree > 2)
has generated kernels of its own, and the executing trace makes 181 of its constraints and 80 of those the D2 kernel evaluates identically
zero.  Here, on random trees: the full-domain quotients of all nine components; the half-domain quotients (q on D1, the high constraints' q on
D2 and on D1) from the generated kernels and from the bytecode interpreter (NB200_JIT=0, and at 2^8 rows, where the LDE is smaller than the
generated kernels' CTA); the interaction trace; the check report; and the sharded route on a one-rank communicator, whose D2 comes from the
half-domain transform at 2^12 rows and from the fused mid kernel's heads at 2^16.  On valid ADD / ADDI programs other than the chain: the
device-counted table multiplicities (Range16 and Range8 counted on DecodingCheck's type-I pieces of immediates of every bit pattern) and the
proofs from device trees.  And the device fill on step records at the edges of u32 (tests/test_add_chain_random_witness_cpu.py)."""
import gc

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import add_chain as AC
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.prover import CudaBackend
from tests import random_witness as rw
from tests.keccak_side_notes import finalized_src_rows
from tests.oracle_backend import OracleBackend, verify
from tests.test_add_chain_cpu import OFFSETS, mixed_program
from tests.test_add_chain_random_witness_cpu import EDGE_IDS, EDGE_SHAPES, edge_steps, edge_want
from tests.test_gpu_sharded_random_witness import commit_sharded, compare, shard_trees
from tests.test_gpu_v1_random_witness import check_full_route, check_half_route, check_report, committed

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    """One context for every test; its one-rank communicator is only used by the sharded commits."""
    c = nb.Context(0)
    c.comm_init(0, 1, nb.Context.comm_unique_id())
    yield c
    gc.collect()
    c.close()


@pytest.mark.parametrize("log_size", [10, 12])
@pytest.mark.parametrize("kind", ["full", "main_random"])
def test_quotients(ctx, kind, log_size):
    m = AC.AddChainMachine(log_size)
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 700 + log_size, kind))
    check_full_route(ctx, m, gpu, orc_p, params, 1)
    assert check_half_route(ctx, m, gpu, orc_p, params, 2) == 1


@pytest.mark.parametrize("log_size,jit", [(8, "0"), (12, "0"), (8, None)], ids=["2^8-NB200_JIT=0", "2^12-NB200_JIT=0", "2^8"])
def test_half_route_with_the_interpreter(ctx, monkeypatch, log_size, jit):
    """The half route through the bytecode interpreter: with NB200_JIT=0, and at 2^8 rows with the generated kernels on (the LDE is
    smaller than their CTA, so the interpreter evaluates there too)."""
    if jit is not None:
        monkeypatch.setenv("NB200_JIT", jit)
    m = AC.AddChainMachine(log_size)
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 710 + log_size, "full"))
    assert check_half_route(ctx, m, gpu, orc_p, params, 3, jit=jit is None) == 1


@pytest.mark.parametrize("log_size", [8, 12])
def test_interaction_trace(ctx, log_size):
    """nb200_gen_interaction_trace of all nine components on random trees 0 and 1 with random lookup elements: every column and claimed
    sum equal the oracle's (the sums do not cancel)."""
    m = AC.AddChainMachine(log_size)
    w = rw.random_trees(m, 720 + log_size, "full")
    sides = []
    for be in (CudaBackend(ctx), OracleBackend()):
        ch = be.channel()
        p = be.prover(m.words, rw.CONFIG)
        p.commit(w.tree0, ch, coset_order=True)
        p.commit(w.tree1, ch, coset_order=True)
        sides.append([p.gen_interaction(k, comp.log_size, max(comp.batching) + 1, w.params) for k, comp in enumerate(m.air.components)])
    assert len(sides[0]) == 9
    for k, ((g_cols, g_sum), (o_cols, o_sum)) in enumerate(zip(*sides)):
        assert g_sum == o_sum, k
        assert np.array_equal(g_cols.download(), o_cols), k
    assert not M.verify_claimed_sums([s for _c, s in sides[0]])


@pytest.mark.parametrize("kind", ["sparse", "full"])
def test_check(ctx, kind):
    m = AC.AddChainMachine(10)
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 730, kind))
    check_report(m, gpu, orc_p, params)


# ---- the sharded route on a one-rank communicator (at least 2^9 rows: at 2^8 the 2^8-row tables are as large as the main component)

@pytest.mark.parametrize("kind", ["full", "main_random"])
def test_sharded_quotients(ctx, kind):
    """2^12 rows: the sharded commit's D2 comes from the half-domain transform."""
    compare(ctx, AC.AddChainMachine(12), kind, 740)


def test_sharded_interaction_trace(ctx):
    """nb200_gen_interaction_trace_sharded for the main component and nb200_gen_interaction_trace on the replicated batches for the others,
    on random trees 0 and 1 with random parameters: every column and claimed sum equal the oracle's."""
    m = AC.AddChainMachine(12)
    w = rw.random_trees(m, 750, "full")
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
    assert len(small) == len(m.air.components) - 1 == 8
    for k, comp in enumerate(m.air.components):
        o_cols, o_sum = orc_p.gen_interaction(k, comp.log_size, max(comp.batching) + 1, w.params)
        assert claimed[k] == o_sum, f"component {k}: claimed sum"
        assert np.array_equal((shard2 if k == 0 else small[k - 1]).download(), o_cols), f"component {k}: interaction trace"


def test_sharded_commit_refuses_the_2p8_chain(ctx):
    """At 2^8 rows BitOpMultiplicity and Multiplicity256 are as large as the main component: they are not the leading batch alone."""
    m = AC.AddChainMachine(8)
    with pytest.raises(AssertionError, match="leading, largest batch"):
        commit_sharded(ctx, m, rw.random_trees(m, 755, "full"))


def test_prove_sharded_equals_prove_and_the_oracle(ctx):
    m = AC.AddChainMachine(12)
    t1 = m.fill_main_trace()
    s_proof, s_claimed, _aux = M.prove_sharded(m, CudaBackend(ctx), t1, None, 0, 1, associated_data=b"add chain")
    p_proof, p_claimed, _aux = M.prove(m, CudaBackend(ctx), t1, None, associated_data=b"add chain")
    o_proof, o_claimed, o_aux = M.prove(m, OracleBackend(), t1, None, associated_data=b"add chain")
    assert s_claimed == p_claimed == o_claimed and M.verify_claimed_sums(o_claimed)
    assert s_proof == p_proof == o_proof
    verify(m, s_proof, o_aux)


# ---- valid ADD / ADDI programs other than the chain: device counts and proofs

def random_program(n, seed):
    """n ADD / ADDI instructions over every register, immediates drawn from all 12-bit patterns."""
    rng = np.random.default_rng(seed)
    op, rd, rs1 = rng.integers(0, 2, n), rng.integers(0, 32, n), rng.integers(0, 32, n)
    rs2, imm = rng.integers(0, 32, n), rng.integers(-2048, 2048, n)
    return [(AC.OP_ADD, int(rd[t]), int(rs1[t]), int(rs2[t])) if op[t] == AC.OP_ADD else (AC.OP_ADDI, int(rd[t]), int(rs1[t]), int(imm[t]))
            for t in range(n)]


PROGRAMS = {"mixed-2^9": lambda: AC.AddChainMachine(9, ops=mixed_program()),
            "40000-in-2^16": lambda: AC.AddChainMachine(16, ops=random_program(40000, 760))}


@pytest.fixture(scope="module", params=list(PROGRAMS))
def program(request):
    return PROGRAMS[request.param]()


def test_device_counts_equal_host_counts_on_other_programs(ctx, program):
    """Every table column counted on the device from the filled trace (nb200_table_multiplicities_first_row) equals the host count; the
    type-I pieces OpC4_7 (Range16) and OpC8_10 (Range8) take every value they can."""
    m = program
    t1 = m.fill_main_trace()
    addi = np.asarray(t1[OFFSETS["ImmC"]]) == 1
    assert len(np.unique(np.asarray(t1[OFFSETS["OpC4_7"]])[addi])) == 16 and len(np.unique(np.asarray(t1[OFFSETS["OpC8_10"]])[addi])) == 8
    _tree0, tree1 = m.device_trees(ctx)
    host = t1[347:]
    dev = [c for b in tree1[1:] for c in b.download()]
    assert len(dev) == len(host)
    for k, (d, h) in enumerate(zip(dev, host)):
        log = int(len(h)).bit_length() - 1
        assert np.array_equal(d, np.asarray(h, np.uint32)[finalized_src_rows(log)]), k


def test_proofs_on_other_programs(ctx, program):
    m = program
    t1 = m.fill_main_trace()
    be = CudaBackend(ctx)
    h_proof, h_claimed, h_aux = M.prove(m, be, t1, None, associated_data=b"add / addi")
    d_proof, d_claimed, d_aux = M.prove(m, be, None, None, associated_data=b"add / addi", resident=m.device_trees(ctx))
    o_proof, o_claimed, o_aux = M.prove(m, OracleBackend(), t1, None, associated_data=b"add / addi")
    assert h_aux["roots"] == d_aux["roots"] == o_aux["roots"]
    assert h_claimed == d_claimed == o_claimed and M.verify_claimed_sums(h_claimed)
    assert h_proof == d_proof == o_proof
    verify(m, d_proof, o_aux)


# ---- the device fill on edge step records

@pytest.mark.parametrize("ls,n_steps,n_prog", EDGE_SHAPES, ids=EDGE_IDS)
def test_device_fill_on_edge_step_records(ctx, ls, n_steps, n_prog):
    steps, final_ctr = edge_steps(ls, n_steps, n_prog, seed=ls * 1000 + n_steps + 1)
    out = ctx.upload(np.random.default_rng(ls).integers(0, 1 << 32, (347, 1 << ls), dtype=np.uint64).astype(np.uint32))
    assert ctx.v1_main_trace(steps, final_ctr, ls, out=out) is out
    bad = np.argwhere(out.download() != edge_want(steps, final_ctr, ls))
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"


# ---- 2^16 rows: many CTAs and waves in every kernel

@pytest.mark.slow
def test_at_2p16(ctx):
    m = AC.AddChainMachine(16)
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 16, "full"))
    check_full_route(ctx, m, gpu, orc_p, params, 6)
    assert check_half_route(ctx, m, gpu, orc_p, params, 7) == 1
    check_report(m, gpu, orc_p, params)


@pytest.mark.slow
def test_sharded_quotients_at_2p16(ctx):
    """The fused pipeline computes D2 with the mid kernel's two forward heads; the add chain's D2 kernel reads 96 tree-1 columns (v1's 87),
    so its column groups end elsewhere than v1's."""
    compare(ctx, AC.AddChainMachine(16), "full", 770)
