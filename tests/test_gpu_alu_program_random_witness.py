"""The ALU program's kernels on the GPU against the oracle, on witnesses where every constraint matters (tests/random_witness.py: `full`,
`main_random`, `sparse`), bit-exact; run on an H100 with `pytest -m gpu`.

Its main component (add_chain.AluMachine: the ADD chain's DecodingCheck types R and I plus SltuChip, SltChip, SllChip, SrlChip and SraChip,
545 constraints, 144 of degree > 2) has generated D1, D2, LogUp, check and count kernels of its own, and its D2 kernel reads 127 tree-1
columns (the ADD chain's: 96, v1's: 87), so the D2 gather and the sharded commit's half-domain extension end their column groups elsewhere.
The executing trace makes 121 of its constraints identically zero, 38 of the D2 kernel's among them
(tests/test_alu_program_random_witness_cpu.py), so the proof comparisons of test_gpu_alu_program.py cannot see a wrong operand there.  Here, on random trees: the full-domain
quotients of all nine components and the half-domain quotients (q on D1, the high constraints' q on D2 and on D1) from the generated kernels
(the module's context traces every kernel it compiles, and the quotient tests fail when one fell back to the interpreter) and from the
bytecode interpreter (NB200_JIT=0, and at 2^8 rows, where the LDE is smaller than the generated kernels' CTA); the interaction trace; the
check report; and the sharded route on a one-rank communicator, whose D2 comes from the half-domain transform at 2^12 rows and from the
fused mid kernel's heads at 2^16.  On valid ALU programs other than the default (bit ops, or shifts and comparisons, on registers that ADDI,
SLLI and ADD keep at full entropy, and 40000 mixed steps in 2^16 rows): the device-counted table multiplicities and the proofs from device trees.  On a `sparse` witness: the count's
unmatched lookups against tests/table_mult_ref.py.  And the device fill on edge step records whose timestamps pass 2^16."""
import gc
import os

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import add_chain as AC
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200 import whole_machine as W
from nexus_zkvm_b200.prover import Air, CudaBackend
from tests import random_witness as rw
from tests import table_mult_ref as tref
from tests.keccak_side_notes import finalized_src_rows
from tests.oracle_backend import OracleBackend, verify
from tests.test_alu_program_cpu import _want, alu_edge_steps
from tests.test_gpu_sharded_random_witness import commit_sharded, compare, shard_trees
from tests.test_gpu_table_multiplicities import _batches
from tests.test_gpu_v1_random_witness import JIT_MIN_LOG_ROWS, check_full_route, check_half_route, check_report, committed
from tests.test_gpu_whole_machine_random_witness import no_fallback

pytestmark = pytest.mark.gpu
N_MAIN = 347
# tree 1 after the main columns: FinalReg's 8 columns, BitOpMultiplicity's And, Or, Xor, RamInitFinal's columns, then Multiplicity8 ... 256
BIT_OP = slice(N_MAIN + 8, N_MAIN + 11)
TABLES = {r: N_MAIN + 11 + W.RAM_COLS + k for k, (r, _len, _ls) in enumerate(W.MULTIPLICITY_TABLES)}


@pytest.fixture(scope="module")
def ctx():
    """One context for every test, with NB200_TRACE on (a generated kernel that cannot be compiled or loaded leaves its program to the
    interpreter with no more than a line on stderr, which no_fallback looks for); its one-rank communicator is only used by the sharded
    commits."""
    old = os.environ.get("NB200_TRACE")
    os.environ["NB200_TRACE"] = "1"
    try:
        c = nb.Context(0)
    finally:
        if old is None:
            del os.environ["NB200_TRACE"]
        else:
            os.environ["NB200_TRACE"] = old
    c.comm_init(0, 1, nb.Context.comm_unique_id())
    yield c
    gc.collect()
    c.close()


@pytest.fixture(scope="module")
def alu():
    """AluMachine(log_size) with the default program, built once per size for the module."""
    cache = {}

    def get(log_size):
        if log_size not in cache:
            cache[log_size] = AC.AluMachine(log_size)
        return cache[log_size]
    yield get
    cache.clear()


@pytest.mark.parametrize("log_size", [10, 12])
@pytest.mark.parametrize("kind", ["full", "main_random"])
def test_quotients(ctx, alu, capfd, kind, log_size):
    m = alu(log_size)
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 800 + log_size, kind))
    check_full_route(ctx, m, gpu, orc_p, params, 1)
    assert check_half_route(ctx, m, gpu, orc_p, params, 2) == 1
    no_fallback(capfd)


@pytest.mark.parametrize("log_size,jit", [(8, "0"), (12, "0"), (8, None)], ids=["2^8-NB200_JIT=0", "2^12-NB200_JIT=0", "2^8"])
def test_half_route_with_the_interpreter(ctx, alu, monkeypatch, log_size, jit):
    """The half route through the bytecode interpreter: with NB200_JIT=0, and at 2^8 rows with the generated kernels on (the LDE is
    smaller than their CTA, so the interpreter evaluates there too)."""
    if jit is not None:
        monkeypatch.setenv("NB200_JIT", jit)
    m = alu(log_size)
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 810 + log_size, "full"))
    assert check_half_route(ctx, m, gpu, orc_p, params, 3, jit=jit is None) == 1


@pytest.mark.parametrize("log_size", [8, 12])
def test_interaction_trace(ctx, alu, capfd, log_size):
    """nb200_gen_interaction_trace of all nine components on random trees 0 and 1 with random lookup elements: every column and claimed
    sum equal the oracle's (the sums do not cancel)."""
    m = alu(log_size)
    w = rw.random_trees(m, 820 + log_size, "full")
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
    if log_size >= JIT_MIN_LOG_ROWS:
        no_fallback(capfd)


@pytest.mark.parametrize("kind", ["sparse", "full"])
def test_check(ctx, alu, kind):
    m = alu(10)
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 830, kind))
    check_report(m, gpu, orc_p, params)


# ---- the sharded route on a one-rank communicator (at least 2^9 rows: at 2^8 the 2^8-row tables are as large as the main component)

@pytest.mark.parametrize("kind", ["full", "main_random"])
def test_sharded_quotients(ctx, alu, kind):
    """2^12 rows: the sharded commit's D2 comes from the half-domain transform."""
    compare(ctx, alu(12), kind, 840)


def test_sharded_interaction_trace(ctx, alu):
    """nb200_gen_interaction_trace_sharded for the main component and nb200_gen_interaction_trace on the replicated batches for the others,
    on random trees 0 and 1 with random parameters: every column and claimed sum equal the oracle's."""
    m = alu(12)
    w = rw.random_trees(m, 850, "full")
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


def test_sharded_commit_refuses_the_2p8_program(ctx, alu):
    """At 2^8 rows BitOpMultiplicity and Multiplicity256 are as large as the main component: they are not the leading batch alone."""
    m = alu(8)
    with pytest.raises(AssertionError, match="leading, largest batch"):
        commit_sharded(ctx, m, rw.random_trees(m, 855, "full"))


def test_prove_sharded_equals_prove_and_the_oracle(ctx, alu):
    m = alu(12)
    t1 = m.fill_main_trace()
    s_proof, s_claimed, _aux = M.prove_sharded(m, CudaBackend(ctx), t1, None, 0, 1, associated_data=b"alu program")
    p_proof, p_claimed, _aux = M.prove(m, CudaBackend(ctx), t1, None, associated_data=b"alu program")
    o_proof, o_claimed, o_aux = M.prove(m, OracleBackend(), t1, None, associated_data=b"alu program")
    assert s_claimed == p_claimed == o_claimed and M.verify_claimed_sums(o_claimed)
    assert s_proof == p_proof == o_proof
    verify(m, s_proof, o_aux)


# ---- valid ALU programs other than the default: device counts and proofs

BIT_OPS = [AC.OP_AND, AC.OP_OR, AC.OP_XOR, AC.OP_ANDI, AC.OP_ORI, AC.OP_XORI]
SHIFTS_AND_COMPARES = [AC.OP_SLL, AC.OP_SRL, AC.OP_SRA, AC.OP_SLLI, AC.OP_SRLI, AC.OP_SRAI, AC.OP_SLT, AC.OP_SLTU, AC.OP_SLTI, AC.OP_SLTIU]


def random_program(n, seed, opcodes):
    """n instructions: x8..x31 loaded with full 32-bit values (ADDI, SLLI by 11, ADDI, SLLI by 11, ADDI), then instructions drawn uniformly
    from `opcodes` that read x8..x31 and write x0..x7, with random immediates and shift amounts, every fourth one an ADD of two of x8..x31
    into a third.  The operands keep full entropy, where results such as SLT's 0 / 1 written back would drain them."""
    rng = np.random.default_rng(seed)
    imm = lambda: int(rng.integers(-2048, 2048))
    src = lambda: int(rng.integers(8, 32))
    ops = [op for r in range(8, 32) for op in ((AC.OP_ADDI, r, 0, imm()), (AC.OP_SLLI, r, r, 11), (AC.OP_ADDI, r, r, imm()),
                                                (AC.OP_SLLI, r, r, 11), (AC.OP_ADDI, r, r, imm()))]
    while len(ops) < n:
        if len(ops) % 4 == 0:
            ops.append((AC.OP_ADD, src(), src(), src()))
            continue
        op = int(rng.choice(opcodes))
        c = {"R": src(), "I": imm()}.get(AC.OP_TYPE[op], int(rng.integers(0, 32)))
        ops.append((op, int(rng.integers(0, 8)), src(), c))
    return ops[:n]


PROGRAMS = {"bit-ops-2^12": lambda: AC.AluMachine(12, ops=random_program(4096, 900, BIT_OPS)),
            "shifts-and-compares-2^12": lambda: AC.AluMachine(12, ops=random_program(4096, 901, SHIFTS_AND_COMPARES)),
            "40000-in-2^16": lambda: AC.AluMachine(16, 40000, seed=902)}


@pytest.fixture(scope="module", params=list(PROGRAMS))
def program(request):
    return request.param, PROGRAMS[request.param]()


def test_device_counts_equal_host_counts_on_other_programs(ctx, program):
    """Every table column counted on the device from the filled trace (nb200_table_multiplicities_first_row) equals the host count.  The
    bit-op program credits every one of BitOpMultiplicity's 3 x 256 bins (many threads add to each of the count's privatised bins); the
    shift and comparison program counts SltChip's and SraChip's Range128 lookups and the shifts' Helper1 in Range8 over most values."""
    name, m = program
    t1 = m.fill_main_trace()
    ops = set(int(o) for o in m.steps[AC.STEP_FIELDS.index("opcode")])
    if name.startswith("bit-ops"):
        assert ops == set(BIT_OPS) | {AC.OP_ADDI, AC.OP_SLLI, AC.OP_ADD}
        assert all(np.all(c != 0) for c in t1[BIT_OP])
    elif name.startswith("shifts"):
        assert ops == set(SHIFTS_AND_COMPARES) | {AC.OP_ADDI, AC.OP_ADD}
        assert not any(np.any(c) for c in t1[BIT_OP])
        assert np.count_nonzero(t1[TABLES["Range128"]]) >= 120 and np.all(t1[TABLES["Range8"]][:8] != 0)
    _tree0, tree1 = m.device_trees(ctx)
    host = t1[N_MAIN:]
    dev = [c for b in tree1[1:] for c in b.download()]
    assert len(dev) == len(host)
    for k, (d, h) in enumerate(zip(dev, host)):
        log = int(len(h)).bit_length() - 1
        assert np.array_equal(d, np.asarray(h, np.uint32)[finalized_src_rows(log)]), k


def test_proofs_on_other_programs(ctx, program):
    _name, m = program
    t1 = m.fill_main_trace()
    be = CudaBackend(ctx)
    h_proof, h_claimed, h_aux = M.prove(m, be, t1, None, associated_data=b"alu program")
    d_proof, d_claimed, d_aux = M.prove(m, be, None, None, associated_data=b"alu program", resident=m.device_trees(ctx))
    o_proof, o_claimed, o_aux = M.prove(m, OracleBackend(), t1, None, associated_data=b"alu program")
    assert h_aux["roots"] == d_aux["roots"] == o_aux["roots"]
    assert h_claimed == d_claimed == o_claimed and M.verify_claimed_sums(h_claimed)
    assert h_proof == d_proof == o_proof
    verify(m, d_proof, o_aux)


# ---- unmatched lookups

def test_unmatched_lookups_match_the_reference(ctx, alu):
    """The first-row count on a `sparse` witness (about 1 % of every tree-1 column replaced), as device_trees runs it: its unmatched count
    and first unmatched (component, fraction, trace row) equal tests/table_mult_ref.py's.  Only these two are compared: the reference
    credits a tuple that a table lists in several rows to every one of them."""
    m = alu(10)
    w = rw.random_trees(m, 860, "sparse")
    _cols, n_want, first_want = tref.multiplicities(m.air, m.preprocessed_columns(), w.tree1)
    assert n_want > 0
    tree0, _ = _batches(ctx, w.tree0)
    tree1, _ = _batches(ctx, w.tree1)
    n, first, _repeated = ctx.table_multiplicities(Air(ctx, m.words), tree0, tree1, first_row=True)
    assert (n, first) == (n_want, first_want)


# ---- the device fill on edge step records

def test_device_fill_on_edge_step_records_past_2p16_timestamps(ctx):
    """2^16 rows and 40000 steps of all 19 opcodes: from the 21845th step on (clk 21845, its write at 3 clk + 3) the timestamps pass 2^16,
    so the CH*Minus borrow is taken on the device for every opcode."""
    ls = 16
    steps, final_ctr = alu_edge_steps(ls, 40000, seed=ls + 100)
    out = ctx.upload(np.random.default_rng(ls).integers(0, 1 << 32, (N_MAIN, 1 << ls), dtype=np.uint64).astype(np.uint32))
    assert ctx.v1_alu_trace(steps, final_ctr, ls, out=out) is out
    bad = np.argwhere(out.download() != _want(steps, final_ctr, ls))
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"


# ---- 2^16 rows: many CTAs and waves in every kernel

@pytest.mark.slow
def test_at_2p16(ctx, alu, capfd):
    m = alu(16)
    gpu, orc_p, params = committed(ctx, m, rw.random_trees(m, 16, "full"))
    check_full_route(ctx, m, gpu, orc_p, params, 6)
    assert check_half_route(ctx, m, gpu, orc_p, params, 7) == 1
    no_fallback(capfd)
    check_report(m, gpu, orc_p, params)


@pytest.mark.slow
def test_sharded_quotients_at_2p16(ctx, alu):
    """The fused pipeline computes D2 with the mid kernel's two forward heads; the ALU program's D2 kernel reads 127 tree-1 columns (the ADD
    chain's 96, v1's 87), so its column groups end elsewhere than theirs."""
    compare(ctx, alu(16), "full", 870)
