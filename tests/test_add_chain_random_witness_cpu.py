"""The ADD chain's generated kernels (add_chain.AddChainMachine, main component with DecodingCheck types R and I) on witnesses where every
constraint matters, and its device fill's row code on step records at the edges of u32, checked without a GPU.

The executing ADD chain leaves every opcode flag but IsAdd / ImmC zero, so 181 of the main component's 486 constraints, 80 of the 110 the
D2 kernel evaluates and 55 of the 73 DecodingCheck constraints are identically zero under it (tests/random_witness.py): a wrong operand in
one of them leaves the kernels equal to the oracle on the executing trace.  Here the comparisons of test_v1_random_witness_cpu.py run on
the `full`, `main_random` and `sparse` witnesses at 2^8 rows: the D1 kernel (variant 0) with its q_high side sum and the D2 kernel
(variant 2) against the oracle's quotients, the LogUp kernel (variant 1) against the oracle's interaction trace, the check kernel
(variant 3) of every component against the oracle's check.  The mutation tests show what the executing trace misses.

The fill's row code (csrc/v1_trace.cuh, compiled as host C++) is compared with add_chain.main_columns on synthetic step records that the
device fill's host check accepts but no ADD chain produces: every u32 word drawn with weight on the carries of 16 and 32 bits, ADDI
immediates of any bit pattern, previous timestamps up to cur - 1 and with a borrow out of the low half, program counters up to 2^32 - 2,
and more or fewer program rows than steps."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import add_chain as AC
from nexus_zkvm_b200 import nexus_v1 as V
from tests import constraint_ref as ref
from tests import oracle_check
from tests import random_witness as rw
from tests import test_constraint_check_cpu as chk
from tests.keccak_side_notes import finalized_src_rows
from tests.test_add_chain_cpu import CSRC, OFFSETS, DRIVER as FILL_DRIVER
from tests.test_d2_high_degree_cpu import DRIVER_HIGH, _d2_masks, _load, _source
from tests.test_jit_codegen_cpu import DRIVER, LOGUP_DRIVER, host_build, parse_component
from tests.test_v1_random_witness_cpu import committed, high_flags, mutate_neighbour_mask, mutate_swap_sub, quotient_mismatches

P = (1 << 31) - 1
u32p = C.POINTER(C.c_uint32)
LOG_SIZE = 8


def _machine():
    """AddChainMachine(LOG_SIZE) and the range of its main component's DecodingCheck constraints (recorded by V._record_decoding_r_i)."""
    seen = []
    orig = V._record_decoding_r_i

    def wrapped(comp, *a):
        first = len(comp.constraints)
        orig(comp, *a)
        seen.append(range(first, len(comp.constraints)))

    V._record_decoding_r_i = wrapped
    try:
        m = AC.AddChainMachine(LOG_SIZE)
    finally:
        V._record_decoding_r_i = orig
    (dec,) = seen
    return m, dec


@pytest.fixture(scope="module")
def chain():
    return _machine()


@pytest.fixture(scope="module")
def sources(chain):
    m, _dec = chain
    h = _load(m.words)
    try:
        return {"d1": _source(h, 0, 0), "logup": _source(h, 0, 1), "d2": _source(h, 0, 2),
                "d2_masks": _d2_masks(h, 0, len(parse_component(m.words, 0)[3]))}
    finally:
        nb.lib().nb200_air_free(h)


@pytest.fixture(scope="module")
def libs(sources, tmp_path_factory):
    d1, d2 = tmp_path_factory.mktemp("d1"), tmp_path_factory.mktemp("d2")
    return host_build(d1, sources["d1"], DRIVER_HIGH), host_build(d2, sources["d2"], DRIVER)


def test_identically_zero_constraints(chain):
    """Under the executing witness, trees 0 and 1 alone make 181 of the 486 main-component constraints identically zero, 80 of the 110 of
    degree > 2 among them, and 55 of the 73 DecodingCheck constraints (47 of their 65 of degree > 2).  Under the random witnesses none is."""
    m, dec = chain
    high = high_flags(m)
    in_dec = np.zeros(len(high), bool)
    in_dec[list(dec)] = True
    assert (len(high), int(high.sum())) == (486, 110)
    assert (int(in_dec.sum()), int((in_dec & high).sum())) == (73, 65)
    _p, _params, trees = committed(m, "padding")
    z = np.array(rw.identically_zero(m.words, 0, trees[:2]))
    assert (int(z.sum()), int((z & high).sum())) == (181, 80)
    assert (int((z & in_dec).sum()), int((z & in_dec & high).sum())) == (55, 47)
    for kind in rw.KINDS:
        _p, _params, trees = committed(m, kind)
        assert not any(rw.identically_zero(m.words, 0, trees)), kind


def test_sparse_corrupts_the_executing_trace(chain):
    """The `sparse` witness of the ADD chain is its executing trace with a few cells replaced, not a padding trace."""
    m, _dec = chain
    t1 = rw.random_trees(m, 11, "sparse").tree1
    exe = ref.flat(m.fill_main_trace())
    same = sum(int((a == b).sum()) for a, b in zip(t1, exe))
    total = sum(a.size for a in exe)
    assert total - total // 20 < same < total
    assert not exe[OFFSETS["IsPadding"]].any()                                    # no padding row in the 2^8-step chain


@pytest.mark.parametrize("kind", ["full", "main_random"])
def test_d1_and_d2_kernels_match_the_oracle(chain, sources, libs, kind):
    m, _dec = chain
    assert quotient_mismatches(m, *libs, sources["d2_masks"], kind) == []


def test_logup_kernel_matches_the_oracle_on_random_trees(chain, sources, tmp_path):
    """The interaction-trace kernel on random trees 0 and 1 with random lookup elements: every column but the last secure one (which
    also gets the coset-order prefix sum outside the kernel) equals the oracle's LogupTraceGenerator."""
    m, _dec = chain
    p, params, trees = committed(m, "full")
    comp = m.air.components[0]
    n_logup = max(comp.batching) + 1
    want, _cs = p.p.gen_interaction(0, comp.log_size, n_logup, np.array(params, dtype=np.uint32))
    lib = host_build(tmp_path, sources["logup"], LOGUP_DRIVER)
    masks = parse_component(m.words, 0)[3]
    zero = np.zeros(1 << comp.log_size, np.uint32)
    keep = [trees[t][c] if (t < 2 and off == 0) else zero for (t, c, off) in masks]
    col_ptrs = (u32p * len(masks))(*[np.ascontiguousarray(a, dtype=np.uint32).ctypes.data_as(u32p) for a in keep])
    prm = np.ascontiguousarray(np.array(params, dtype=np.uint32).reshape(-1, 4))
    out = np.zeros((4 * n_logup, 1 << comp.log_size), np.uint32)
    lib.run_rows(col_ptrs, prm.ctypes.data_as(u32p), out.ctypes.data_as(u32p), C.c_uint32(comp.log_size), C.c_uint32(1 << comp.log_size))
    assert n_logup > 1 and np.array_equal(out[:4 * (n_logup - 1)], want[:4 * (n_logup - 1)])


@pytest.mark.parametrize("kind", ["sparse", "full"])
def test_check_kernel_matches_the_oracle(chain, tmp_path, kind):
    """Per constraint of each of the nine components, the failing row count and first failing row of the host-compiled check kernel equal
    the oracle's check, and the numpy restatement agrees with both."""
    m, dec = chain
    _p, params, trees = committed(m, kind)
    assert len(m.air.components) == 9
    for k in range(len(m.air.components)):
        st, src = chk.kernel_source(m.words, k)
        assert st == 0
        (tmp_path / str(k)).mkdir()
        got = chk.run_host_kernel(chk.host_build(tmp_path / str(k), src), m.words, k, trees, params)
        want = oracle_check.check(m.words, k, trees, params)
        assert got == want, k
        assert ref.check(m.words, k, trees, params) == want, k
        if k == 0:
            failing = [i for i, (a, _b) in enumerate(want) if a]
            if kind == "full":
                assert len(failing) == len(want)
            else:                                 # the broken cells: DecodingCheck constraints fail on rows of their own
                assert len(failing) > len(want) // 4 and sum(i in dec for i in failing) > len(dec) // 2


# ---- mutations: a one-token change inside a DecodingCheck constraint that the executing trace makes identically zero

@pytest.mark.parametrize("where,how", [("d1", "neighbour_mask"), ("d1", "swap_sub"), ("d2", "neighbour_mask"), ("d2", "swap_sub")])
def test_mutation_is_seen_by_the_full_witness_only(chain, sources, libs, tmp_path, where, how):
    m, dec = chain
    high = high_flags(m)
    _p, _params, trees = committed(m, "padding")
    zero = rw.identically_zero(m.words, 0, trees[:2])
    # in D1 a low-degree constraint (the D2 kernel does not hold it), in D2 a high one; both DecodingCheck's and zero under the executing trace
    candidates = [k for k in dec if zero[k] and high[k] == (where == "d2")]
    assert candidates
    allowed = sources["d2_masks"] if where == "d2" else [True] * len(sources["d2_masks"])
    if how == "neighbour_mask":
        k, src = mutate_neighbour_mask(sources[where], m, candidates, allowed)
    else:
        k, src = mutate_swap_sub(sources[where], m, candidates)
    assert src != sources[where] and zero[k] and k in dec
    lib = host_build(tmp_path, src, DRIVER_HIGH if where == "d1" else DRIVER)
    pair = (lib, libs[1]) if where == "d1" else (libs[0], lib)
    assert quotient_mismatches(m, *pair, sources["d2_masks"], "padding", libs[0]) == [], (k, "the executing trace sees the mutation")
    bad = quotient_mismatches(m, *pair, sources["d2_masks"], "full", libs[0])
    assert bad, (k, "the full witness misses the mutation")
    assert all(("D2 kernel" in b) == (where == "d2") for b in bad), bad       # only the mutated kernel's sums are off


# ---- the device fill's row code on edge step records

F = {n: i for i, n in enumerate(AC.STEP_FIELDS)}
# (log_size, n_steps, program rows): full and padded traces, final counters on padding rows and fewer of them than steps, a single step,
# and at 2^15 steps timestamps past 2^16, where a previous timestamp's low half can exceed the current one's (the CH*Minus borrow)
EDGE_SHAPES = [(8, 256, 256), (10, 700, 900), (12, 4096, 100), (9, 1, 512), (15, 1 << 15, 3)]
EDGE_IDS = ["2^8-full", "700-in-2^10", "2^12-100-prog", "1-in-2^9", "2^15-borrow"]


def edgy_u32(rng, n):
    """n u32 words: a quarter uniform, the rest drawn from 0, 0xFFFF, 0xFFFC..0x10003 and 0xFFFFFFFC..0xFFFFFFFF (the carries out of 16
    and 32 bits, and the wrap of x + 4)."""
    pick = rng.integers(0, 4, n)
    out = rng.integers(0, 1 << 32, n, dtype=np.uint64)
    edges = np.concatenate([[0, 0xFFFF], np.arange(0xFFFC, 0x10004), np.arange(0xFFFFFFFC, 0x100000000)]).astype(np.uint64)
    out[pick > 0] = edges[rng.integers(0, edges.size, int((pick > 0).sum()))]
    return out.astype(np.uint32)


def edge_steps(log_size, n_steps, n_prog, seed):
    """(steps, final_ctr): a step record of n_steps ADD / ADDI steps that nb200_v1_main_trace's host check accepts (valid_steps), built
    from edges rather than from an execution, and n_prog random final program counters."""
    rng = np.random.default_rng(seed)
    s = np.zeros((len(AC.STEP_FIELDS), n_steps), np.uint64)
    op = rng.integers(0, 2, n_steps)
    s[F["opcode"]] = op
    for f in ("pc", "word", "value_b", "value_c", "rd_prev"):
        s[F[f]] = edgy_u32(rng, n_steps)
    s[F["rd"]], s[F["rs1"]] = rng.integers(0, 32, n_steps), rng.integers(0, 32, n_steps)
    s[F["op_c"]] = np.where(op == AC.OP_ADD, rng.integers(0, 32, n_steps), edgy_u32(rng, n_steps))
    clk = np.arange(1, n_steps + 1, dtype=np.uint64)
    for k in (1, 2, 3):
        cur = 3 * clk + k
        below = (rng.random(n_steps) * cur).astype(np.uint64)                # uniform in [0, cur)
        # a low half at or above cur's (prev still below cur): the borrow out of the low 16 bits of cur - 1 - prev
        hi = cur >> np.uint64(16)
        lo = (cur & np.uint64(0xFFFF)) + (rng.random(n_steps) * (0x10000 - (cur & np.uint64(0xFFFF)))).astype(np.uint64)
        borrow = ((hi - np.minimum(hi, 1)) << np.uint64(16)) | lo
        choice = rng.integers(0, 4, n_steps)
        prev = np.select([choice == 0, choice == 1, (choice == 2) & (hi > 0)], [cur - 1, np.zeros_like(cur), borrow], below)
        s[F[f"ts{k}_prev"]] = prev
    ctr = edgy_u32(rng, n_steps)
    s[F["pc_ctr_prev"]] = np.where(ctr == 0xFFFFFFFF, 0xFFFFFFFE, ctr)
    s[F["pc_ctr_prev"], 0] = 0xFFFFFFFE
    steps = s.astype(np.uint32)
    final_ctr = rng.integers(0, 1 << 32, n_prog, dtype=np.uint64).astype(np.uint32)
    assert valid_steps(steps, final_ctr, log_size)
    return steps, final_ctr


def valid_steps(steps, final_ctr, log_size):
    """nb200_v1_main_trace's host check (csrc/v1_trace.cu), restated."""
    n_steps = steps.shape[1]
    s = {f: steps[i].astype(np.uint64) for i, f in enumerate(AC.STEP_FIELDS)}
    clk = np.arange(1, n_steps + 1, dtype=np.uint64)
    return (n_steps <= 1 << log_size and final_ctr.size <= 1 << log_size and np.all(s["opcode"] <= 1) and np.all(s["rd"] < 32)
            and np.all(s["rs1"] < 32) and np.all((s["opcode"] == 1) | (s["op_c"] < 32)) and np.all(s["pc_ctr_prev"] != 0xFFFFFFFF)
            and all(np.all(s[f"ts{k}_prev"] < 3 * clk + k) for k in (1, 2, 3)))


def edge_want(steps, final_ctr, log_size):
    """The numpy columns of the step record, finalized: (347, 2^log_size)."""
    t = AC.main_columns(steps, final_ctr, log_size)
    return np.stack([limb for name, _ in V.MAIN_COLUMNS for limb in t[name]])[:, finalized_src_rows(log_size)]


@pytest.fixture(scope="module")
def host_fill(tmp_path_factory):
    d = tmp_path_factory.mktemp("v1_fill")
    src, so = d / "fill.cc", d / "fill.so"
    src.write_text(FILL_DRIVER)
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-w", "-I", CSRC, str(src), "-o", str(so)], check=True)
    return C.CDLL(str(so))


@pytest.mark.parametrize("ls,n_steps,n_prog", EDGE_SHAPES, ids=EDGE_IDS)
def test_host_fill_on_edge_step_records(host_fill, ls, n_steps, n_prog):
    steps, final_ctr = edge_steps(ls, n_steps, n_prog, seed=ls * 1000 + n_steps)
    want = edge_want(steps, final_ctr, ls)
    got = np.full((347, 1 << ls), 0, np.uint32)                                      # the device clears the batch first
    st = np.ascontiguousarray(steps)
    host_fill.v1_fill_host(C.c_uint32(n_steps), st.ctypes.data_as(u32p), C.c_uint32(final_ctr.size), final_ctr.ctypes.data_as(u32p),
                           C.c_uint32(ls), got.ctypes.data_as(u32p))
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"
    # the edges show: both carries of Pc + 4 and of b + c, the low one of the program counter's + 1 (its high one needs 2^32 - 1, which the
    # host check refuses), and a borrow where the timestamps pass 2^16
    exec_rows = want[OFFSETS["IsPadding"]] == 0
    for name, limb in (("PcCarry", 0), ("PcCarry", 1), ("CarryFlag", 0), ("CarryFlag", 1), ("ProgCtrCarry", 0)):
        assert n_steps < 64 or want[OFFSETS[name] + limb][exec_rows].any(), (name, limb)
    if 3 * n_steps + 3 >= 1 << 16:
        assert all(want[OFFSETS["CH1Minus"] + 2 * k].any() for k in range(3))
    if n_steps >= 64:
        assert want[OFFSETS["OpC11"]].any() and want[OFFSETS["OpC4_7"]].any() and want[OFFSETS["OpC8_10"]].any()

