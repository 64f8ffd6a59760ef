"""The whole machine's generated kernels (whole_machine.NexusV1KeccakMachine: the v1 main component with KeccakChip, the eight base
extensions and the six keccak components) on witnesses where every constraint matters, checked without a GPU.

The machine's own witness leaves 146 of the main component's 414 constraints identically zero, and 200 of the keccak memory check's 802
(tests/random_witness.py), so a comparison on it cannot see a wrong operand inside them.  Here, for every component that has a generated
source, the host-compiled kernels run on the `full`, `main_random` and `sparse` witnesses at 2^8 main rows with 15 permutations: the
constraint kernel (variant 0) and the main component's D2 kernel (variant 2) against the oracle's quotients, the LogUp kernel (variant 1)
against the oracle's interaction trace, the check kernel (variant 3) against the oracle's check.  The mutation tests show what the valid
witness misses: a one-token change inside a constraint that only the whole machine has passes the valid-witness comparison and fails the
`full` one."""
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200 import nexus_v1 as V
from nexus_zkvm_b200 import whole_machine as W
from oracle import pyoracle as orc
from tests import constraint_ref as ref
from tests import oracle_check
from tests import random_witness as rw
from tests import test_constraint_check_cpu as chk
from tests.test_d2_high_degree_cpu import DRIVER_HIGH, _d2_masks, _load, _source
from tests.test_jit_codegen_cpu import DRIVER, LOGUP_DRIVER, host_build, parse_component
from tests.test_v1_random_witness_cpu import committed, high_flags, mutate_neighbour_mask, mutate_swap_sub, quotient_mismatches

P = (1 << 31) - 1
u32p = C.POINTER(C.c_uint32)
N_COMPONENTS = 15
MAIN, MEMORY_CHECK = 0, 9
# the components each generated variant exists for (jit.cu jit_specialised: a constraint or LogUp program of at least 64 instructions, a D2
# kernel where such a program has constraints of degree above 2, a check kernel wherever there are constraints).  Only the main component
# (log_expand 2) is evaluated on the half domains, so only its D2 kernel runs.
HAS_SOURCE = {0: [0, 1, 2, 3, 9, 10, 11, 12, 13], 1: [0, 1, 3, 9, 10, 11, 12, 13], 2: [0, 1, 3, 9, 10, 11, 12, 13], 3: list(range(N_COMPONENTS))}


@pytest.fixture(scope="module")
def wm():
    return W.NexusV1KeccakMachine(8, 15, seed=1)


@pytest.fixture(scope="module")
def sources(wm):
    """{(component, variant): generated CUDA C or None}, and the main component's D2 column set."""
    h = _load(wm.words)
    try:
        src = {(k, which): _source(h, k, which) for k in range(N_COMPONENTS) for which in range(4)}
        src["d2_masks"] = _d2_masks(h, MAIN, len(parse_component(wm.words, MAIN)[3]))
        return src
    finally:
        nb.lib().nb200_air_free(h)


def _host_build(path, src, which):
    path.mkdir(parents=True)
    if which == 3:
        return chk.host_build(path, src)
    return host_build(path, src, {0: DRIVER_HIGH, 1: LOGUP_DRIVER, 2: DRIVER}[which])


@pytest.fixture(scope="module")
def libs(sources, tmp_path_factory):
    """Every generated source compiled for the host, concurrently: the keccak round components' constraint and LogUp sources take half a
    minute each with g++ -O1."""
    root = tmp_path_factory.mktemp("whole_machine")
    todo = {key: s for key, s in sources.items() if key != "d2_masks" and s is not None and (key[1] != 2 or key[0] == MAIN)}
    with ThreadPoolExecutor(max_workers=max(1, min(len(todo), os.cpu_count() or 1))) as ex:
        built = {key: ex.submit(_host_build, root / f"{key[0]}_{key[1]}", s, key[1]) for key, s in todo.items()}
        return {key: f.result() for key, f in built.items()}


def test_every_component_has_the_sources_it_should(wm, sources):
    assert len(wm.air.components) == N_COMPONENTS
    for which, comps in HAS_SOURCE.items():
        assert [k for k in range(N_COMPONENTS) if sources[(k, which)] is not None] == comps, which


def _census(wm, trees):
    return [int(np.sum(rw.identically_zero(wm.words, k, trees))) for k in range(N_COMPONENTS)]


def test_identically_zero_census(wm):
    """Under the machine's own witness: the constraints that trees 0 and 1 alone make identically zero, then with the generated interaction
    trace as well, per component.  The main component keeps v1's 145 and 42 of the 45 it evaluates on D2, KeccakChip's booleanity on the
    always-zero IsCustomKeccak adds one; BitOpMultiplicity's multiplicities are zero (no bit-op lookup), RamInitFinal's output constraint
    reads only the zero output columns (no exit code or public output), and the keccak memory check has 200 on columns the witness never
    sets.  Under `full` and `main_random` none is left; `sparse` keeps RamInitFinal's, which reads only preprocessed columns."""
    _p, _params, trees = committed(wm, "padding")
    assert _census(wm, trees[:2]) == [146, 0, 0, 1, 0, 0, 0, 0, 0, 200, 0, 0, 0, 0, 0]
    assert _census(wm, trees) == [217, 0, 2, 1, 0, 0, 0, 0, 0, 200, 0, 0, 0, 0, 0]
    high = high_flags(wm, MAIN)
    assert (len(high), int(high.sum())) == (414, 45)
    for t in (trees[:2], trees):
        assert int((np.array(rw.identically_zero(wm.words, MAIN, t)) & high).sum()) == 42
    for kind in ("full", "main_random"):
        _p, _params, trees = committed(wm, kind)
        assert _census(wm, trees) == [0] * N_COMPONENTS, kind
    _p, _params, trees = committed(wm, "sparse")
    assert _census(wm, trees) == [0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0]


@pytest.mark.parametrize("kind", ["full", "main_random"])
def test_constraint_kernels_match_the_oracle(wm, sources, libs, kind):
    """Every component's constraint kernel (all constraints, and the high-degree ones on the side), and the main component's D2 kernel."""
    bad = {}
    for k in HAS_SOURCE[0]:
        d2 = (libs[(k, 2)], sources["d2_masks"]) if k == MAIN else (None, None)
        got = quotient_mismatches(wm, libs[(k, 0)], d2[0], d2[1], kind, k=k)
        if got:
            bad[k] = got
    assert bad == {}


def finalize_last(last, log_size):
    """LogupColGenerator::finalize_last on the last secure column's four coordinate columns (committed order), as the library does outside
    the kernel (interp.cu logup_finalize_last): the claimed sum, then each coordinate less claimed / 2^log_size, prefix-summed in coset
    (trace) order.  Returns (columns, claimed sum)."""
    n = 1 << log_size
    pos = np.asarray(orc.finalize_column(np.arange(n, dtype=np.uint32)), dtype=np.int64)   # committed row i holds trace row pos[i]
    claimed = [int(c.astype(np.int64).sum() % P) for c in last]
    shift = M.F.qm31_mul_m31(tuple(claimed), M.F.m31_inv(n % P))
    out = np.empty_like(last)
    for i, c in enumerate(last):
        trace = np.empty(n, np.int64)
        trace[pos] = (c.astype(np.int64) - shift[i]) % P
        out[i] = (np.cumsum(trace) % P)[pos]
    return out, tuple(claimed)


def test_logup_kernels_match_the_oracle_on_random_trees(wm, libs):
    """Every generated interaction-trace kernel on random trees 0 and 1 with random lookup elements: every column, the last secure one after
    the coset-order prefix sum the library applies outside the kernel, and the claimed sum equal the oracle's LogupTraceGenerator."""
    p, params, trees = committed(wm, "full")
    prm = np.ascontiguousarray(np.array(params, dtype=np.uint32).reshape(-1, 4))
    bad = []
    for k in HAS_SOURCE[1]:
        comp = wm.air.components[k]
        n_logup = max(comp.batching) + 1
        want, want_sum = p.p.gen_interaction(k, comp.log_size, n_logup, np.array(params, dtype=np.uint32))
        want = np.asarray(want, dtype=np.uint32).reshape(4 * n_logup, -1)
        masks = parse_component(wm.words, k)[3]
        zero = np.zeros(1 << comp.log_size, np.uint32)
        keep = [np.ascontiguousarray(trees[t][c] if (t < 2 and off == 0) else zero, dtype=np.uint32) for (t, c, off) in masks]
        col_ptrs = (u32p * len(masks))(*[a.ctypes.data_as(u32p) for a in keep])
        out = np.zeros((4 * n_logup, 1 << comp.log_size), np.uint32)
        libs[(k, 1)].run_rows(col_ptrs, prm.ctypes.data_as(u32p), out.ctypes.data_as(u32p), C.c_uint32(comp.log_size),
                              C.c_uint32(1 << comp.log_size))
        out[-4:], got_sum = finalize_last(out[-4:], comp.log_size)
        if not np.array_equal(out, want) or got_sum != tuple(int(x) for x in want_sum):
            bad.append(k)
    assert bad == []


@pytest.mark.parametrize("kind", ["sparse", "full"])
def test_check_kernels_match_the_oracle(wm, libs, kind):
    """Per constraint of every component, the failing row count and first failing row of the host-compiled check kernel equal the oracle's
    check, and the numpy restatement agrees with both."""
    _p, params, trees = committed(wm, kind)
    failing, n_constraints = [], []
    for k in range(N_COMPONENTS):
        got = chk.run_host_kernel(libs[(k, 3)], wm.words, k, trees, params)
        want = oracle_check.check(wm.words, k, trees, params)
        assert got == want, k
        assert ref.check(wm.words, k, trees, params) == want, k
        failing.append(sum(1 for a, _b in want if a))
        n_constraints.append(len(want))
    if kind == "full":                                       # every constraint fails somewhere
        assert failing == n_constraints
    else:                                                    # the broken cells reach the main component and the keccak ones
        assert all(failing[k] for k in (MAIN, MEMORY_CHECK, 10, 11)), failing


# ---- mutations: a one-token change of the emitted source inside a constraint that only the whole machine has and its witness zeroes

def keccak_chip_booleanity(wm):
    """Index of KeccakChip's constraint IsCustomKeccak * (1 - IsCustomKeccak) in the main component: the one constraint whose only column
    is IsCustomKeccak's."""
    names = [n for n, _w in V.MAIN_COLUMNS]
    col = sum(w for _n, w in V.MAIN_COLUMNS[:names.index("IsCustomKeccak")])
    comp = wm.air.components[MAIN]

    def leaves(n, seen):
        op, a, b, _k = comp.nodes[n]
        if op in ("mask", "maske"):
            seen.add(comp.masks[a])
        elif op not in ("const", "param"):
            leaves(a, seen)
            if op not in ("neg", "btoe"):
                leaves(b, seen)
        return seen

    found = [i for i, n in enumerate(comp.constraints) if leaves(n, set()) == {(1, col, 0)}]
    assert len(found) == 1, found
    return found[0]


@pytest.mark.parametrize("where,how", [("keccak_chip", "swap_sub"), ("memory_check", "swap_sub"), ("memory_check", "neighbour_mask")])
def test_mutation_is_seen_by_the_full_witness_only(wm, sources, libs, tmp_path, where, how):
    """KeccakChip's booleanity in the main component, or one of the keccak memory check's 200 constraints that the machine's witness zeroes,
    computes y - x for x - y, or reads the next zero column: the valid-witness comparison passes, the `full` one fails."""
    k_comp = MAIN if where == "keccak_chip" else MEMORY_CHECK
    _p, _params, trees = committed(wm, "padding")
    zero = rw.identically_zero(wm.words, k_comp, trees[:2])
    candidates = [keccak_chip_booleanity(wm)] if where == "keccak_chip" else [i for i, z in enumerate(zero) if z]
    n_masks = len(parse_component(wm.words, k_comp)[3])
    if how == "swap_sub":
        k, src = mutate_swap_sub(sources[(k_comp, 0)], wm, candidates)
    else:
        k, src = mutate_neighbour_mask(sources[(k_comp, 0)], wm, candidates, [True] * n_masks, k_comp)
    assert src != sources[(k_comp, 0)] and zero[k]
    lib = host_build(tmp_path, src, DRIVER_HIGH)
    d2 = (libs[(MAIN, 2)], sources["d2_masks"]) if k_comp == MAIN else (None, None)
    good = libs[(k_comp, 0)]
    assert quotient_mismatches(wm, lib, *d2, "padding", good, k=k_comp) == [], (k, "the valid witness sees the mutation")
    bad = quotient_mismatches(wm, lib, *d2, "full", good, k=k_comp)
    assert bad, (k, "the full witness misses the mutation")
    assert not any("D2 kernel" in b for b in bad), bad          # only the mutated kernel's sums are off
