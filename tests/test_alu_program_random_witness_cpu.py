"""The ALU program's generated kernels (add_chain.AluMachine: the main component with DecodingCheck types R and I and SltuChip, SltChip,
SllChip, SrlChip and SraChip) on witnesses where every constraint matters, checked without a GPU.

The executing ALU program raises every flag of the 19 instructions, so far fewer constraints vanish under it than under the ADD chain (181
of 486): none of the five chips' constraints and none of DecodingCheck's type-I-with-shift constraints does.  The comparisons of
test_add_chain_random_witness_cpu.py run here on the `full`, `main_random` and `sparse` witnesses at 2^8 rows (tests/random_witness.py):
the D1 kernel (variant 0) with its q_high side sum and the D2 kernel (variant 2) against the oracle's quotients, the LogUp kernel (variant
1) against the oracle's interaction trace, and the check kernel (variant 3) of every component against the oracle's check."""
import ctypes as C

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import nexus_v1 as V
from tests import constraint_ref as ref
from tests import oracle_check
from tests import random_witness as rw
from tests import test_constraint_check_cpu as chk
from tests.test_alu_program_cpu import CHIP_CONSTRAINTS, chip_ranges
from tests.test_d2_high_degree_cpu import DRIVER_HIGH, _d2_masks, _load, _source
from tests.test_jit_codegen_cpu import DRIVER, LOGUP_DRIVER, host_build, parse_component
from tests.test_v1_random_witness_cpu import committed, high_flags, quotient_mismatches

u32p = C.POINTER(C.c_uint32)
LOG_SIZE = 8


@pytest.fixture(scope="module")
def program():
    """AluMachine(LOG_SIZE), {chip: range of its constraints}, and the range of DecodingCheck's type-I-with-shift constraints (the last 15
    that V._record_decoding_r_i records)."""
    seen = []
    orig = V._record_decoding_r_i

    def wrapped(comp, *a):
        first = len(comp.constraints)
        orig(comp, *a)
        seen.append(range(first, len(comp.constraints)))

    V._record_decoding_r_i = wrapped
    try:
        m, chips = chip_ranges(LOG_SIZE)
    finally:
        V._record_decoding_r_i = orig
    (dec,) = seen
    return m, chips, dec, range(dec.stop - 15, dec.stop)


@pytest.fixture(scope="module")
def sources(program):
    m = program[0]
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


def test_identically_zero_constraints(program):
    """Under the executing witness, trees 0 and 1 alone make 121 of the main component's 545 constraints identically zero (the ADD chain:
    181 of 486), 38 of the 144 of degree > 2 among them, and 17 of the 73 DecodingCheck ones (the ADD chain: 55).  None of the new chips'
    constraints and none of type I with a shift amount is.  Under the random witnesses none is."""
    m, chips, dec, shift_i = program
    assert {k: len(v) for k, v in chips.items()} == CHIP_CONSTRAINTS
    high = high_flags(m)
    assert (len(high), int(high.sum())) == (545, 144)
    _p, _params, trees = committed(m, "padding")
    z = np.array(rw.identically_zero(m.words, 0, trees[:2]))
    assert (int(z.sum()), int((z & high).sum()), int(z[list(dec)].sum())) == (121, 38, 17)
    assert not any(z[i] for r in chips.values() for i in r)
    assert not any(z[i] for i in shift_i)
    for kind in rw.KINDS:
        _p, _params, trees = committed(m, kind)
        assert not any(rw.identically_zero(m.words, 0, trees)), kind


@pytest.mark.parametrize("kind", ["full", "main_random"])
def test_d1_and_d2_kernels_match_the_oracle(program, sources, libs, kind):
    assert quotient_mismatches(program[0], *libs, sources["d2_masks"], kind) == []


def test_logup_kernel_matches_the_oracle_on_random_trees(program, sources, tmp_path):
    """The interaction-trace kernel on random trees 0 and 1 with random lookup elements: every column but the last secure one (which
    also gets the coset-order prefix sum outside the kernel) equals the oracle's LogupTraceGenerator."""
    m = program[0]
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
def test_check_kernel_matches_the_oracle(program, tmp_path, kind):
    """Per constraint of each of the nine components, the failing row count and first failing row of the host-compiled check kernel equal
    the oracle's check, and the numpy restatement agrees with both."""
    m, chips, _dec, _shift_i = program
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
            failing = {i for i, (a, _b) in enumerate(want) if a}
            if kind == "full":
                assert len(failing) == len(want)
            else:                                 # the broken cells: most of the new chips' constraints fail on rows of their own
                new = [i for r in chips.values() for i in r]
                assert sum(i in failing for i in new) > len(new) // 2
