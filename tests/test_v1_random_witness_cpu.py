"""The v1 main component's generated kernels on witnesses where every constraint matters, checked without a GPU.

The padding witness makes a third of the v1 constraints, and 42 of the 45 the D2 kernel evaluates, identically zero
(tests/random_witness.py), so the host-compiled comparisons of test_jit_codegen_cpu.py, test_d2_high_degree_cpu.py and
test_constraint_check_cpu.py cannot see a wrong operand inside them.  Here the same comparisons run on the `full`, `main_random` and `sparse`
witnesses at 2^8 rows: the D1 kernel (variant 0) with its q_high side sum and the D2 kernel (variant 2) against the oracle's quotients, the
LogUp kernel (variant 1) against the oracle's interaction trace, the check kernel (variant 3) against the oracle's check.  The mutation tests
show what the padding witness misses: a one-token change inside a constraint that is zero under it passes the padding comparison and fails
the `full` one."""
import ctypes as C
import re

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from oracle import pyoracle as orc
from tests import constraint_ref as ref
from tests import oracle_check
from tests import random_witness as rw
from tests import test_constraint_check_cpu as chk
from tests.test_d2_high_degree_cpu import DRIVER_HIGH, _d2_masks, _load, _source, _walk_degrees
from tests.test_jit_codegen_cpu import DRIVER, LOGUP_DRIVER, coeff_table, host_build, parse_component

P = (1 << 31) - 1
u32p = C.POINTER(C.c_uint32)
LOG_SIZE = 8


@pytest.fixture(scope="module")
def v1():
    from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
    return NexusV1Machine(LOG_SIZE)


@pytest.fixture(scope="module")
def sources(v1):
    h = _load(v1.words)
    try:
        return {"d1": _source(h, 0, 0), "logup": _source(h, 0, 1), "d2": _source(h, 0, 2),
                "d2_masks": _d2_masks(h, 0, len(parse_component(v1.words, 0)[3]))}
    finally:
        nb.lib().nb200_air_free(h)


@pytest.fixture(scope="module")
def libs(v1, sources, tmp_path_factory):
    d1, d2 = tmp_path_factory.mktemp("d1"), tmp_path_factory.mktemp("d2")
    return host_build(d1, sources["d1"], DRIVER_HIGH), host_build(d2, sources["d2"], DRIVER)


_committed = {}


def committed(m, kind, seed=11):
    """(oracle prover, params, trees as committed) of the witness `kind` ("padding" or a random_witness kind), one per kind and size."""
    key = (m.log_size, kind, seed)
    if key not in _committed:
        w = rw.padding(m) if kind == "padding" else rw.random_trees(m, seed, kind)
        _committed[key] = rw.on_oracle(m, w)
    return _committed[key]


def high_flags(m):
    return np.array([d > 2 for d in _walk_degrees(m.air.components[0])])


def quotient_mismatches(m, lib1, lib2, d2_masks, kind, dinv_from=None):
    """Where the host-run D1 kernel (every constraint into a0..a3, the high ones into h0..h3) and D2 kernel (the high ones, from the columns
    they read) differ from the oracle's quotients with all coefficients / with the low-degree ones zeroed, over canonic(eval_log): [] when
    they agree everywhere.  The oracle's quotients carry 1 / vanishing, one field element per block of 2^log_size rows, recovered from one
    row of the D1 kernel's sum, or of the sum of the D1 kernel `dinv_from` when the kernel under test is not to be trusted with it."""
    p, params, trees = committed(m, kind)
    log_size, log_expand, n, masks = parse_component(m.words, 0)
    elog = log_size + log_expand
    high = high_flags(m)
    coeffs = np.random.default_rng(3).integers(0, P, size=(n, 4), dtype=np.uint32)
    prm_q = np.array(params, dtype=np.uint32)
    want_all = p.p.constraint_quotients(0, elog, prm_q, coeffs)
    want_high = p.p.constraint_quotients(0, elog, prm_q, np.where(high[:, None], coeffs, 0).astype(np.uint32))
    ext = {}
    for (t, c, _off) in masks:
        if (t, c) not in ext:
            ext[(t, c)] = np.ascontiguousarray(orc.evaluate(orc.interpolate(trees[t][c]), elog), dtype=np.uint32)
    prm = np.ascontiguousarray(prm_q.reshape(-1, 4))
    tab = coeff_table(coeffs)
    rows = 1 << elog
    dinv = np.ones(1 << log_expand, np.uint32)
    ptrs = lambda sel: (u32p * len(masks))(*[ext[(t, c)].ctypes.data_as(u32p) if sel[i] else None for i, (t, c, _o) in enumerate(masks)])
    acc = [np.zeros(rows, np.uint32) for _ in range(8)]
    lib1.run_rows(ptrs([True] * len(masks)), prm.ctypes.data_as(u32p), tab.ctypes.data_as(u32p), dinv.ctypes.data_as(u32p),
                  *[a.ctypes.data_as(u32p) for a in acc], C.c_uint32(elog), C.c_uint32(rows))
    acc2 = [np.zeros(rows, np.uint32) for _ in range(4)]
    lib2.run_rows(ptrs(d2_masks), prm.ctypes.data_as(u32p), tab.ctypes.data_as(u32p), dinv.ctypes.data_as(u32p),
                  *[a.ctypes.data_as(u32p) for a in acc2], C.c_uint32(elog), C.c_uint32(rows))
    got_all, got_high, got_d2 = np.stack(acc[:4]), np.stack(acc[4:]), np.stack(acc2)
    if dinv_from is not None:
        acc = [np.zeros(rows, np.uint32) for _ in range(8)]
        dinv_from.run_rows(ptrs([True] * len(masks)), prm.ctypes.data_as(u32p), tab.ctypes.data_as(u32p), dinv.ctypes.data_as(u32p),
                           *[a.ctypes.data_as(u32p) for a in acc], C.c_uint32(elog), C.c_uint32(rows))
    ref_all = np.stack(acc[:4])
    bad = []
    for blk in range(1 << log_expand):
        sl = slice(blk << log_size, (blk + 1) << log_size)
        g, w_ = got_all[:, sl].astype(object), want_all[:, sl].astype(object)
        nz = np.argwhere(ref_all[0, sl] != 0)
        assert nz.size, "degenerate block"
        r0 = int(nz[0][0])
        d = int(w_[0][r0]) * pow(int(ref_all[0, sl][r0]), P - 2, P) % P
        if not np.array_equal((g * d) % P, w_):
            bad.append(f"block {blk}: D1 kernel, every constraint")
        if not np.array_equal((got_high[:, sl].astype(object) * d) % P, want_high[:, sl].astype(object)):
            bad.append(f"block {blk}: D1 kernel, the high constraints")
        if not np.array_equal((got_d2[:, sl].astype(object) * d) % P, want_high[:, sl].astype(object)):
            bad.append(f"block {blk}: D2 kernel")
    return bad


def test_identically_zero_constraints(v1):
    """Under the padding witness, trees 0 and 1 alone make 145 of the 413 v1 constraints identically zero, 42 of the 45 of degree > 2
    among them; the generated interaction trace's zero columns add LogUp constraints to those.  Under the random witnesses none is."""
    high = high_flags(v1)
    assert (len(high), int(high.sum())) == (413, 45)
    _p, _params, trees = committed(v1, "padding")
    z = np.array(rw.identically_zero(v1.words, 0, trees[:2]))
    assert (int(z.sum()), int((z & high).sum())) == (145, 42)
    z3 = np.array(rw.identically_zero(v1.words, 0, trees))
    assert int(z3.sum()) > 145 and not (z & ~z3).any() and int((z3 & high).sum()) == 42
    for kind in rw.KINDS:
        _p, _params, trees = committed(v1, kind)
        assert not any(rw.identically_zero(v1.words, 0, trees)), kind


def test_oracle_quotients_on_a_domain_of_the_callers_choice(v1):
    """The oracle's quotients on the committed LDE domain (eval_log = log_size + 1, one below the component's): on a valid witness the
    quotient of the constraints of degree <= 2 is a polynomial of 2^(log_size + 1) coefficients, so there it is the evaluation of the same
    polynomial.  (On the random witnesses the quotients are not polynomials; the kernels are compared with the oracle row by row.)"""
    p, params, _trees = committed(v1, "padding")
    log_size, log_expand, n, _masks = parse_component(v1.words, 0)
    elog = log_size + log_expand
    high = high_flags(v1)
    coeffs = np.random.default_rng(8).integers(0, P, size=(n, 4), dtype=np.uint32)
    low = np.where(high[:, None], 0, coeffs).astype(np.uint32)
    prm = np.array(params, dtype=np.uint32)
    q = p.p.constraint_quotients(0, elog, prm, low)
    assert np.array_equal(p.p.constraint_quotients(0, None, prm, low), q)
    cf = [np.asarray(orc.interpolate(np.ascontiguousarray(q[i])), dtype=np.uint32) for i in range(4)]
    half = 1 << (elog - 1)
    assert not any(c[half:].any() for c in cf)
    q_lde = p.p.constraint_quotients(0, elog - 1, prm, low)
    assert np.array_equal(q_lde, np.stack([orc.evaluate(np.ascontiguousarray(c[:half]), elog - 1) for c in cf]))
    with pytest.raises(orc.OracleError):
        p.p.constraint_quotients(0, log_size, prm, low)


@pytest.mark.parametrize("kind", ["full", "main_random"])
def test_d1_and_d2_kernels_match_the_oracle(v1, sources, libs, kind):
    assert quotient_mismatches(v1, *libs, sources["d2_masks"], kind) == []


def test_logup_kernel_matches_the_oracle_on_random_trees(v1, sources, tmp_path):
    """The interaction-trace kernel on random trees 0 and 1 with random lookup elements: every column but the last secure one (which
    also gets the coset-order prefix sum outside the kernel) equals the oracle's LogupTraceGenerator."""
    p, params, trees = committed(v1, "full")
    comp = v1.air.components[0]
    n_logup = max(comp.batching) + 1
    want, _cs = p.p.gen_interaction(0, comp.log_size, n_logup, np.array(params, dtype=np.uint32))
    lib = host_build(tmp_path, sources["logup"], LOGUP_DRIVER)
    masks = parse_component(v1.words, 0)[3]
    zero = np.zeros(1 << comp.log_size, np.uint32)
    keep = [trees[t][c] if (t < 2 and off == 0) else zero for (t, c, off) in masks]
    col_ptrs = (u32p * len(masks))(*[np.ascontiguousarray(a, dtype=np.uint32).ctypes.data_as(u32p) for a in keep])
    prm = np.ascontiguousarray(np.array(params, dtype=np.uint32).reshape(-1, 4))
    out = np.zeros((4 * n_logup, 1 << comp.log_size), np.uint32)
    lib.run_rows(col_ptrs, prm.ctypes.data_as(u32p), out.ctypes.data_as(u32p), C.c_uint32(comp.log_size), C.c_uint32(1 << comp.log_size))
    assert np.array_equal(out[:4 * (n_logup - 1)], want[:4 * (n_logup - 1)])


@pytest.mark.parametrize("kind", ["sparse", "full"])
def test_check_kernel_matches_the_oracle(v1, tmp_path, kind):
    """Per constraint, the failing row count and first failing row of the host-compiled check kernel equal the oracle's check, and the
    numpy restatement agrees with both, for every component of the v1 machine."""
    _p, params, trees = committed(v1, kind)
    n = 1 << LOG_SIZE
    for k in range(len(v1.air.components)):
        st, src = chk.kernel_source(v1.words, k)
        assert st == 0
        (tmp_path / str(k)).mkdir()
        got = chk.run_host_kernel(chk.host_build(tmp_path / str(k), src), v1.words, k, trees, params)
        want = oracle_check.check(v1.words, k, trees, params)
        assert got == want, k
        assert ref.check(v1.words, k, trees, params) == want, k
        if k == 0:
            failing = [(a, b) for a, b in want if a]
            if kind == "full":                    # every constraint fails
                assert len(failing) == len(want)
            else:                                 # the broken cells: constraints fail on subsets of their own, row 0 among them
                assert len(failing) > len(want) // 4 and len({a for a, _b in failing}) > 4 and max(a for a, _b in failing) < n
                assert any(b == 0 for _a, b in failing)


# ---- mutations: a one-token change of the emitted source inside a constraint that the padding witness makes identically zero

def _zero_masks(m):
    """Per mask of the v1 component: its column is zero in every row of the padding witness (trees 0 and 1)."""
    _p, _params, trees = committed(m, "padding")
    return [t < 2 and not np.any(trees[t][c]) for (t, c, _o) in parse_component(m.words, 0)[3]]


def _statements(src, k):
    """(first line, accumulation line) of constraint k's statements in a generated quotient kernel: the lines after the previous
    constraint's accumulation, up to constraint k's own `rr = qadd(rr, qmulb(ldq(coeff + 12 k), ...))`."""
    lines = src.split("\n")
    end = next((i for i, s in enumerate(lines) if re.search(rf"qmulb\(ldq\(coeff \+ {12 * k}\), b\[\d+\]\)", s)), None)
    if end is None:
        return lines, None, None
    start = max((i for i in range(end) if "rr = q" in lines[i] or "Q rr = s.rr" in lines[i]), default=0) + 1
    return lines, start, end


def mutate_neighbour_mask(src, m, candidates, allowed):
    """Constraint k (the first of `candidates` where this applies) reads mask M + 1 instead of mask M, where both masks are columns of
    their own that are zero under the padding witness (so every value under it is unchanged) and M + 1 is in `allowed`."""
    masks = parse_component(m.words, 0)[3]
    zero = _zero_masks(m)
    src = src.decode()
    for k in candidates:
        lines, start, end = _statements(src, k)
        for i in range(start or 0, end or 0):
            g = re.fullmatch(r"(\s*b\[\d+\] = __ldg\(ccols\[)(\d+)(\] \+ row\);)", lines[i])
            if not g:
                continue
            mk = int(g.group(2))
            if mk + 1 < len(masks) and zero[mk] and zero[mk + 1] and allowed[mk + 1] and masks[mk + 1][2] == 0 and masks[mk + 1][:2] != masks[mk][:2]:
                lines[i] = f"{g.group(1)}{mk + 1}{g.group(3)}"
                return k, "\n".join(lines).encode()
    raise AssertionError("no constraint to mutate: the generated source changed")


def mutate_swap_sub(src, m, candidates):
    """Constraint k (the first of `candidates` where this applies) computes y - x instead of x - y in the subtraction that gives its value,
    or the factor its last product multiplies by: the constraint's value changes sign, which a constraint that is zero on every row hides."""
    src = src.decode()
    for k in candidates:
        lines, start, end = _statements(src, k)
        if end is None or end - 2 < start:
            continue
        acc = re.search(r"b\[(\d+)\]\)\);", lines[end]).group(1)
        last = re.fullmatch(r"\s*b\[(\d+)\] = mul\(b\[(\d+)\], b\[(\d+)\]\);", lines[end - 1])
        for i, want in ((end - 1, {acc}), (end - 2, last and last.group(1) == acc and {last.group(2), last.group(3)})):
            g = re.fullmatch(r"(\s*b\[(\d+)\] = sub\()b\[(\d+)\], b\[(\d+)\](\);)", lines[i])
            if g and want and g.group(2) in want and g.group(3) != g.group(4):
                lines[i] = f"{g.group(1)}b[{g.group(4)}], b[{g.group(3)}]{g.group(5)}"
                return k, "\n".join(lines).encode()
    raise AssertionError("no constraint to mutate: the generated source changed")


@pytest.mark.parametrize("where,how", [("d1", "neighbour_mask"), ("d1", "swap_sub"), ("d2", "neighbour_mask"), ("d2", "swap_sub")])
def test_mutation_is_seen_by_the_full_witness_only(v1, sources, libs, tmp_path, where, how):
    high = high_flags(v1)
    _p, _params, trees = committed(v1, "padding")
    zero = rw.identically_zero(v1.words, 0, trees[:2])
    # in D1 a low-degree constraint (the D2 kernel does not hold it), in D2 a high one; both zero under the padding witness
    candidates = [k for k in range(len(high)) if zero[k] and high[k] == (where == "d2")]
    allowed = sources["d2_masks"] if where == "d2" else [True] * len(sources["d2_masks"])
    if how == "neighbour_mask":
        k, src = mutate_neighbour_mask(sources[where], v1, candidates, allowed)
    else:
        k, src = mutate_swap_sub(sources[where], v1, candidates)
    assert src != sources[where] and zero[k]
    lib = host_build(tmp_path, src, DRIVER_HIGH if where == "d1" else DRIVER)
    pair = (lib, libs[1]) if where == "d1" else (libs[0], lib)
    assert quotient_mismatches(v1, *pair, sources["d2_masks"], "padding", libs[0]) == [], (k, "the padding witness sees the mutation")
    bad = quotient_mismatches(v1, *pair, sources["d2_masks"], "full", libs[0])
    assert bad, (k, "the full witness misses the mutation")
    assert all(("D2 kernel" in b) == (where == "d2") for b in bad), bad       # only the mutated kernel's sums are off
