"""The half-coset route evaluates only the constraints of degree above 2 on D2 (csrc/prove.cu, quotient_mode), checked without a GPU.

A constraint of degree d <= 2 has a quotient C / Z of circle degree at most 2^(log_size + 1) - in the span of the first half of the
circle-FFT basis at log_expand 2 - so the upper half of the composition comes from the high-degree constraints alone.  These tests
check the degrees the library derives from the bytecode against a walk over the recorded expressions, the v1 column set D2 reads,
the generated D1 / D2 kernels against the oracle, and the algebra itself on the oracle's quotients."""
import ctypes as C
import re

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from oracle import pyoracle as orc
from tests.oracle_backend import OracleBackend
from tests.test_jit_codegen_cpu import DRIVER, _draw, _flat, coeff_table, host_build, parse_component

P = (1 << 31) - 1
u32p = C.POINTER(C.c_uint32)


def _load(words):
    w = np.ascontiguousarray(words, dtype=np.uint32)
    h = C.c_void_p()
    assert nb.lib().nb200_air_load(None, w.ctypes.data_as(u32p), C.c_size_t(w.size), C.byref(h)) == 0
    return h


def _degrees(h, k, n):
    d = (C.c_uint32 * n)()
    assert nb.lib().nb200_air_constraint_degrees(h, C.c_uint32(k), d, C.c_size_t(n)) == 0
    return list(d)


def _d2_masks(h, k, n):
    f = (C.c_uint8 * n)()
    assert nb.lib().nb200_air_d2_masks(h, C.c_uint32(k), f, C.c_size_t(n)) == 0
    return [bool(x) for x in f]


def _source(h, k, which):
    p = C.c_void_p()
    if nb.lib().nb200_air_kernel_source(h, C.c_uint32(k), C.c_int(which), C.byref(p)) != 0:
        return None
    s = C.string_at(p)
    nb.lib().nb200_free(p)
    return s


def _walk_degrees(comp):
    """degree of every recorded constraint expression, by a walk over the component's node DAG (air.py)"""
    memo = {}

    def deg(n):
        if n in memo:
            return memo[n]
        op, a, b, _k = comp.nodes[n]
        if op in ("mask", "maske"):
            d = 1
        elif op in ("const", "param"):
            d = 0
        elif op in ("neg", "btoe"):
            d = deg(a)
        elif op in ("mul", "mul_eb"):
            d = deg(a) + deg(b)
        else:
            d = max(deg(a), deg(b))
        memo[n] = d
        return d

    return [deg(n) for n in comp.constraints]


def _machines():
    from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
    return {"nexus_v1": NexusV1Machine(8), "add_1": M.AddMachine(log_size=8, n_lanes=1),
            "add_2_pairs": M.AddMachine(log_size=8, n_lanes=2, logup_in_pairs=True),
            "add_3": M.AddMachine(log_size=8, n_lanes=3), "prover2_shaped": M.MultiMachine(list(range(4, 12)))}


@pytest.mark.parametrize("name", ["nexus_v1", "add_1", "add_2_pairs", "add_3", "prover2_shaped"])
def test_constraint_degrees_match_the_expression_dag(name):
    m = _machines()[name]
    h = _load(m.words)
    try:
        for k, comp in enumerate(m.air.components):
            assert _degrees(h, k, len(comp.constraints)) == _walk_degrees(comp), f"component {k}"
    finally:
        nb.lib().nb200_air_free(h)


def test_v1_d2_column_set():
    m = _machines()["nexus_v1"]
    comp = m.air.components[0]
    h = _load(m.words)
    try:
        deg = _degrees(h, 0, len(comp.constraints))
        used = _d2_masks(h, 0, len(comp.masks))
        src = _source(h, 0, 2).decode()
    finally:
        nb.lib().nb200_air_free(h)
    assert comp.log_expand == 2
    assert sorted((d, deg.count(d)) for d in set(deg)) == [(1, 11), (2, 357), (3, 23), (4, 22)]
    cols = {(comp.masks[i][0], comp.masks[i][1]) for i in range(len(comp.masks)) if used[i]}
    per_tree = [sum(1 for t, _ in cols if t == tree) for tree in range(3)]
    assert per_tree == [1, 87, 0]
    # the D2 kernel adds exactly the 45 high constraints, each with its own coefficient
    high = [k for k, d in enumerate(deg) if d > 2]
    assert len(high) == 45
    assert sorted({int(x) // 12 for x in re.findall(r"coeff \+ (\d+)\b", src)}) == high
    assert src.count("rr = qadd(rr, qmulb(ldq(coeff + ") + src.count("rr = qmac_tab(") + src.count("rr = qmacq(") == 45


def test_component_without_high_constraints_has_no_d2_kernel():
    m = _machines()["prover2_shaped"]
    h = _load(m.words)
    try:
        for k, comp in enumerate(m.air.components):
            has_high = any(d > 2 for d in _walk_degrees(comp))
            if not has_high:
                assert _source(h, k, 2) is None
    finally:
        nb.lib().nb200_air_free(h)


def _committed(kind, seed):
    """(machine, oracle prover, parameter table, [tree0, tree1, tree2] columns on the trace domain) as Machine::prove commits them"""
    if kind == "nexus_v1":
        from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
        m = NexusV1Machine(8)
        t1 = m.fill_main_trace(seed=seed)
    else:
        lanes, pairs = kind
        m = M.AddMachine(log_size=8, n_lanes=lanes, logup_in_pairs=pairs)
        cols, mult = m.fill_main_trace(seed=seed + lanes, n_padding=2)
        t1 = list(cols) + [mult]
    be = OracleBackend()
    ch = be.channel()
    p = be.prover(m.words, dict(pow_bits=5, log_blowup=1, log_last=0, n_queries=3))
    tree0 = [orc.finalize_column(c) for c in _flat(m.preprocessed_columns())]
    tree1 = [orc.finalize_column(c) for c in _flat(t1)]
    p.commit(m.preprocessed_columns(), ch, coset_order=True)
    p.commit(t1, ch, coset_order=True)
    params = [(0, 0, 0, 0)] * m.air.n_params
    _draw(m, ch, params)
    inter = []
    for k, comp in enumerate(m.air.components):
        c, cs = p.gen_interaction(k, comp.log_size, max(comp.batching) + 1, params)
        inter.append(c)
        params[comp.cumsum_shift_param] = M.F.qm31_mul_m31(cs, M.F.m31_inv((1 << comp.log_size) % P))
    p.commit_interaction(inter, ch)
    return m, p, params, [tree0, tree1, [c for block in inter for c in block]]


def _coeffs(q):
    return np.stack([np.asarray(orc.interpolate(np.ascontiguousarray(q[i], dtype=np.uint32)), dtype=np.uint32) for i in range(4)])


KINDS = [(1, False), (2, True), (3, False), "nexus_v1"]


@pytest.mark.parametrize("kind", KINDS)
def test_upper_half_comes_from_the_high_constraints_alone(kind):
    """On the oracle: the composition of the degree <= 2 constraints has an all-zero upper half of coefficients, so lo from every
    constraint and hi from the high ones give the coefficients of the full evaluation word for word."""
    m, p, params, _trees = _committed(kind, 9)
    log_size, log_expand, n, _masks = parse_component(m.words, 0)
    assert log_expand == 2
    elog = log_size + log_expand
    high = np.array([d > 2 for d in _walk_degrees(m.air.components[0])])
    coeffs = np.random.default_rng(5).integers(0, P, size=(n, 4), dtype=np.uint32)
    prm = np.array(params, dtype=np.uint32)
    full = _coeffs(p.p.constraint_quotients(0, elog, prm, coeffs))
    low = _coeffs(p.p.constraint_quotients(0, elog, prm, np.where(high[:, None], 0, coeffs).astype(np.uint32)))
    hi_only = _coeffs(p.p.constraint_quotients(0, elog, prm, np.where(high[:, None], coeffs, 0).astype(np.uint32)))
    half = 1 << (elog - 1)
    assert not low[:, half:].any()
    assert np.array_equal(hi_only[:, half:], full[:, half:])
    assert np.array_equal((low[:, :half].astype(np.uint64) + hi_only[:, :half]) % P, full[:, :half])


DRIVER_HIGH = r'''
extern "C" void run_rows(const unsigned* const* cols, const unsigned* params, const unsigned* coeff, const unsigned* dinv,
                         unsigned* a0, unsigned* a1, unsigned* a2, unsigned* a3, unsigned* h0, unsigned* h1, unsigned* h2, unsigned* h3,
                         unsigned EL, unsigned rows) {
  blockDim.x = 1; threadIdx.x = 0;
  for (unsigned i = 0; i < NB_NMASKS; ++i) ccols[i] = cols[i];
  for (unsigned r = 0; r < rows; ++r) { blockIdx.x = r; nbjit(cols, params, coeff, dinv, a0, a1, a2, a3, EL, 0u, h0, h1, h2, h3); }
}
'''


@pytest.mark.parametrize("kind", KINDS)
def test_generated_d1_and_d2_kernels_match_the_oracle(tmp_path, kind):
    """The constraint kernel sums every constraint into a0..a3 and the high ones into h0..h3; the D2 kernel, given only the columns
    its constraints read (the others are null), sums the high ones.  Both are run on the host over the whole evaluation domain."""
    m, p, params, trees = _committed(kind, 9)
    log_size, log_expand, n, masks = parse_component(m.words, 0)
    elog = log_size + log_expand
    high = np.array([d > 2 for d in _walk_degrees(m.air.components[0])])
    coeffs = np.random.default_rng(3).integers(0, P, size=(n, 4), dtype=np.uint32)
    prm_q = np.array(params, dtype=np.uint32)
    want_all = p.p.constraint_quotients(0, elog, prm_q, coeffs)
    want_high = p.p.constraint_quotients(0, elog, prm_q, np.where(high[:, None], coeffs, 0).astype(np.uint32))

    h = _load(m.words)
    try:
        src1, src2 = _source(h, 0, 0), _source(h, 0, 2)
        used = _d2_masks(h, 0, len(masks))
    finally:
        nb.lib().nb200_air_free(h)
    assert src2 is not None and src2.startswith(b"// constraint quotients on D2")
    ext = {}
    for (t, c, _off) in masks:
        if (t, c) not in ext:
            ext[(t, c)] = np.ascontiguousarray(orc.evaluate(orc.interpolate(trees[t][c]), elog), dtype=np.uint32)
    prm = np.ascontiguousarray(prm_q.reshape(-1, 4))
    tab = coeff_table(coeffs)
    rows = 1 << elog
    dinv = np.ones(1 << log_expand, np.uint32)
    ptrs = lambda sel: (u32p * len(masks))(*[ext[(t, c)].ctypes.data_as(u32p) if sel[i] else None for i, (t, c, _o) in enumerate(masks)])

    (tmp_path / "d1").mkdir()
    (tmp_path / "d2").mkdir()
    lib1 = host_build(tmp_path / "d1", src1, DRIVER_HIGH)
    acc = [np.zeros(rows, np.uint32) for _ in range(8)]
    lib1.run_rows(ptrs([True] * len(masks)), prm.ctypes.data_as(u32p), tab.ctypes.data_as(u32p), dinv.ctypes.data_as(u32p),
                  *[a.ctypes.data_as(u32p) for a in acc], C.c_uint32(elog), C.c_uint32(rows))
    lib2 = host_build(tmp_path / "d2", src2, DRIVER)
    acc2 = [np.zeros(rows, np.uint32) for _ in range(4)]
    lib2.run_rows(ptrs(used), prm.ctypes.data_as(u32p), tab.ctypes.data_as(u32p), dinv.ctypes.data_as(u32p),
                  *[a.ctypes.data_as(u32p) for a in acc2], C.c_uint32(elog), C.c_uint32(rows))
    got_all, got_high, got_d2 = np.stack(acc[:4]), np.stack(acc[4:]), np.stack(acc2)
    assert np.array_equal(got_high, got_d2)
    # the oracle's quotients carry 1 / vanishing: one field element per block of 2^log_size rows, recovered from got_all
    for blk in range(1 << log_expand):
        sl = slice(blk << log_size, (blk + 1) << log_size)
        g, w_ = got_all[:, sl].astype(object), want_all[:, sl].astype(object)
        r0 = int(np.argwhere(g[0] != 0)[0][0])
        d = int(w_[0][r0]) * pow(int(g[0][r0]), P - 2, P) % P
        assert np.array_equal((g * d) % P, w_), f"block {blk}: every constraint"
        assert np.array_equal((got_high[:, sl].astype(object) * d) % P, want_high[:, sl].astype(object)), f"block {blk}: high constraints"
