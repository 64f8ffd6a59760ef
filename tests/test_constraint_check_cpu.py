"""The constraint check (nb200_check_constraints) WITHOUT a GPU: the CUDA C that nb200_air_kernel_source(..., 3) emits is compiled as host
C++ behind this file's shim — warp intrinsics and atomics with their one-thread meanings — and run row by row; its report (failing rows and
first failing coset row per constraint) must equal the oracle's check (tests/oracle_check.py: orc::run_program on every trace row) on valid
and broken witnesses.  The per-warp aggregation across 32 lanes is exercised by the GPU tests (tests/test_gpu_constraint_check.py)."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from oracle import pyoracle as orc
from tests import constraint_ref as ref
from tests import oracle_check
from tests.oracle_backend import OracleBackend

P = (1 << 31) - 1
u32p = C.POINTER(C.c_uint32)

SHIM = r'''
#include <cstdint>
#include <cstring>
struct uint4 { unsigned x, y, z, w; };
struct uint2 { unsigned x, y; };
#define __device__
#define __forceinline__ inline
#define __noinline__
#define __global__
#define __restrict__
#define __launch_bounds__(...)
#define __constant__
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned s) { return (unsigned)(((((unsigned long long)hi) << 32) | lo) >> (s & 31)); }
static inline unsigned __brev(unsigned x) { unsigned r = 0; for (int i = 0; i < 32; ++i) r |= ((x >> i) & 1u) << (31 - i); return r; }
struct Idx { unsigned x; };
static Idx blockIdx, blockDim, threadIdx;
static inline void __syncthreads() {}
// a warp of one thread
static inline unsigned __activemask() { return 1u; }
static inline unsigned __ballot_sync(unsigned, bool p) { return p ? 1u : 0u; }
static inline unsigned __reduce_min_sync(unsigned, unsigned v) { return v; }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __ffs(unsigned x) { return __builtin_ffs((int)x); }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p = o + v; return o; }
static inline unsigned atomicMin(unsigned* p, unsigned v) { unsigned o = *p; if (v < o) *p = v; return o; }
'''

DRIVER = r'''
extern "C" void run_rows(const unsigned* const* cols, const unsigned* params, unsigned* nfail, unsigned* first, unsigned rows) {
  blockDim.x = 1; threadIdx.x = 0;
  for (unsigned i = 0; i < NB_NMASKS; ++i) ccols[i] = cols[i];   // the library fills the __constant__ table before the launch
  for (unsigned r = 0; r < rows; ++r) { blockIdx.x = r; nbjit(params, nfail, first); }
}
'''


def kernel_source(words, comp, which=3):
    w = np.ascontiguousarray(words, dtype=np.uint32)
    h = C.c_void_p()
    assert nb.lib().nb200_air_load(None, w.ctypes.data_as(u32p), C.c_size_t(w.size), C.byref(h)) == 0
    src = C.c_void_p()
    st = nb.lib().nb200_air_kernel_source(h, C.c_uint32(comp), C.c_int(which), C.byref(src))
    out = C.string_at(src) if st == 0 else None
    if st == 0:
        nb.lib().nb200_free(src)
    nb.lib().nb200_air_free(h)
    return st, out


def host_build(path, source):
    src = source.decode()
    asm = 'asm("mad.wide.u32 %0, %1, 2, %2;" : "=l"(y) : "r"((u32)(x >> 32)), "l"((u64)(u32)x));'
    assert src.count(asm) == 1, "the generated prelude changed: update the host shim of this test"
    src = src.replace(asm, "y = (u64)(u32)(x >> 32) * 2ull + (u64)(u32)x;")
    cu = path / "check_host.cc"
    cu.write_text(SHIM + src + DRIVER)
    so = path / "check_host.so"
    subprocess.run(["/usr/bin/g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-w", str(cu), "-o", str(so)], check=True)
    return C.CDLL(str(so))


def witness(m, t1):
    """The Machine::prove sequence on the oracle up to the tree-2 commit: (trees [tree][col] in committed order, params, components' log sizes)."""
    be = OracleBackend()
    ch = be.channel()
    p = be.prover(m.words, dict(pow_bits=5, log_blowup=1, log_last=0, n_queries=3))
    p.commit(m.preprocessed_columns(), ch, coset_order=True)
    p.commit(t1, ch, coset_order=True)
    params = [(0, 0, 0, 0)] * m.air.n_params
    for rel in (getattr(m, "relations", None) or [m.range256]):
        rel.draw(ch, params)
    inter = []
    for k, comp in enumerate(m.air.components):
        c, cs = p.gen_interaction(k, comp.log_size, max(comp.batching) + 1, params)
        inter.append(c)
        params[comp.cumsum_shift_param] = M.F.qm31_mul_m31(cs, M.F.m31_inv((1 << comp.log_size) % P))
    tree0 = [orc.finalize_column(c) for c in ref.flat(m.preprocessed_columns())]
    tree1 = [orc.finalize_column(c) for c in t1]
    tree2 = [np.array(c, dtype=np.uint32) for block in inter for c in block]
    return [tree0, tree1, tree2], params


def mutated(m, t1, case):
    """(trees, params) of one of the broken witnesses (or the valid one), built from the valid trace t1."""
    trees, params = witness(m, t1)
    ref.apply_case(m, trees, params, case)
    return trees, params


def run_host_kernel(lib, words, comp, trees, params):
    _ls, masks, prog = ref.parse_component(words, comp)
    n_constraints = sum(1 for ins in prog if ins[0] in (17, 18))
    cols = [np.ascontiguousarray(trees[t][c], dtype=np.uint32) for (t, c, _o) in masks]
    ptrs = (u32p * max(len(cols), 1))(*[c.ctypes.data_as(u32p) for c in cols])
    prm = np.ascontiguousarray(np.array(params, dtype=np.uint32).reshape(-1, 4))
    nfail = np.zeros(n_constraints, np.uint32)
    first = np.full(n_constraints, 0xFFFFFFFF, np.uint32)
    lib.run_rows(ptrs, prm.ctypes.data_as(u32p), nfail.ctypes.data_as(u32p), first.ctypes.data_as(u32p), C.c_uint32(1 << _ls))
    return [(int(a), None if b == 0xFFFFFFFF else int(b)) for a, b in zip(nfail, first)]


@pytest.mark.parametrize("kind", ref.KINDS, ids=ref.KIND_IDS)
def test_host_compiled_check_kernel_matches_the_reference(tmp_path, kind):
    m, t1 = ref.make_machine(kind)
    libs = {}
    for k in range(len(m.air.components)):
        st, src = kernel_source(m.words, k)
        assert st == 0
        (tmp_path / str(k)).mkdir()
        libs[k] = host_build(tmp_path / str(k), src)
    main = m.air.components[0]
    n = 1 << main.log_size
    for case in ref.cases(kind):
        trees, params = mutated(m, t1, case)
        reports = {}
        for k in range(len(m.air.components)):
            want = oracle_check.check(m.words, k, trees, params)
            got = run_host_kernel(libs[k], m.words, k, trees, params)
            assert got == want, (case, k)
            assert ref.check(m.words, k, trees, params) == want, (case, k)   # the numpy restatement agrees with the oracle
            reports[k] = [(i, a, b) for i, (a, b) in enumerate(got) if a]
        if case == "valid":
            assert all(not r for r in reports.values()), reports
            continue
        assert reports[0], case                          # every broken case is seen in the main component, and only there
        assert all(not r for k, r in reports.items() if k), case
        if case == "cumsum_shift":                       # the last LogUp constraint, on every row
            n_main = len(main.constraints)
            assert reports[0] == [(n_main - 1, n, 0)]
        if case == "edges":
            assert any(b == 0 for (_i, _a, b) in reports[0]), reports[0]


def test_machine_check_constraints_on_the_oracle():
    """machine.check_constraints drives the oracle backend too: the valid witness holds, a changed limb of a 2^4-row component is named."""
    m, t1 = ref.make_machine("multi")
    report, balanced = M.check_constraints(m, oracle_check.OracleCheckBackend(), t1, None)
    assert balanced and set(report) == set(range(len(m.air.components))) and not any(report.values())
    t1 = [c.copy() for c in t1]
    t1[3][5] = (int(t1[3][5]) + 1) % 256                 # an ADD limb, before the interaction trace
    report, balanced = M.check_constraints(m, oracle_check.OracleCheckBackend(), t1, None)
    assert not balanced and report[0] and all(first == 5 for (_k, _d, _n, first) in report[0])
    assert not any(r for k, r in report.items() if k)


def test_check_source_variant_and_key():
    """Variant 3 is produced without a device for every component, short programs included, and its cache key differs from the others'."""
    m = M.MultiMachine([4, 5, 8])
    lib = nb.lib()
    lib.nb200_kernel_source_key.restype = C.c_uint64
    lib.nb200_kernel_source_key.argtypes = [C.c_char_p]
    for k in range(len(m.air.components)):
        st, src = kernel_source(m.words, k, 3)
        assert st == 0 and src.startswith(b"// constraint check")
        others = [s for st_w, s in (kernel_source(m.words, k, w) for w in (0, 1, 2)) if st_w == 0]
        keys = {lib.nb200_kernel_source_key(s) for s in others + [src]}
        assert len(keys) == len(others) + 1
    assert kernel_source(m.words, 0, 4)[0] == 2          # NB200_ERR_ARG
