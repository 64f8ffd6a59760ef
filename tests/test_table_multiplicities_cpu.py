"""Table multiplicities counted from the recorded AIR (nb200_table_multiplicities) WITHOUT a GPU:
  * the classification of every fraction (nb200_air_lookup_tables) is pinned per machine against what air.py records;
  * the count kernel's CUDA C (nb200_air_count_kernel_source) is compiled as host C++ behind this file's shim (atomics, warp intrinsics and
    the grid-stride loop with their one-thread meanings) and run on small witnesses of all four machines: its columns equal the machines'
    own host multiplicity columns;
  * the numpy reference (tests/table_mult_ref.py) agrees with the same host columns.
Shared-memory bins, the 32-lane aggregation and the real atomics are exercised by tests/test_gpu_table_multiplicities.py."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200.keccak import KeccakMachine
from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
from oracle import pyoracle as orc
from tests import table_mult_ref as ref

P = (1 << 31) - 1
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)
KIND = {0: "ignored", 1: "table", 2: "lookup", 3: "bad"}

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
#define __shared__
template <class T> static inline T __ldg(const T* p) { return *p; }
template <class T> static inline T __ldcg(const T* p) { return *p; }
static inline void __threadfence() {}
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned s) { return (unsigned)(((((unsigned long long)hi) << 32) | lo) >> (s & 31)); }
static inline unsigned __brev(unsigned x) { unsigned r = 0; for (int i = 0; i < 32; ++i) r |= ((x >> i) & 1u) << (31 - i); return r; }
struct Idx { unsigned x; };
static Idx blockIdx, blockDim, threadIdx, gridDim;
static inline void __syncthreads() {}
// a warp of one thread, a grid of one thread
static inline unsigned __activemask() { return 1u; }
static inline unsigned __ballot_sync(unsigned, bool p) { return p ? 1u : 0u; }
static inline unsigned __reduce_min_sync(unsigned, unsigned v) { return v; }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __ffs(unsigned x) { return __builtin_ffs((int)x); }
static inline unsigned atomicCAS(unsigned* p, unsigned cmp, unsigned v) { unsigned o = *p; if (o == cmp) *p = v; return o; }
static inline unsigned atomicOr(unsigned* p, unsigned v) { unsigned o = *p; *p = o | v; return o; }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p = o + v; return o; }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { unsigned long long o = *p; *p = o + v; return o; }
static inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) { unsigned long long o = *p; if (v < o) *p = v; return o; }
'''

DRIVER = r'''
unsigned nbsh[2 * 4096];   // the private bins of the one CTA (two words each)
extern "C" void run(const unsigned* const* cols, unsigned mode, unsigned comp, const unsigned* tbase, unsigned* slots, unsigned* keys, unsigned kw,
                    unsigned mask, unsigned long long* cnt, unsigned nsh, unsigned long long* um, unsigned* err) {
  blockDim.x = 1; threadIdx.x = 0; blockIdx.x = 0; gridDim.x = 1;
  for (unsigned i = 0; i < NB_NMASKS; ++i) ccols[i] = cols[i];
  nbjit(mode, comp, tbase, slots, keys, kw, mask, cnt, nsh, um, err);
}
'''


def machines():
    """Small witnesses: (name, machine, tree-1 host columns in commitment order)."""
    add = M.AddMachine(log_size=8, n_lanes=2)
    cols, mult = add.fill_main_trace(seed=4, n_padding=3)
    multi = M.MultiMachine([4, 5, 8, 6])
    v1 = NexusV1Machine(8)
    kc = KeccakMachine(2, seed=5)
    return [("add", add, list(cols) + [mult]), ("multi", multi, multi.fill_main_trace(seed=2)), ("nexus_v1", v1, v1.fill_main_trace(seed=3)),
            ("keccak", kc, kc.fill_main_trace())]


def load(words):
    w = np.ascontiguousarray(words, dtype=np.uint32)
    h = C.c_void_p()
    assert nb.lib().nb200_air_load(None, w.ctypes.data_as(u32p), C.c_size_t(w.size), C.byref(h)) == 0
    return h


def lookup_tables(h, comp, n):
    kind, rel, arg = (np.zeros(n, np.uint32) for _ in range(3))
    st = nb.lib().nb200_air_lookup_tables(h, C.c_uint32(comp), kind.ctypes.data_as(u32p), rel.ctypes.data_as(u32p), arg.ctypes.data_as(u32p), C.c_size_t(n))
    assert st == 0
    return [(KIND[int(k)], int(r), int(a)) for k, r, a in zip(kind, rel, arg)]


def count_source(h, comp):
    p = C.c_void_p()
    st = nb.lib().nb200_air_count_kernel_source(h, C.c_uint32(comp), C.byref(p))
    if st != 0:
        return st, None
    src = C.string_at(p)
    nb.lib().nb200_free(p)
    return 0, src


def test_classification_pinned_per_machine():
    for name, m, _t1 in machines():
        h = load(m.words)
        want = ref.classify(m.air)
        for k, comp in enumerate(m.air.components):
            got = lookup_tables(h, k, len(comp.fracs))
            exp = [(kind, rel.z, x if kind != "ignored" else len(comp.lookups[i][2])) for i, (kind, rel, x) in enumerate(want[k])]
            assert got == exp, (name, k)
        nb.lib().nb200_air_free(h)
        counts = [[sum(1 for (kd, _r, _x) in row if kd == kind) for kind in ("table", "lookup", "ignored")] for row in want]
        rels = lambda kind: {rel.name for row in want for (kd, rel, _x) in row if kd == kind}
        if name == "nexus_v1":
            main = [(rel.name, kd) for (kd, rel, _x) in want[0]]
            assert main.count(("Range256", "lookup")) == 170 and main.count(("Range32", "lookup")) == 5
            assert counts[1] == [1, 0, 0] and counts[2] == [1, 0, 0]
            assert rels("table") == {"Range256", "Range32"}
            assert rels("ignored") == {"BitOp", "LoadStore", "ProgramCheck", "RegisterCheck", "Range8", "Range16", "Range128"}
            # the is_type_u-gated Range256 lookups have a numerator that is not a constant
            gated = [i for i, (kd, rel, _x) in enumerate(want[0]) if kd == "lookup" and rel.name == "Range256"
                     and m.air.components[0].nodes[m.air.components[0].lookups[i][1].id][0] != "const"]
            assert gated
        if name == "keccak":
            assert [c[0] for c in counts] == [0, 0, 0, 16, 16, 1]
            assert rels("table") == {"KeccakXor", "KeccakBitNotAnd", "KeccakBitRotate"}
            assert rels("ignored") == {"KeccakState", "LoadStore"}
            assert counts[0][1] == 0 and counts[1][1] > 0 and counts[2][1] > 0
            for k in (1, 2):
                assert {rel.name for (kd, rel, _x) in want[k] if kd == "lookup"} == {"KeccakXor", "KeccakBitNotAnd", "KeccakBitRotate"}
        if name == "multi":
            assert rels("table") == {"Range256", "BitOp"} and not rels("ignored")
        if name == "add":
            assert counts == [[0, 24, 0], [1, 0, 0]]


def test_python_reference_equals_the_machines_host_columns():
    for name, m, t1 in machines():
        cols, n_unmatched, _first = ref.multiplicities(m.air, m.preprocessed_columns(), t1)
        host = ref.flat(t1)
        assert n_unmatched == 0, name
        assert cols and all(np.array_equal(v, host[c]) for c, v in cols.items()), name


def host_build(path, source):
    src = source.decode()
    asm = 'asm("mad.wide.u32 %0, %1, 2, %2;" : "=l"(y) : "r"((u32)(x >> 32)), "l"((u64)(u32)x));'
    assert src.count(asm) == 1, "the generated prelude changed: update the host shim of this test"
    src = src.replace(asm, "y = (u64)(u32)(x >> 32) * 2ull + (u64)(u32)x;")
    cu = path / "count_host.cc"
    cu.write_text(SHIM + src + DRIVER)
    so = path / "count_host.so"
    subprocess.run(["/usr/bin/g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-w", str(cu), "-o", str(so)], check=True)
    return C.CDLL(str(so))


def host_count(tmp_path, m, t1):
    """The library's orchestration (prove.cu table_multiplicities) with the host-compiled kernels: {tree-1 column: finalized column}, um."""
    h = load(m.words)
    trees = [[orc.finalize_column(c) for c in ref.flat(m.preprocessed_columns())], [orc.finalize_column(c) for c in ref.flat(t1)]]
    kinds = [lookup_tables(h, k, len(comp.fracs)) for k, comp in enumerate(m.air.components)]
    bins, tbase, cols_of = 0, {}, []
    for k, comp in enumerate(m.air.components):
        tbase[k] = []
        for kind, _r, col in kinds[k]:
            if kind == "table":
                tbase[k].append(bins)
                cols_of.append((col, bins, 1 << comp.log_size))
                bins += 1 << comp.log_size
    kw = 2 + max(len(comp.lookups[i][2]) for k, comp in enumerate(m.air.components) for i, (kd, _r, _c) in enumerate(kinds[k]) if kd == "table")
    cap = 1024
    while cap < 2 * bins:
        cap *= 2
    slots = np.full(cap, 0xFFFFFFFF, np.uint32)
    keys = np.zeros(bins * kw, np.uint32)
    cnt = np.zeros(bins, np.uint64)
    um = np.array([0, (1 << 64) - 1], np.uint64)
    err = np.zeros(1, np.uint32)
    nsh = bins if bins <= 4096 else 0   # private (shared-memory) bins as the library chooses them: ADD and v1 here
    libs = {}
    for k, comp in enumerate(m.air.components):
        st, src = count_source(h, k)
        if st:
            assert st == 6 and not any(kd in ("table", "lookup") for kd, _r, _c in kinds[k])
            continue
        (tmp_path / str(k)).mkdir()
        libs[k] = host_build(tmp_path / str(k), src)
    nb.lib().nb200_air_free(h)

    def run(k, mode):
        comp = m.air.components[k]
        cols = [np.ascontiguousarray(trees[t][c]) if t < 2 else np.zeros(1 << comp.log_size, np.uint32) for (t, c, _o) in comp.masks]
        ptrs = (u32p * max(len(cols), 1))(*[c.ctypes.data_as(u32p) for c in cols])
        tb = np.array(tbase[k] or [0], np.uint32)
        libs[k].run(ptrs, C.c_uint32(mode), C.c_uint32(k), tb.ctypes.data_as(u32p), slots.ctypes.data_as(u32p), keys.ctypes.data_as(u32p),
                    C.c_uint32(kw), C.c_uint32(cap - 1), cnt.ctypes.data_as(u64p), C.c_uint32(nsh if mode else 0), um.ctypes.data_as(u64p),
                    err.ctypes.data_as(u32p))

    for k in libs:
        if tbase[k]:
            run(k, 0)
    assert err[0] == 0
    for k in libs:
        if any(kd == "lookup" for kd, _r, _c in kinds[k]):
            run(k, 1)
    out = {col: (cnt[b:b + n] % np.uint64(P)).astype(np.uint32) for col, b, n in cols_of}
    return out, trees, um, err


@pytest.mark.parametrize("name", ["add", "multi", "nexus_v1", "keccak"])
def test_host_compiled_count_kernel_equals_the_host_columns(tmp_path, name):
    (_n, m, t1), = [x for x in machines() if x[0] == name]
    out, trees, um, _err = host_count(tmp_path, m, t1)
    assert int(um[0]) == 0 and int(um[1]) == (1 << 64) - 1
    assert out
    for col, v in out.items():
        assert np.array_equal(v, trees[1][col]), (name, col)


def test_host_compiled_count_kernel_reports_the_first_unmatched_lookup(tmp_path):
    """A Range256-checked limb of 256 on one row: one unmatched lookup, named by component, fraction and trace row."""
    m = NexusV1Machine(8)
    t1 = [c.copy() for c in m.fill_main_trace(seed=3)]
    want_cols, _n, _f = ref.multiplicities(m.air, m.preprocessed_columns(), t1)
    kinds = ref.classify(m.air)[0]
    i = next(i for i, (kd, rel, _x) in enumerate(kinds) if kd == "lookup" and rel.name == "Range256"
             and m.air.components[0].nodes[m.air.components[0].lookups[i][1].id][0] == "const")
    (t, col, _o), = ref._leaves(m.air.components[0], m.air.components[0].lookups[i][2][0])
    assert t == 1
    t1[col][37] = 256
    cols, n_unmatched, first = ref.multiplicities(m.air, m.preprocessed_columns(), t1)
    assert n_unmatched == 1 and first == (0, i, 37)
    out, _trees, um, _err = host_count(tmp_path, m, t1)
    assert int(um[0]) == 1 and int(um[1]) == (0 << 48) | (i << 28) | 37
    for c, v in cols.items():
        assert np.array_equal(out[c], orc.finalize_column(v))


def test_count_source_and_key():
    """The count source exists exactly where a component has a table or a lookup, and its cache key differs from the other variants'."""
    m = M.MultiMachine([4, 5, 8])
    lib = nb.lib()
    lib.nb200_kernel_source_key.restype = C.c_uint64
    lib.nb200_kernel_source_key.argtypes = [C.c_char_p]
    h = load(m.words)
    for k in range(len(m.air.components)):
        st, src = count_source(h, k)
        assert st == 0 and src.startswith(b"// table multiplicities")
        others = []
        for which in range(4):
            p = C.c_void_p()
            if lib.nb200_air_kernel_source(h, C.c_uint32(k), C.c_int(which), C.byref(p)) == 0:
                others.append(C.string_at(p))
                lib.nb200_free(p)
        assert len({lib.nb200_kernel_source_key(s) for s in others + [src]}) == len(others) + 1
    nb.lib().nb200_air_free(h)
    kc = KeccakMachine(2)
    h = load(kc.words)
    assert count_source(h, 0)[0] == 6                     # the memory check: State and LoadStore only, no table
    nb.lib().nb200_air_free(h)


def test_host_compiled_count_kernel_on_a_full_entropy_witness(tmp_path):
    """Random tree-1 values (half uniform in [0, P), the rest P - 1, 0, 1, bytes, 16-bit values): numerators near 2^31 carry out of the low
    word of a private bin many times; the columns and the unmatched report equal the reference's."""
    from tests.random_witness import mixed
    m = NexusV1Machine(8)
    rng = np.random.default_rng(8)
    t1 = [mixed(rng, len(c)) for c in ref.flat(m.fill_main_trace(seed=8))]
    cols, n_want, first_want = ref.multiplicities(m.air, m.preprocessed_columns(), t1)
    assert n_want > 0
    out, _trees, um, _err = host_count(tmp_path, m, t1)
    k, i, r = first_want
    assert int(um[0]) == n_want and int(um[1]) == (k << 48) | (i << 28) | r
    for c, v in cols.items():
        assert np.array_equal(out[c], orc.finalize_column(v)), c
