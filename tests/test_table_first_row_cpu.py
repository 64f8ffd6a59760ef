"""The first-row table count (nb200_table_multiplicities_first_row) WITHOUT a GPU: the generated count kernels (nb200_air_count_kernel_source)
and the resolve (csrc/table_first_row.cuh) compiled as host C++ and run in the library's order (build, resolve, probe) on the whole machine,
whose Range8 table lists the value 0 nine times.  The build's slot winners are scrambled among the rows of their tuple and the bins claim
in shuffled order, as racing threads would; the columns must still equal the host fill's and the numpy first-row reference's.  Also: the
resolve hashes and compares keys exactly as the generated source does, and its kernels compile for sm_90a without spills."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import whole_machine as W
from oracle import pyoracle as orc
from tests import table_mult_ref as ref
from tests.random_witness import mixed
from tests.test_table_multiplicities_cpu import count_source, host_build, load, lookup_tables

P = (1 << 31) - 1
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "nexus_zkvm_b200", "csrc")
NVCC = os.environ.get("NB200_NVCC", "/usr/local/cuda/bin/nvcc")
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)

RESOLVE = r'''
#include "table_first_row.cuh"
using namespace nb;
// the claim kernel over the bins in the order given, then the slot kernel; returns the occupied slots
extern "C" u32 resolve(u32* slots, const u32* keys, u32 kw, u64 cap, const u32* tables, u32 n_tables, const u32* bins, u32 n_bins, u64* owner) {
  for (u64 s = 0; s < cap; ++s) owner[s] = ~0ull;
  for (u32 i = 0; i < n_bins; ++i) {
    u64* o = owner + first_row::key_slot(slots, keys, kw, (u32)(cap - 1), bins[i]);
    const u64 claim = first_row::first_row_claim(tables, n_tables, bins[i]);
    if (claim < *o) *o = claim;
  }
  u32 distinct = 0;
  for (u64 s = 0; s < cap; ++s) distinct += first_row::own_slot(slots, owner, s);
  return distinct;
}
extern "C" u32 key_hash(u32 rel, u32 len, const u32* v) { return first_row::key_hash(rel, len, v); }
extern "C" int key_same(const u32* k, u32 rel, u32 len, const u32* v) { return first_row::key_same(k, rel, len, v); }
'''

# appended to a generated count source: its own hash and key comparisons
GENERATED_HASH = rb'''
extern "C" unsigned gen_hash(unsigned rel, unsigned len, const unsigned* v) { return khash(rel, len, v); }
extern "C" int gen_same(const unsigned* k, unsigned rel, unsigned len, const unsigned* v) { return (ksame(k, rel, len, v) ? 1 : 0) | (ksame_cg(k, rel, len, v) ? 2 : 0); }
'''


def first_row_reference(air, tree0, tree1):
    """numpy: ({tree-1 column of a table fraction: multiplicities mod P, trace order}, n_unmatched, first unmatched or None, n_repeated), a
    tuple listed by several table rows of one relation counted on the first of them in (component, fraction, trace row) order."""
    trees = [ref.flat(tree0), ref.flat(tree1)]
    kinds = ref.classify(air)
    tables = {}   # (id(relation), tuple length) -> [(values (rows, len), column)], component and fraction order
    for k, comp in enumerate(air.components):
        for i, (kind, rel, col) in enumerate(kinds[k]):
            if kind == "table":
                vals = np.stack([ref.evaluate(comp, v, trees) for v in comp.lookups[i][2]], axis=1)
                tables.setdefault((id(rel), vals.shape[1]), []).append((vals, col))
    out = {col: np.zeros(len(v), np.int64) for ts in tables.values() for (v, col) in ts}
    owners, n_repeated = {}, 0
    for key, ts in tables.items():
        keys = ref._rows_key(np.concatenate([v for v, _c in ts]))
        uniq, first = np.unique(keys, return_index=True)          # the first index of each tuple, in (component, fraction, row) order
        n_repeated += len(keys) - len(uniq)
        col_of = np.concatenate([np.full(len(v), c) for v, c in ts])
        row_of = np.concatenate([np.arange(len(v)) for v, _c in ts])
        owners[key] = (uniq, col_of[first], row_of[first])
    n_unmatched, first_bad = 0, None
    for k, comp in enumerate(air.components):
        for i, (kind, rel, _x) in enumerate(kinds[k]):
            if kind != "lookup":
                continue
            _rel, num, vals = comp.lookups[i]
            nv = ref.evaluate(comp, num, trees)
            lv = np.stack([ref.evaluate(comp, v, trees) for v in vals], axis=1)
            hit = np.zeros(len(nv), bool)
            if (id(rel), lv.shape[1]) in owners:
                uniq, cols, rows = owners[(id(rel), lv.shape[1])]
                lk = ref._rows_key(lv)
                pos = np.minimum(np.searchsorted(uniq, lk), len(uniq) - 1)
                hit = uniq[pos] == lk
                for c in np.unique(cols[pos[hit]]):
                    sel = hit.copy()
                    sel[hit] = cols[pos[hit]] == c
                    np.add.at(out[int(c)], rows[pos[sel]], nv[sel])
            bad = np.nonzero(~hit & (nv != 0))[0]
            if len(bad):
                n_unmatched += len(bad)
                if first_bad is None:
                    first_bad = (k, i, int(bad[0]))
    return {c: (v % P).astype(np.uint32) for c, v in out.items()}, n_unmatched, first_bad, n_repeated


@pytest.fixture(scope="module")
def whole():
    return W.NexusV1KeccakMachine(8, 15, seed=1)


@pytest.fixture(scope="module")
def kernels(whole, tmp_path_factory):
    """({component: its host-compiled count kernel}, the host-compiled resolve)."""
    d = tmp_path_factory.mktemp("first_row")
    h = load(whole.words)
    libs = {}
    for k in range(len(whole.air.components)):
        st, src = count_source(h, k)
        if st == 0:
            (d / str(k)).mkdir()
            libs[k] = host_build(d / str(k), src)
    nb.lib().nb200_air_free(h)
    src, so = d / "resolve.cc", d / "resolve.so"
    src.write_text(RESOLVE)
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-w", "-I", CSRC, str(src), "-o", str(so)], check=True)
    res = C.CDLL(str(so))
    res.resolve.restype = C.c_uint32
    res.key_hash.restype = C.c_uint32
    return libs, res


def scramble(slots, keys, kw, rng):
    """Each occupied slot gets a random bin of its key, as if another of the key's rows had won the build's race."""
    k2 = keys.reshape(-1, kw)
    _u, inv = np.unique(ref._rows_key(k2.astype(np.int64)), return_inverse=True)
    order = np.argsort(inv, kind="stable")
    start = np.searchsorted(inv[order], np.arange(inv.max() + 1))
    size = np.diff(np.append(start, len(inv)))
    pick = order[start + (rng.random(len(size)) * size).astype(np.int64)]
    occ = slots != 0xFFFFFFFF
    slots[occ] = pick[inv[slots[occ]]].astype(np.uint32)


def host_first_row_count(kernels, m, t1, seed):
    """nb200_table_multiplicities_first_row's steps with the host-compiled kernels: ({tree-1 column: finalized column}, um, n_repeated,
    slots after the resolve, keys, key width, [(column, first bin, log size)] in bin order)."""
    libs, res = kernels
    h = load(m.words)
    trees = [[orc.finalize_column(c) for c in ref.flat(m.preprocessed_columns())], [orc.finalize_column(c) for c in ref.flat(t1)]]
    kinds = [lookup_tables(h, k, len(comp.fracs)) for k, comp in enumerate(m.air.components)]
    nb.lib().nb200_air_free(h)
    bins, tbase, cols_of = 0, {}, []
    for k, comp in enumerate(m.air.components):
        tbase[k] = []
        for kind, _r, col in kinds[k]:
            if kind == "table":
                tbase[k].append(bins)
                cols_of.append((col, bins, comp.log_size))
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
    nsh = bins if bins <= 4096 else 0

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
    rng = np.random.default_rng(seed)
    scramble(slots, keys, kw, rng)
    tables = np.array([x for _c, b, ls in cols_of for x in (b, ls)], np.uint32)
    order = rng.permutation(bins).astype(np.uint32)
    owner = np.zeros(cap, np.uint64)
    distinct = res.resolve(slots.ctypes.data_as(u32p), keys.ctypes.data_as(u32p), C.c_uint32(kw), C.c_uint64(cap), tables.ctypes.data_as(u32p),
                           C.c_uint32(len(cols_of)), order.ctypes.data_as(u32p), C.c_uint32(bins), owner.ctypes.data_as(u64p))
    for k in libs:
        if any(kd == "lookup" for kd, _r, _c in kinds[k]):
            run(k, 1)
    out = {col: (cnt[b:b + (1 << ls)] % np.uint64(P)).astype(np.uint32) for col, b, ls in cols_of}
    return out, um, bins - int(distinct), slots, keys, kw, cols_of


def _range8(m):
    """(tree-1 column, relation index) of Multiplicity8's table fraction."""
    (kind, rel, col), = ref.classify(m.air)[4]
    assert kind == "table" and rel.name == "Range8"
    return col, rel.z


@pytest.mark.parametrize("seed", [1, 2])
def test_whole_machine_first_row_count_equals_the_host_columns(kernels, whole, seed):
    m = whole
    t1 = [c.copy() for c in ref.flat(m.fill_main_trace())]
    host = [c.copy() for c in t1]
    rng = np.random.default_rng(seed)
    table_cols = sorted({col for row in ref.classify(m.air) for (kind, _r, col) in row if kind == "table"})
    for c in table_cols:                                                  # the count must not read what the columns held
        t1[c] = rng.integers(0, 1 << 32, len(t1[c]), dtype=np.uint64).astype(np.uint32)
    out, um, n_repeated, slots, keys, kw, cols_of = host_first_row_count(kernels, m, t1, seed)
    assert int(um[0]) == 0 and n_repeated == 8
    assert sorted(out) == table_cols
    for c, v in out.items():
        assert np.array_equal(v, orc.finalize_column(host[c])), c
    want, n_unmatched, _first, ref_repeated = first_row_reference(m.air, m.preprocessed_columns(), host)
    assert n_unmatched == 0 and ref_repeated == 8
    for c, v in want.items():
        assert np.array_equal(v, host[c]), c
    # the slot of the key (Range8, 0) names the bin of trace row 0 (finalized position 0) of Multiplicity8's table
    col, z = _range8(m)
    (b8,) = [b for c, b, _ls in cols_of if c == col]
    k2 = keys.reshape(-1, kw)
    rows0 = [b for b in range(b8, b8 + 16) if k2[b, 0] == z and k2[b, 1] == 1 and k2[b, 2] == 0]
    assert len(rows0) == 9
    assert np.count_nonzero(slots == b8) == 1 and not np.isin(slots, [b for b in rows0 if b != b8]).any()


def test_whole_machine_first_row_count_on_a_full_entropy_main_witness(kernels, whole):
    """The main component's columns random (bytes, 16-bit values, 0, 1, P - 1, uniform): its Range8 lookups of 0 fire, and their count
    lands on Multiplicity8's trace row 0 alone; columns and the unmatched report equal the numpy first-row reference's."""
    m = whole
    t1 = [c.copy() for c in ref.flat(m.fill_main_trace())]
    rng = np.random.default_rng(3)
    n_main = sum(1 for (t, _c, _o) in m.air.components[0].masks if t == 1)
    for c in range(n_main):
        t1[c] = mixed(rng, len(t1[c]))
    want, n_want, first_want, _rep = first_row_reference(m.air, m.preprocessed_columns(), t1)
    assert n_want > 0
    out, um, n_repeated, *_rest = host_first_row_count(kernels, m, t1, 4)
    k, i, r = first_want
    assert int(um[0]) == n_want and int(um[1]) == (k << 48) | (i << 28) | r
    assert n_repeated == 8
    col, _z = _range8(m)
    assert want[col][0] > 0 and not want[col][8:].any()
    for c, v in want.items():
        assert np.array_equal(out[c], orc.finalize_column(v)), c


def test_resolve_hash_and_key_comparison_equal_the_generated_source(kernels, whole, tmp_path):
    _libs, res = kernels
    h = load(whole.words)
    st, src = count_source(h, 4)                                          # Multiplicity8's count source
    nb.lib().nb200_air_free(h)
    assert st == 0
    gen = host_build(tmp_path, src + GENERATED_HASH)
    gen.gen_hash.restype = C.c_uint32
    rng = np.random.default_rng(11)
    for length in (0, 1, 2, 3, 4, 5, 8, 17, 200):
        for _ in range(40):
            rel = int(rng.integers(0, 1 << 32))
            v = rng.integers(0, 1 << 32, max(length, 1), dtype=np.uint64).astype(np.uint32)
            if rng.random() < 0.5:
                v %= np.uint32(P)
            vp = v.ctypes.data_as(u32p)
            assert res.key_hash(C.c_uint32(rel), C.c_uint32(length), vp) == gen.gen_hash(C.c_uint32(rel), C.c_uint32(length), vp)
            key = np.concatenate([np.array([rel, length], np.uint32), v[:length]])
            cases = [key.copy()]
            for j in range(len(key)):                                     # one word different: relation, length or a value
                bad = key.copy()
                bad[j] ^= np.uint32(1 << int(rng.integers(0, 32)))
                cases.append(bad)
            for k in cases:
                kp = k.ctypes.data_as(u32p)
                want = res.key_same(kp, C.c_uint32(rel), C.c_uint32(length), vp)
                assert gen.gen_same(kp, C.c_uint32(rel), C.c_uint32(length), vp) == 3 * want
                assert want == (k is cases[0])


def test_resolve_kernels_compile_for_sm90a_without_spills(tmp_path):
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++", "-Xcudafe",
                        "--diag_suppress=177", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-x", "cu", "-c",
                        os.path.join(CSRC, "table_first_row.cu"), "-o", str(tmp_path / "table_first_row.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    blocks = re.split(r"Compiling entry function '", r.stderr)[1:]
    ours = {b.split("'")[0]: b for b in blocks}
    for k in ("table_first_row_claim_kernel", "table_first_row_slot_kernel"):
        (name,) = [n for n in ours if k in n]
        spills = [int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", ours[name])]
        assert spills and max(spills) == 0, (k, ours[name])
