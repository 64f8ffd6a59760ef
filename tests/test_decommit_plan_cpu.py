"""The decommitment walk planned on the host (nb200_merkle_decommit_plan), which the prover runs for every tree before ONE gather of
everything the walks name: the values and hashes it points at, read from the oracle's own columns and tree, must be exactly the oracle's
MerkleProver::decommit output, in order.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from oracle import pyoracle as orc

P = (1 << 31) - 1
u32p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)


def plan(max_log, logs, queries):
    L = nb.lib()
    logs = np.asarray(logs, dtype=np.uint32)
    ks = sorted(queries)
    qls = np.array(ks, dtype=np.uint32)
    cnt = np.array([len(queries[k]) for k in ks], dtype=np.uint64)
    pos = np.array([p for k in ks for p in queries[k]], dtype=np.uint64)
    vp, hp = u64p(), u64p()
    nv, nh = C.c_size_t(), C.c_size_t()
    st = L.nb200_merkle_decommit_plan(C.c_uint32(max_log), logs.ctypes.data_as(u32p), C.c_size_t(logs.size), qls.ctypes.data_as(u32p),
                                      cnt.ctypes.data_as(u64p), pos.ctypes.data_as(u64p), C.c_size_t(len(ks)),
                                      C.byref(vp), C.byref(nv), C.byref(hp), C.byref(nh))
    assert st == 0
    vals = np.ctypeslib.as_array(vp, shape=(max(3 * nv.value, 1),))[:3 * nv.value].reshape(-1, 3).copy()
    hashes = np.ctypeslib.as_array(hp, shape=(max(2 * nh.value, 1),))[:2 * nh.value].reshape(-1, 2).copy()
    L.nb200_free(C.cast(vp, C.c_void_p)); L.nb200_free(C.cast(hp, C.c_void_p))
    return vals, hashes


CASES = {
    "one size": ([6] * 5, {6: [0, 1, 7, 33, 63]}),
    "mixed sizes, shuffled": ([5, 7, 3, 7, 5, 2, 7, 3], {7: [3, 4, 100], 5: [1, 30], 3: [6], 2: [0, 3]}),
    "queries at the largest size only": ([9, 9, 4, 4, 1], {9: [0, 17, 18, 19, 511]}),
    "fri-layer shaped": ([10] * 4, {10: [2, 3, 500, 501, 1022, 1023]}),
    "first-layer shaped": ([8] * 4 + [6] * 4 + [3] * 4, {8: [10, 11, 200, 201], 6: [2, 3, 50, 51], 3: [0, 1, 6, 7]}),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_plan_names_what_the_oracle_decommitment_holds(name):
    logs, queries = CASES[name]
    rng = np.random.default_rng(len(name))
    cols = [rng.integers(0, P, 1 << l, dtype=np.uint32) for l in logs]
    max_log = max(logs)
    _root, layers = orc.merkle_commit(cols, want_layers=True)
    o_qv, o_hw, o_cw = orc.merkle_decommit(cols, queries)
    vals, hashes = plan(max_log, logs, queries)
    got = [int(cols[c][r]) for c, r, _q in vals]
    assert [v for v, (_c, _r, q) in zip(got, vals) if q] == [int(x) for x in o_qv]
    assert [v for v, (_c, _r, q) in zip(got, vals) if not q] == [int(x) for x in o_cw]
    node = lambda l, i: bytes(layers[32 * ((1 << l) - 1 + i):32 * ((1 << l) + i)])
    assert [node(int(l), int(i)) for l, i in hashes] == o_hw


def test_plan_rejects_a_column_larger_than_the_tree():
    L = nb.lib()
    logs = np.array([5, 6], dtype=np.uint32)
    vp, hp = u64p(), u64p()
    nv, nh = C.c_size_t(), C.c_size_t()
    assert L.nb200_merkle_decommit_plan(C.c_uint32(5), logs.ctypes.data_as(u32p), C.c_size_t(2), None, None, None, C.c_size_t(0),
                                        C.byref(vp), C.byref(nv), C.byref(hp), C.byref(nh)) != 0
