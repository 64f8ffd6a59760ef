"""The keccak precompile extension recorded as data (nexus_zkvm_b200/keccak.py) without a GPU: the permutation against hashlib, the witness
against every constraint of the six components (the oracle's check and the numpy restatement in tests/constraint_ref.py), the LogUp balance
of the State / Xor / BitNotAnd / BitRotate relations, the generated kernels of every component compiled for sm_90a, and an oracle proof that
its verifier accepts."""
import ctypes as C
import hashlib
import os
import re
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import field as F
from nexus_zkvm_b200 import keccak as K
from nexus_zkvm_b200 import machine as M
from tests import oracle_check
from tests.oracle_backend import OracleBackend, verify

P = (1 << 31) - 1
u32p = C.POINTER(C.c_uint32)
NVCC = os.environ.get("NB200_NVCC", "/usr/local/cuda/bin/nvcc")
# the largest local-memory spill (stores or loads, bytes, any function of the kernel) that `nvcc -Xptxas -v` may report for a generated
# keccak kernel (DESIGN §4, keccak row)
MAX_SPILL_BYTES = 2048


def _single_block(msg, rate, pad):
    """The padded block of a one-block message XORed into the zero state, as (25, 1) uint64 lanes."""
    blk = bytearray(msg) + bytes([pad]) + bytes(rate - len(msg) - 1)
    blk[-1] |= 0x80
    st = np.zeros((25, 1), np.uint64)
    for i in range(rate // 8):
        st[i, 0] = int.from_bytes(blk[8 * i:8 * i + 8], "little")
    return st


def _squeeze(st, n):
    return b"".join(int(st[i, 0]).to_bytes(8, "little") for i in range(25))[:n]


@pytest.mark.parametrize("msg", [b"", b"abc", bytes(range(135))])
def test_permutation_matches_hashlib(msg):
    assert _squeeze(K.keccak_f(_single_block(msg, 136, 0x06)), 32) == hashlib.sha3_256(msg).digest()
    assert _squeeze(K.keccak_f(_single_block(msg[:167], 168, 0x1F)), 64) == hashlib.shake_128(msg[:167]).digest(64)


def test_air_shape():
    """Component order, sizes, fractions and columns of keccak_extensions() (class docstring of KeccakMachine)."""
    m = K.KeccakMachine(6)
    assert m.log_sizes == [6, 10, 9, 12, 12, 11]
    assert [len(c.fracs) for c in m.air.components] == [2 + 2 * 200, 1042, 1042, 16, 16, 1]
    assert [c.log_expand for c in m.air.components] == [1] * 6
    # 2 states, 3 x 400 limbs, 2 x 200 carries, is_padding | 213 lanes + is_padding (x 2) | 16 + 16 + 1 multiplicities
    assert m.air.n_columns() == [1 + 2 * 9 + 4 + 4, 2001 + 2 * 1705 + 33, 4 * (201 + 2 * 521 + 8 + 8 + 1)]
    assert [r.size for r in m.relations] == [5, 3, 3, 200, 4]


@pytest.fixture(scope="module")
def small():
    m = K.KeccakMachine(4, seed=3)
    return m, m.fill_main_trace()


def test_witness_satisfies_every_constraint(small):
    m, t1 = small
    report, _balanced = M.check_constraints(m, oracle_check.OracleCheckBackend(), t1, None)
    assert set(report) == set(range(6)) and not any(report.values()), report
    # every row of every component holds a full round: the round components' outputs are the permutation's
    assert np.array_equal(m.outputs, K.keccak_f(m.inputs))


def test_one_flipped_byte_is_caught(small):
    """A byte of a rotation's output lane in round 0 breaks exactly that rotation constraint at that row; a byte of the round's output
    state (a chi XOR) satisfies every constraint once the interaction trace is regenerated, but the Xor and State sums no longer balance."""
    m, t1 = small
    rnd = m.air.components[1]
    row = 37
    # the first rotation (theta: rot(C[1], 1)) allocates its low / high / out lanes after the input state and C's 20 XOR lanes
    out_lane = (25 + 20 + 2) * K.LANE_SIZE
    bad = [b.copy() for b in t1]
    bad[1][out_lane + 3, row] ^= 1
    report, _ = M.check_constraints(m, oracle_check.OracleCheckBackend(), bad, None)
    assert not any(report[k] for k in (0, 2, 3, 4, 5))
    (k, degree, n_rows, first), = report[1]
    assert (degree, n_rows, first) == (1, 1, row)
    assert k == 3                               # rotate_left's constraint for byte 3 of the first rotated lane
    # a byte of the output state (the iota XOR's result: the last lane before is_padding)
    bad = [b.copy() for b in t1]
    bad[1][-1 - K.LANE_SIZE, row] ^= 0x10
    report, _ = M.check_constraints(m, oracle_check.OracleCheckBackend(), bad, None)
    assert not any(report.values())
    _proof, claimed, aux = M.prove(m, OracleBackend(), t1, None)
    total = _sum(claimed)
    assert total == m.net_load_store(aux["params"])
    ch, prover, params, claimed_bad, _roots, _ls = M._commit_trees(m, OracleBackend(), bad, None, None, b"", None)
    assert _sum(claimed_bad) != m.net_load_store(params)


def _sum(claimed):
    tot = (0, 0, 0, 0)
    for c in claimed:
        tot = F.qm31_add(tot, c)
    return tot


def test_oracle_proves_and_verifies_and_sums_balance(small):
    """The oracle proves the machine and its verifier accepts; the sum of the six claimed sums is the memory check's net LoadStore
    contribution recomputed from the side note alone, so State, Xor, BitNotAnd and BitRotate balance."""
    m, t1 = small
    proof, claimed, aux = M.prove(m, OracleBackend(), t1, None, associated_data=b"kc")
    verify(m, proof, aux)
    assert _sum(claimed) == m.net_load_store(aux["params"])
    assert not M.verify_claimed_sums(claimed)     # the LoadStore side is the main component's (KeccakChip), not part of this machine


def _kernel_source(words, comp, which):
    w = np.ascontiguousarray(words, dtype=np.uint32)
    h = C.c_void_p()
    assert nb.lib().nb200_air_load(None, w.ctypes.data_as(u32p), C.c_size_t(w.size), C.byref(h)) == 0
    src = C.c_void_p()
    st = nb.lib().nb200_air_kernel_source(h, C.c_uint32(comp), C.c_int(which), C.byref(src))
    out = C.string_at(src) if st == 0 else None
    if st == 0:
        nb.lib().nb200_free(src)
    nb.lib().nb200_air_n_constraints.restype = C.c_uint32
    n = int(nb.lib().nb200_air_n_constraints(h, C.c_uint32(comp)))
    deg = np.zeros(max(n, 1), np.uint32)
    assert nb.lib().nb200_air_constraint_degrees(h, C.c_uint32(comp), deg.ctypes.data_as(u32p), C.c_size_t(n)) == 0
    nb.lib().nb200_air_free(h)
    return st, out, int(deg[:n].max())


def _ptxas(src, tmp, name):
    cu = tmp / f"{name}.cu"
    cu.write_bytes(src)
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++", "-cubin",
                        "-Xptxas", "-v", str(cu), "-o", str(tmp / f"{name}.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    spills = [int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", r.stderr)]
    return max(spills or [0])


@pytest.mark.slow
def test_every_kernel_source_compiles_for_sm90a_without_spills(tmp_path):
    """nb200_air_kernel_source gives the constraint (0), LogUp (1) and check (3) kernels of every component, the D2 kernel (2) exactly where
    a constraint has degree above 2, and each compiles for sm_90a with no more local-memory spill than DESIGN §4 states.  BitRotateTable's
    one-fraction program is too short to specialise (NB200_ERR_STATE: the bytecode interpreter runs it) except for the check."""
    m = K.KeccakMachine(6)
    jobs = []
    for comp in range(len(m.air.components)):
        for which in (0, 1, 2, 3):
            st, src, max_deg = _kernel_source(m.words, comp, which)
            if which == 2 and max_deg <= 2:
                assert st != 0, comp
                continue
            if comp == 5 and which != 3:
                assert st == 6, (comp, which)
                continue
            assert st == 0 and src, (comp, which)
            jobs.append((f"c{comp}w{which}", src))
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        spills = dict(zip([n for n, _ in jobs], ex.map(lambda j: _ptxas(j[1], tmp_path, j[0]), jobs)))
    assert all(v <= MAX_SPILL_BYTES for v in spills.values()), sorted(spills.items())
