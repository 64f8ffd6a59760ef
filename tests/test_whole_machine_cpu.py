"""The v1 main component, its eight base extensions and the keccak extension as one machine (nexus_zkvm_b200/whole_machine.py) without a GPU:
the recorded shape in the reference's order, an oracle proof that its verifier accepts with claimed sums that cancel, the sums broken by a
wrong final value or counter in RamInitFinal or by a missing init fraction, and RamInitFinal's device fill (csrc/ram_init_final.cuh,
compiled as host C++ behind a driver that runs the kernels' steps in order) equal to the numpy columns on edge side notes."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from nexus_zkvm_b200 import air as A
from nexus_zkvm_b200 import keccak as K
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200 import whole_machine as W
from tests.keccak_side_notes import finalized_src_rows
from tests.oracle_backend import OracleBackend, verify

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "nexus_zkvm_b200", "csrc")
NVCC = os.environ.get("NB200_NVCC", "/usr/local/cuda/bin/nvcc")
RAM0 = 347 + 8 + 3                              # RamInitFinal's first column in tree 1 (after the main component, FinalReg, BitOpMultiplicity)


@pytest.fixture(scope="module")
def small():
    m = W.NexusV1KeccakMachine(8, 15, seed=1)
    return m, m.fill_main_trace()


def test_air_shape(small):
    m, _t1 = small
    assert len(m.air.components) == 15
    assert m.log_sizes == [8, 5, 8, m.ram_log_size, 4, 4, 5, 7, 8] + m.keccak.log_sizes
    assert [r.name for r in m.relations] == ["BitOp", "LoadStore", "KeccakXor", "KeccakBitNotAnd", "KeccakState", "KeccakBitRotate", "ProgramCheck",
                                             "RegisterCheck", "Range8", "Range16", "Range32", "Range128", "Range256"]
    comps = m.air.components
    assert [len(c.constraints) for c in comps[:9]] == [414, 1, 3, 17, 1, 1, 1, 1, 1]
    assert [len(c.fracs) for c in comps[:9]] == [253, 2, 3, 11, 1, 1, 1, 1, 1]
    assert [c.log_expand for c in comps] == [2] + [1] * 14
    keccak_cols = m.keccak.air.n_columns()
    assert keccak_cols == [27, 5444, 5040]
    assert m.air.n_columns() == [27 + 1 + 5 + 8 + 5 + keccak_cols[0], 347 + 8 + 3 + 10 + 5 + keccak_cols[1], 1012 + 4 + 12 + 44 + 20 + keccak_cols[2]]
    # the keccak components are recorded as KeccakMachine records them, only their parameter indices differ
    for c, kc in zip(comps[9:], m.keccak.air.components):
        assert (c.log_size, len(c.constraints), len(c.fracs), c.batching) == (kc.log_size, len(kc.constraints), len(kc.fracs), kc.batching)


def test_memory_simulation_exercises_overlaps_and_carries(small):
    m, _t1 = small
    _inputs, addresses, timestamps, ia, iv = W.memory_simulation(m.n_perms, m.n_buffers, m.seed)
    assert np.array_equal(ia, m.init_addresses) and np.all(np.diff(ia.astype(np.int64)) > 0)
    assert int(timestamps.max()) >= 2                                       # some byte is permuted three times or more
    offsets = np.diff(np.unique(addresses).astype(np.int64))
    assert np.any((offsets < K.STATE_SIZE) & (offsets % 8 != 0))               # buffers overlap at a non-multiple of 8
    assert np.any((addresses.astype(np.int64) & 0xFFFF) > 0xFFFF - K.STATE_SIZE + 1)   # a buffer crosses a 2^16 boundary
    assert m.init_addresses.size == np.unique((addresses[:, None].astype(np.int64) + np.arange(K.STATE_SIZE)).ravel()).size


def _sum(claimed):
    from nexus_zkvm_b200 import field as F
    tot = (0, 0, 0, 0)
    for c in claimed:
        tot = F.qm31_add(tot, c)
    return tot


def test_oracle_proves_and_verifies_and_sums_cancel(small):
    m, t1 = small
    proof, claimed, aux = M.prove(m, OracleBackend(), t1, None, associated_data=b"whole")
    verify(m, proof, aux)
    assert len(claimed) == 15
    assert M.verify_claimed_sums(claimed)


def _claimed(m, t1):
    return M._commit_trees(m, OracleBackend(), t1, None, None, b"", None)[3]


@pytest.mark.parametrize("col", [5, 6, 9])
def test_a_wrong_final_value_or_counter_breaks_the_sums(small, col):
    """One final value (column 5) or final counter byte (6, 9) of RamInitFinal changed at one row, with Range256's multiplicities recounted
    so that only the LoadStore relation can be off."""
    m, t1 = small
    ram = m.ram_init_final_columns()
    ram[col, 3] = (ram[col, 3] + 1) % 256
    _main, h256, h32 = m._main_and_hist(0)
    bad = list(t1)
    bad[347:347 + 11 + W.RAM_COLS + 5] = m.base_extension_columns(h256, h32, ram)
    assert not np.array_equal(bad[RAM0 + col], t1[RAM0 + col])
    assert not M.verify_claimed_sums(_claimed(m, bad))


def test_dropping_the_init_fraction_breaks_the_sums(small, monkeypatch):
    m, t1 = small

    def without_init(air, log_size, rel_ls, rel256):
        c = air.component(log_size, 1)
        for n in W.RAM_PREPROCESSED:
            c.get_preprocessed_column(n)
        addr = [c.next_trace_mask() for _ in range(4)]
        flag, final_value = c.next_trace_mask(), c.next_trace_mask()
        counter = [c.next_trace_mask() for _ in range(4)]
        c.add_to_relation(rel_ls, -flag, [addr[0] + addr[1] * 256, addr[2] + addr[3] * 256, final_value, counter[0] + counter[1] * 256,
                                          counter[2] + counter[3] * 256])
        for v in addr + [final_value] + counter:
            c.add_to_relation(rel256, 1, [v])
        c.finalize_logup()
        return c

    monkeypatch.setattr(W, "_ram_init_final_component", without_init)
    m2 = W.NexusV1KeccakMachine(8, 15, seed=1)
    assert len(m2.air.components[3].fracs) == 10
    assert not M.verify_claimed_sums(_claimed(m2, t1))


DRIVER = r'''
#include "ram_init_final.cuh"
#include <algorithm>
#include <vector>
using namespace nb;
// the steps of nb200_ram_init_final_trace in order: keys, sort, run heads and their inclusive scan, each row's last element, the rows
extern "C" u32 ram_fill_host(u32 n_perms, const u64* inputs, const u32* addresses, const u32* timestamps, u32 n_init, const u32* init_addresses,
                             const uint8_t* init_values, u32 log_size, u32* out) {
  const u32 n_acc = n_perms * keccak::STATE, n = n_acc + n_init;
  std::vector<std::pair<u64, u32>> kv(n);
  for (u32 e = 0; e < n; ++e) kv[e] = {ram::access_key(addresses, init_addresses, n_acc, e), e};
  std::sort(kv.begin(), kv.end());
  std::vector<u32> rank(n);
  for (u32 e = 0, acc = 0; e < n; ++e) {
    acc += (e == 0 || ram::key_address(kv[e].first) != ram::key_address(kv[e - 1].first));
    rank[e] = acc;
  }
  const u32 n_rows = n ? rank[n - 1] : 0;
  if (n_rows > (1u << log_size)) return n_rows;
  std::vector<u32> row_src(1u << log_size);
  for (u32 e = 0; e < n; ++e)
    if (e + 1 == n || ram::key_address(kv[e].first) != ram::key_address(kv[e + 1].first)) row_src[rank[e] - 1] = kv[e].second;
  std::vector<u64> outputs((size_t)n_perms * 25);
  for (u32 p = 0; p < n_perms; ++p) {
    u64 a[25];
    for (int k = 0; k < 25; ++k) a[k] = inputs[(size_t)p * 25 + k];
    ram::keccak_f(a);
    for (int k = 0; k < 25; ++k) outputs[(size_t)p * 25 + k] = a[k];
  }
  const size_t rows = (size_t)1 << log_size;
  for (u32 i = 0; i < rows; ++i) {
    const u32 r = (u32)finalized_src_row(i, log_size);
    u32 v[ram::COLS] = {0};
    if (r < n_rows) ram::final_row(row_src[r], n_acc, outputs.data(), addresses, timestamps, init_addresses, init_values, v);
    for (u32 c = 0; c < ram::COLS; ++c) out[c * rows + i] = v[c];
  }
  return n_rows;
}
'''


@pytest.fixture(scope="module")
def host_fill(tmp_path_factory):
    d = tmp_path_factory.mktemp("ram_fill")
    src, so = d / "fill.cc", d / "fill.so"
    src.write_text(DRIVER)
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-w", "-I", CSRC, str(src), "-o", str(so)], check=True)
    lib = C.CDLL(str(so))
    lib.ram_fill_host.restype = C.c_uint32
    u32p, u64p, u8p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_uint8)

    def run(inputs, addresses, timestamps, init_addresses, init_values, log_size):
        inp = np.ascontiguousarray(inputs, dtype=np.uint64)
        addr = np.ascontiguousarray(addresses, dtype=np.uint32)
        ts = np.ascontiguousarray(timestamps, dtype=np.uint32)
        ia = np.ascontiguousarray(init_addresses, dtype=np.uint32)
        iv = np.ascontiguousarray(init_values, dtype=np.uint8)
        out = np.full((W.RAM_COLS, 1 << log_size), 0xDEADBEEF, np.uint32)
        n_rows = lib.ram_fill_host(C.c_uint32(inp.shape[0]), inp.ctypes.data_as(u64p), addr.ctypes.data_as(u32p), ts.ctypes.data_as(u32p),
                                   C.c_uint32(ia.size), ia.ctypes.data_as(u32p), iv.ctypes.data_as(u8p), C.c_uint32(log_size), out.ctypes.data_as(u32p))
        return out, int(n_rows)
    return run


def edge_side_notes():
    """(name, side note, initial memory) of the fill's edge cases."""
    rng = np.random.default_rng(7)

    def perms(addresses, ts_max=50):
        n = len(addresses)
        return (rng.integers(0, 1 << 64, (n, 25), dtype=np.uint64, endpoint=False), np.array(addresses, np.uint64),
                rng.integers(0, ts_max, (n, K.STATE_SIZE), dtype=np.uint64))

    out = []
    m = W.NexusV1KeccakMachine(8, 15, seed=1)                       # repeated and overlapping buffers, from the memory simulation
    out.append(("simulation", m.side_note(), m.initial_memory()))
    inputs, addresses, ts = perms([1000, 1100, 1000, 1203, 1100])   # repeated and overlapping, with init entries before, between and after
    ia = np.array(sorted(set(range(990, 1500, 3)) | {5, 1 << 31}), np.uint32)
    out.append(("untouched init", (inputs, addresses, ts), (ia, rng.integers(0, 256, ia.size).astype(np.uint8))))
    out.append(("single permutation", perms([77]), (np.arange(77, 277, dtype=np.uint32), rng.integers(0, 256, 200).astype(np.uint8))))
    inputs, addresses, ts = perms([0xFFFF - 100, 0x3FFFF - 199, 0x1FFFF - 7])      # 0xFFFF carries inside the 200 bytes
    ts[:, 3] = 0xFFFF
    ts[1, 5] = 0xFFFFFF
    ts[2, 9] = (1 << 32) - 2                                        # the largest accepted timestamp: counter 2^32 - 1
    out.append(("0xffff carries", (inputs, addresses, ts), (np.zeros(0, np.uint32), np.zeros(0, np.uint8))))
    top = (1 << 32) - K.STATE_SIZE                                  # the largest accepted address
    ia = np.array([top - 3, top + 199], np.uint32)
    out.append(("largest address", perms([top, top - 50]), (ia, np.array([9, 250], np.uint8))))
    return out


@pytest.mark.parametrize("case", edge_side_notes(), ids=lambda c: c[0])
def test_host_fill_equals_the_numpy_columns(host_fill, case):
    _name, side_note, (ia, iv) = case
    addr, _v, _c = W.last_access(*side_note, ia, iv)
    log_size = W.ram_log_size(addr.size)
    want = W.ram_init_final_columns(*side_note, ia, iv, log_size)[:, finalized_src_rows(log_size)]
    got, n_rows = host_fill(*side_note, ia, iv, log_size)
    assert n_rows == addr.size
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"
    # a batch one row too small is refused with the count
    if log_size > K.LOG_N_LANES and addr.size > 1 << (log_size - 1):
        assert host_fill(*side_note, ia, iv, log_size - 1)[1] == addr.size


def test_untouched_init_entries_keep_their_value_with_counter_zero():
    ia, iv = np.array([10, 500], np.uint32), np.array([3, 4], np.uint8)
    inputs, addresses, ts = np.zeros((1, 25), np.uint64), np.array([100], np.uint64), np.zeros((1, 200), np.uint64)
    addr, val, ctr = W.last_access(inputs, addresses, ts, ia, iv)
    assert addr.size == 202 and (addr[0], val[0], ctr[0]) == (10, 3, 0) and (addr[-1], val[-1], ctr[-1]) == (500, 4, 0)
    out_bytes = np.concatenate([K._lane_bytes(l) for l in K.keccak_f(np.zeros((25, 1), np.uint64))])[:, 0]
    assert np.array_equal(val[1:201], out_bytes) and np.all(ctr[1:201] == 1)


def test_fill_kernels_compile_for_sm90a_without_spills(tmp_path):
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++", "-Xcudafe",
                        "--diag_suppress=177", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-x", "cu", "-c",
                        os.path.join(CSRC, "ram_init_final.cu"), "-o", str(tmp_path / "ram_init_final.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    # ptxas prints each entry function's properties after its name; CUB's own sort and scan kernels are not held to this
    blocks = re.split(r"Compiling entry function '", r.stderr)[1:]
    ours = {b.split("'")[0]: b for b in blocks if "ram_" in b.split("'")[0]}
    for k in ("ram_keys_kernel", "ram_heads_kernel", "ram_tails_kernel", "ram_outputs_kernel", "ram_rows_kernel"):
        (name,) = [n for n in ours if k in n]
        spills = [int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", ours[name])]
        assert spills and max(spills) == 0, (k, ours[name])
