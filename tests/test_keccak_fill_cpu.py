"""The keccak extension's device trace filler (csrc/keccak_trace.cuh, csrc/keccak_trace.cu) checked without a GPU: the per-row code the
kernels run is compiled as host C++ behind a thin driver that calls it for every row, exactly as the kernels' bodies do, and must equal
KeccakMachine.fill_main_trace() after the finalize permutation, multiplicities included; and the kernels compile for sm_90a within the
spill that DESIGN §4 states."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from nexus_zkvm_b200 import keccak as K
from tests.keccak_side_notes import edge_machine, finalized_main_trace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "nexus_zkvm_b200", "csrc")
NVCC = os.environ.get("NB200_NVCC", "/usr/local/cuda/bin/nvcc")
# the largest local-memory spill (stores or loads, bytes, any kernel) `nvcc -Xptxas -v` may report for keccak_trace.cu (DESIGN §4)
MAX_SPILL_BYTES = 512

DRIVER = r'''
#include "keccak_trace.cuh"
#include <vector>
using namespace nb;
struct HostInc { void operator()(u32* p) const { ++*p; } };
extern "C" void keccak_fill_host(u32 n_perms, const u64* inputs, const u32* addresses, const u32* timestamps, u32 mem_log, u32 r0, u32 r1,
                                 u32* mem, u32* rnd0, u32* rnd1, u32* mult) {
  for (u32 i = 0; i < (1u << mem_log); ++i) keccak::mem_row(inputs, addresses, timestamps, n_perms, mem_log, i, mem + i, (size_t)1 << mem_log);
  std::vector<u32> hist(2 * 65536 + (1u << keccak::ROTATE_LOG), 0);
  keccak::CountSink<HostInc> count{hist.data(), hist.data() + 65536, hist.data() + 2 * 65536};
  const u32 logs[2] = {r0, r1}, rounds[2] = {16, 8}, offsets[2] = {0, 16};
  u32* outs[2] = {rnd0, rnd1};
  for (int k = 0; k < 2; ++k) {
    const size_t n = (size_t)1 << logs[k];
    for (u32 i = 0; i < n; ++i) {
      keccak::ColumnSink s{outs[k] + i, n};
      outs[k][(keccak::ROUND_COLS - 1) * n + i] = keccak::round_component_row(inputs, n_perms, rounds[k], offsets[k], logs[k], i, s);
      keccak::round_component_row(inputs, n_perms, rounds[k], offsets[k], logs[k], i, count);
    }
  }
  for (u32 e = 0; e < keccak::MULT_WORDS; ++e) mult[e] = keccak::mult_word(hist.data(), hist.data() + 65536, hist.data() + 2 * 65536, e);
}
'''


@pytest.fixture(scope="module")
def host_fill(tmp_path_factory):
    d = tmp_path_factory.mktemp("keccak_fill")
    src, so = d / "fill.cc", d / "fill.so"
    src.write_text(DRIVER)
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-w", "-I", CSRC, str(src), "-o", str(so)], check=True)
    lib = C.CDLL(str(so))
    u32p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)

    def run(m):
        inputs, addresses, timestamps = m.side_note()
        mem_log, (r0, r1) = m.mem_log_size, m.round_log_sizes
        out = [np.zeros((2001, 1 << mem_log), np.uint32), np.zeros((1705, 1 << r0), np.uint32), np.zeros((1705, 1 << r1), np.uint32),
               np.zeros(32 * 4096 + 2048, np.uint32)]
        lib.keccak_fill_host(C.c_uint32(m.n_perms), inputs.ctypes.data_as(u64p), addresses.ctypes.data_as(u32p), timestamps.ctypes.data_as(u32p),
                             C.c_uint32(mem_log), C.c_uint32(r0), C.c_uint32(r1), *[o.ctypes.data_as(u32p) for o in out])
        return out[:3] + [out[3][:32 * 4096].reshape(32, 4096), out[3][32 * 4096:].reshape(1, 2048)]
    return run


def _check(got, want):
    names = ["memory check", "KeccakRound 0", "KeccakRound 1", "bitwise multiplicities", "rotate multiplicity"]
    for name, g, w in zip(names, got, want):
        assert g.shape == w.shape, name
        bad = np.argwhere(g != w)
        assert bad.size == 0, f"{name}: {len(bad)} cells differ, first (column, position) {tuple(bad[0])}"


@pytest.mark.parametrize("n_perms", [(1 << 4) - 1, (1 << 6) - 1, 37, 1 << 4])
def test_host_fill_equals_numpy_trace(host_fill, n_perms):
    m = K.KeccakMachine(None, seed=n_perms, n_perms=n_perms)
    _check(host_fill(m), finalized_main_trace(m))


@pytest.mark.parametrize("n_perms", [1, 37, 64])
def test_host_fill_equals_numpy_trace_on_edge_side_notes(host_fill, n_perms):
    m = edge_machine(n_perms, seed=n_perms)
    got, want = host_fill(m), finalized_main_trace(m)
    _check(got, want)
    # the edge cases are present: carries set in the memory check and both the zero and the all-ones state as inputs
    assert want[0][1600:2000].any()
    if n_perms > 1:
        assert (m.inputs == np.uint64((1 << 64) - 1)).all(axis=0).any() and (m.inputs == 0).all(axis=0).any()


def test_explicit_side_note_is_the_seeded_one():
    """A machine built from another machine's side note has the same trace."""
    a = K.KeccakMachine(4, seed=5)
    inputs, addresses, timestamps = a.side_note()
    b = K.KeccakMachine(inputs=inputs, addresses=addresses, timestamps=timestamps)
    assert b.n_perms == a.n_perms and b.log_sizes == a.log_sizes
    for x, y in zip(a.fill_main_trace(), b.fill_main_trace()):
        assert np.array_equal(np.asarray(x), np.asarray(y))


def test_side_note_ranges_are_checked():
    inputs = np.zeros((2, 25), np.uint64)
    ts = np.zeros((2, 200), np.uint64)
    with pytest.raises(AssertionError):
        K.KeccakMachine(inputs=inputs, addresses=[0, (1 << 32) - 199], timestamps=ts)
    ts[1, 3] = (1 << 32) - 1
    with pytest.raises(AssertionError):
        K.KeccakMachine(inputs=inputs, addresses=[0, 0], timestamps=ts)


def test_fill_kernels_compile_for_sm90a_within_the_stated_spill(tmp_path):
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++", "-Xcudafe",
                        "--diag_suppress=177", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-x", "cu", "-c",
                        os.path.join(CSRC, "keccak_trace.cu"), "-o", str(tmp_path / "keccak_trace.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    entries = re.findall(r"Compiling entry function '(\w+)'", r.stderr)
    for k in ("keccak_mem_fill_kernel", "keccak_mult_kernel", "keccak_round_count_kernel", "keccak_round_fill_kernel"):
        assert sum(k in e for e in entries) == 1, (k, entries)
    spills = [int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", r.stderr)]
    assert max(spills) <= MAX_SPILL_BYTES, r.stderr
