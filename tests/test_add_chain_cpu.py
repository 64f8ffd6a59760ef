"""The reference's ADD-chain benchmark as an executing v1 trace (nexus_zkvm_b200/add_chain.py) without a GPU: the program's encodings and
execution, oracle proofs whose verifier accepts and whose claimed sums cancel (full and padded runs), no constraint failing on the executing
witness, corruptions that break a named constraint or the sums (every new DecodingCheck constraint among them), the device fill's per-row code
(csrc/v1_trace.cuh, compiled as host C++) equal to the numpy columns, the recorded AIR of the existing machines unchanged by the new keyword,
and the fill kernel compiled for sm_90a without spills."""
import ctypes as C
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest

from nexus_zkvm_b200 import add_chain as AC
from nexus_zkvm_b200 import machine as M
from nexus_zkvm_b200 import nexus_v1 as V
from tests import oracle_check
from tests import random_witness as rw
from tests.keccak_side_notes import finalized_src_rows
from tests.oracle_backend import OracleBackend, verify

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "nexus_zkvm_b200", "csrc")
NVCC = os.environ.get("NB200_NVCC", "/usr/local/cuda/bin/nvcc")
OFFSETS = {}
_o = 0
for _name, _size in V.MAIN_COLUMNS:
    OFFSETS[_name] = _o
    _o += _size
# the recorded AIR of NexusV1Machine(8) and of the whole machine NexusV1KeccakMachine(8, 15, seed=1), and their generated kernels: the
# digests from before record_main_component had its `decoding` keyword, which defaults off
KERNELS_SHA256 = {"v1": "67987233cc90ce90e43a029849c8d552fcef706c0db2a8f86acb49ea4ee1073a", "whole": "7f5fa2efe90eca357f18e1cae8c147a368616f5712c71852f3d29930c1abe26a"}
WORDS_SHA256 = {"v1": "5b97eb4115659d3a2bffe80c7ea8e9dbf7c1e0dad48820bf43d3ea53c4bb22a4", "whole": "bce3b683c32d2d2069fa894ebc8fe531821422b0cff84ccabf9ff6bf3fd48e65"}


def _decode(word):
    w = int(word)
    return {"opcode": w & 0x7F, "rd": (w >> 7) & 31, "funct3": (w >> 12) & 7, "rs1": (w >> 15) & 31, "rs2": (w >> 20) & 31, "funct7": w >> 25,
            "imm": ((w >> 20) ^ 0x800) - 0x800}


def test_program_encodings_and_execution():
    words, ops = AC.add_chain_program(10)
    assert words.size == 1024 and int(words[0]) == 0x00100093                       # addi x1, x0, 1
    d = _decode(words[0])
    assert (d["opcode"], d["rd"], d["rs1"], d["imm"], d["funct3"]) == (0b0010011, 1, 0, 1, 0)
    for t in range(1, words.size):                                               # add x_k, x_j, x_i with (i, j, k) = (0, 1, 2) + t - 1 mod 32
        d = _decode(words[t])
        i = (t - 1) % 32
        assert (d["opcode"], d["funct3"], d["funct7"]) == (0b0110011, 0, 0)
        assert (d["rd"], d["rs1"], d["rs2"]) == ((i + 2) % 32, (i + 1) % 32, i) == ops[t][1:]
    steps, (final, final_ts) = AC.execute(ops)
    # the recurrence directly: x1 = 1, then x_k = x_j + x_i (x0 stays 0)
    x = [0] * 32
    x[1] = 1
    for _op, rd, rs1, rs2 in ops[1:]:
        if rd:
            x[rd] = (x[rs1] + x[rs2]) & 0xFFFFFFFF
    assert list(final) == x
    f = {n: steps[i] for i, n in enumerate(AC.STEP_FIELDS)}
    assert np.array_equal(f["pc"], AC.ELF_TEXT_START + 4 * np.arange(1024)) and np.all(f["pc_ctr_prev"] == 0)
    assert np.sum(f["rd"] == 0) == 1024 // 32                                     # x0 is written once every 32 instructions
    assert np.all(f["ts3_prev"] < 3 * np.arange(1, 1025) + 3) and int(final_ts.max()) == 3 * 1024 + 3


@pytest.fixture(scope="module", params=[(8, None), (10, None), (10, 700)], ids=["2^8", "2^10", "700-in-2^10"])
def machine(request):
    ls, n = request.param
    m = AC.AddChainMachine(ls, n)
    return m, m.fill_main_trace()


def test_oracle_proves_verifies_and_sums_cancel(machine):
    m, t1 = machine
    assert m.log_sizes == [m.log_size, 5, 8, 4, 4, 4, 5, 7, 8]
    proof, claimed, aux = M.prove(m, OracleBackend(), t1, None, associated_data=b"add chain")
    verify(m, proof, aux)
    assert len(claimed) == 9 and M.verify_claimed_sums(claimed)
    # the main component's ProgramCheck and RegisterCheck lookups carry nonzero numerators: its sum alone does not vanish
    assert claimed[0] != (0, 0, 0, 0)


def _failures(m, t1, comps=None):
    w = rw.Witness(rw.ref.flat(m.preprocessed_columns()), t1)
    _p, params, trees = rw.on_oracle(m, w)
    out = {}
    for k in (comps if comps is not None else range(len(m.air.components))):
        out[k] = [(i, a, r) for i, (a, r) in enumerate(oracle_check.check(m.words, k, trees, params)) if a]
    return out


def test_no_constraint_fails_on_the_executing_witness(machine):
    m, t1 = machine
    assert all(not v for v in _failures(m, t1).values())


def _decoding_range(monkeypatch, *args):
    """(machine, indices of its main component's DecodingCheck constraints)."""
    seen = []
    orig = V._record_decoding_r_i

    def wrapped(m, *a):
        first = len(m.constraints)
        orig(m, *a)
        seen.append(range(first, len(m.constraints)))

    monkeypatch.setattr(V, "_record_decoding_r_i", wrapped)
    mach = AC.AddChainMachine(*args[:2], ops=args[2] if len(args) > 2 else None)
    return mach, seen[0]


def _corrupt(t1, name, limb, row, value):
    bad = list(t1)
    c = bad[OFFSETS[name] + limb].copy()
    c[row] = value % ((1 << 31) - 1)
    bad[OFFSETS[name] + limb] = c
    return bad


@pytest.mark.parametrize("name,limb", [("ValueA", 1), ("CarryFlag", 0), ("InstrVal", 2), ("Reg3TsPrev", 0)])
def test_corruption_is_caught(name, limb):
    m = AC.AddChainMachine(8)
    t1 = m.fill_main_trace()
    row = 77
    bad = _corrupt(t1, name, limb, row, int(t1[OFFSETS[name] + limb][row]) + 1)
    fails = _failures(m, bad, comps=[0])[0]
    claimed = M._commit_trees(m, OracleBackend(), bad, None, None, b"", None)[3]
    # the failing constraints hold the corrupted row, or the corruption only shows in the sums
    assert any(r == row for _i, _a, r in fails) or not M.verify_claimed_sums(claimed), (name, fails)
    assert fails, name                                                           # each of these also breaks an AIR constraint


def mixed_program():
    """ADD and ADDI over every register, immediates of every sign and bit pattern, rd = rs1 / rs2 / x0."""
    rng = np.random.default_rng(5)
    ops = []
    for t in range(480):
        if t % 2:
            ops.append((AC.OP_ADD, int(rng.integers(0, 32)), int(rng.integers(0, 32)), int(rng.integers(0, 32))))
        else:
            ops.append((AC.OP_ADDI, int(rng.integers(0, 32)), int(rng.integers(0, 32)), int(rng.integers(-2048, 2048))))
    return ops


def test_another_add_addi_program_proves_and_checks():
    m = AC.AddChainMachine(9, ops=mixed_program())
    t1 = m.fill_main_trace()
    assert all(not v for v in _failures(m, t1).values())
    claimed = M._commit_trees(m, OracleBackend(), t1, None, None, b"", None)[3]
    assert M.verify_claimed_sums(claimed)


def test_every_decoding_constraint_is_broken_by_some_corruption(monkeypatch):
    """Each corruption is applied at its own row of a mixed ADD / ADDI trace: a decoding column or an instruction byte off by one, an
    opcode flag raised (alone, or with the instruction byte that flag's funct3 / funct7 reads changed), or a shift flag raised on an ADDI
    row with one of its pieces changed.  Every DecodingCheck constraint fails on at least one of those rows."""
    m, dec = _decoding_range(monkeypatch, 9, None, mixed_program())
    t1 = m.fill_main_trace()
    imm_c = t1[OFFSETS["ImmC"]]
    add_rows = [r for r in range(1, 480) if imm_c[r] == 0]
    addi_rows = [r for r in range(1, 480) if imm_c[r] == 1]
    pieces = [("OpA0", 0), ("OpA1_4", 0), ("OpB0", 0), ("OpB1_4", 0), ("OpC0_3", 0), ("OpC4", 0), ("OpC4_7", 0), ("OpC8_10", 0), ("OpC11", 0),
              ("OpA", 0), ("OpB", 0), ("OpC", 0)] + [("ValueC", k) for k in range(4)] + [("InstrVal", k) for k in range(4)]
    flags = V.TYPE_R_OPS + V.IS_LOAD + ["IsJalr"]
    cases = []                                                                   # (rows to take it from, [(column, limb, delta or None = set 1)])
    for rows in (add_rows, addi_rows):
        cases += [(rows, [(n, k, 1)]) for n, k in pieces]
        for f in flags:
            cases += [(rows, [(f, 0, None)]), (rows, [(f, 0, None), ("InstrVal", 1, 16)]), (rows, [(f, 0, None), ("InstrVal", 3, 2)])]
    for f in V.ALU_IMM_SHIFT:
        cases += [(addi_rows, [(f, 0, None), (n, k, 1)]) for n, k in pieces] + [(addi_rows, [(f, 0, None)])]
    bad = [c.copy() for c in t1]
    taken = {id(add_rows): 0, id(addi_rows): 0}
    for rows, case in cases:
        row = rows[taken[id(rows)]]
        taken[id(rows)] += 1
        for name, limb, delta in case:
            c = bad[OFFSETS[name] + limb]
            c[row] = 1 if delta is None else (int(c[row]) + delta) % ((1 << 31) - 1)
    fails = {i for i, _a, _r in _failures(m, bad, comps=[0])[0]}
    missing = [i for i in dec if i not in fails]
    assert len(dec) == 73 and not missing, missing


DRIVER = r'''
#include "v1_trace.cuh"
using namespace nb;
extern "C" void v1_fill_host(u32 n_steps, const u32* steps, u32 n_prog, const u32* final_ctr, u32 log_size, u32* out) {
  const size_t n = (size_t)1 << log_size;
  for (u32 i = 0; i < n; ++i) v1::main_row(steps, n_steps, final_ctr, n_prog, log_size, i, out + i, n);
}
extern "C" u32 v1_col_offset(u32 k) {
  const u32 t[] = {v1::col::Pc, v1::col::PcNext, v1::col::OpA, v1::col::OpB, v1::col::OpC, v1::col::CarryFlag, v1::col::ImmC, v1::col::InstrVal,
                   v1::col::ValueA, v1::col::ValueAEffective, v1::col::ValueB, v1::col::ValueC, v1::col::IsAdd, v1::col::IsPadding,
                   v1::col::ValueAEffectiveFlag, v1::col::ValueAEffectiveFlagAux, v1::col::ValueAEffectiveFlagAuxInv, v1::col::Reg1Address,
                   v1::col::Reg2Address, v1::col::Reg3Address, v1::col::Reg1ValPrev, v1::col::Reg2ValPrev, v1::col::Reg3ValPrev,
                   v1::col::Reg1TsPrev, v1::col::ProgCtrPrev, v1::col::ProgCtrCur, v1::col::ProgCtrCarry, v1::col::FinalPrgMemoryCtr,
                   v1::col::CReg1TsPrev, v1::col::CH1Minus, v1::col::OpC0_3, v1::col::OpC4_7, v1::col::OpC8_10, v1::col::OpC11, v1::col::OpA1_4,
                   v1::col::OpB1_4, v1::col::OpC4, v1::col::OpA0, v1::col::OpB0, v1::col::PcCarry};
  return t[k];
}
'''
COL_NAMES = ["Pc", "PcNext", "OpA", "OpB", "OpC", "CarryFlag", "ImmC", "InstrVal", "ValueA", "ValueAEffective", "ValueB", "ValueC", "IsAdd",
             "IsPadding", "ValueAEffectiveFlag", "ValueAEffectiveFlagAux", "ValueAEffectiveFlagAuxInv", "Reg1Address", "Reg2Address", "Reg3Address",
             "Reg1ValPrev", "Reg2ValPrev", "Reg3ValPrev", "Reg1TsPrev", "ProgCtrPrev", "ProgCtrCur", "ProgCtrCarry", "FinalPrgMemoryCtr",
             "CReg1TsPrev", "CH1Minus", "OpC0_3", "OpC4_7", "OpC8_10", "OpC11", "OpA1_4", "OpB1_4", "OpC4", "OpA0", "OpB0", "PcCarry"]


@pytest.fixture(scope="module")
def host_fill(tmp_path_factory):
    d = tmp_path_factory.mktemp("v1_fill")
    src, so = d / "fill.cc", d / "fill.so"
    src.write_text(DRIVER)
    subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-w", "-I", CSRC, str(src), "-o", str(so)], check=True)
    lib = C.CDLL(str(so))
    lib.v1_col_offset.restype = C.c_uint32
    u32p = C.POINTER(C.c_uint32)

    def run(m):
        st = np.ascontiguousarray(m.steps, np.uint32)
        ctr = np.ascontiguousarray(m.final_ctr, np.uint32)
        out = np.zeros((347, 1 << m.log_size), np.uint32)                       # the device clears the batch first
        lib.v1_fill_host(C.c_uint32(st.shape[1]), st.ctypes.data_as(u32p), C.c_uint32(ctr.size), ctr.ctypes.data_as(u32p), C.c_uint32(m.log_size),
                         out.ctypes.data_as(u32p))
        return out
    run.lib = lib
    return run


def test_column_offsets_are_the_layouts(host_fill):
    assert [host_fill.lib.v1_col_offset(k) for k in range(len(COL_NAMES))] == [OFFSETS[n] for n in COL_NAMES]


@pytest.mark.parametrize("ls,n", [(8, None), (10, 700), (9, "mixed"), (12, 1)])
def test_host_fill_equals_the_numpy_columns(host_fill, ls, n):
    m = AC.AddChainMachine(ls, ops=mixed_program()) if n == "mixed" else AC.AddChainMachine(ls, n)
    want = np.stack(m.fill_main_trace()[:347])[:, finalized_src_rows(ls)]
    got = host_fill(m)
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{len(bad)} cells differ, first (column, position) {tuple(bad[0])}"


def _sha(words):
    return hashlib.sha256(np.ascontiguousarray(words, np.uint32).tobytes()).hexdigest()


def test_existing_machines_record_the_same_air():
    from nexus_zkvm_b200 import whole_machine as W
    assert _sha(V.NexusV1Machine(8).words) == WORDS_SHA256["v1"]
    assert _sha(W.NexusV1KeccakMachine(8, 15, seed=1).words) == WORDS_SHA256["whole"]


def test_existing_machines_generate_the_same_kernels():
    from nexus_zkvm_b200 import build as B
    from nexus_zkvm_b200 import whole_machine as W
    for name, m in (("v1", V.NexusV1Machine(8)), ("whole", W.NexusV1KeccakMachine(8, 15, seed=1))):
        digest = hashlib.sha256(b"".join(src for _key, src in B.kernel_sources(m.words, short_checks=True))).hexdigest()
        assert digest == KERNELS_SHA256[name], name



def test_fill_kernel_compiles_for_sm90a_without_spills(tmp_path):
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ccbin", "/usr/bin/g++", "-Xcudafe",
                        "--diag_suppress=177", "--expt-relaxed-constexpr", "-Xptxas", "-v", "-x", "cu", "-c",
                        os.path.join(CSRC, "v1_trace.cu"), "-o", str(tmp_path / "v1_trace.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    blocks = re.split(r"Compiling entry function '", r.stderr)[1:]
    (block,) = [b for b in blocks if "v1_main_trace_kernel" in b.split("'")[0]]
    spills = [int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", block)]
    assert spills and max(spills) == 0, block
