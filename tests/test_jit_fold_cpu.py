"""Which constraints the code generator (csrc/jit.cu) folds, checked on the emitted CUDA C without a GPU.

A LogUp constraint coeff * (diff * den - num) whose den is linear in the parameters is emitted as diff * (coeff * den) - coeff * num,
with the products coeff * alpha^i and coeff * z computed once per CTA: one qmacq per folded constraint and no QM31 product by the
coefficient.  That the folded kernel computes the same quotients is checked against the oracle by test_jit_codegen_cpu.py."""
import ctypes as C
import re

import numpy as np
import pytest

import nexus_zkvm_b200 as nb
from nexus_zkvm_b200 import air as A
from nexus_zkvm_b200 import machine as M

# 64-bit products per call site in the generated code (qmac and everything built on it: 16; qmulb: 4; mul: 1)
PRODUCTS = {"qmac": 16, "qmul": 16, "qmac_tab": 16, "qmacq": 16, "qmulb": 4, "mul": 1}
# ... and per instruction of the unfolded emission (CONSTRE: qmac_tab, CONSTRB: qmulb)
OP_PRODUCTS = {A.OP_MULE: 16, A.OP_CONSTRE: 16, A.OP_MULEB: 4, A.OP_CONSTRB: 4, A.OP_MULB: 1}


def _source(words):
    w = np.ascontiguousarray(words, dtype=np.uint32)
    h = C.c_void_p()
    assert nb.lib().nb200_air_load(None, w.ctypes.data_as(C.POINTER(C.c_uint32)), C.c_size_t(w.size), C.byref(h)) == 0
    p = C.c_void_p()
    assert nb.lib().nb200_air_kernel_source(h, C.c_uint32(0), C.c_int(0), C.byref(p)) == 0
    src = C.string_at(p).decode()
    nb.lib().nb200_free(p)
    nb.lib().nb200_air_free(h)
    return src


def _program(words):
    """the constraint program of component 0 as (op, dst, a, b) rows (bytecode layout: nexus_zkvm_b200/air.py)"""
    w = [int(x) for x in words]
    i = 4 + 3
    i += 1 + 3 * w[i]
    n_instr = w[i + 2]
    i += 3
    return [tuple(w[i + 4 * k:i + 4 * k + 4]) for k in range(n_instr)]


def _per_row_products(src):
    body = src[src.index("void chunk0("):src.index('extern "C"')]   # the chunks run per row; the prologue once per CTA
    return sum(n * len(re.findall(r"(?<![A-Za-z0-9_])" + f + r"\(", body)) for f, n in PRODUCTS.items())


def _machine(kind):
    if kind == "nexus_v1":
        from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
        return NexusV1Machine(8)
    lanes, pairs = kind
    return M.AddMachine(log_size=8, n_lanes=lanes, logup_in_pairs=pairs)


@pytest.mark.parametrize("kind,folded", [("nexus_v1", 253), ((1, False), 12), ((2, True), 0)])
def test_logup_constraints_fold(kind, folded):
    m = _machine(kind)
    src = _source(m.words)
    prog = _program(m.words)
    assert src.count("rr = qmacq(") == folded
    n_logup = sum(1 for p in prog if p[0] == A.OP_CONSTRE)
    assert src.count("rr = qmac_tab(") == n_logup - folded
    if folded == 0:
        assert "nbfold" not in src and "qmacq" not in src
    else:
        assert "__syncthreads();\n  chunk0(" in src   # the folded products are complete before the first chunk reads them


def test_folding_removes_a_quarter_of_the_v1_products():
    m = _machine("nexus_v1")
    prog = _program(m.words)
    unfolded = sum(OP_PRODUCTS.get(p[0], 0) for p in prog)
    folded = _per_row_products(_source(m.words))
    assert folded <= 0.75 * unfolded, (folded, unfolded)


def test_unfolded_count_matches_the_unfolded_emission():
    """the paired machine folds nothing: its call-site count is the per-instruction count the v1 comparison above assumes"""
    m = _machine((2, True))
    assert _per_row_products(_source(m.words)) == sum(OP_PRODUCTS.get(p[0], 0) for p in _program(m.words))
