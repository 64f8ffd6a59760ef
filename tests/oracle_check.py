"""The oracle's constraint check (tests/oracle_check.cc: orc::run_program on every trace row, stwo's assert_constraints_on_polys) as a
Python function and as a backend for nexus_zkvm_b200.machine.check_constraints.  The shared object is compiled on first use into a
temporary directory, named after its sources, so the tree stays read-only."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import pyoracle as orc
from tests.oracle_backend import OracleBackend, _OracleProver

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "oracle_check.cc")
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for f in [SRC] + sorted(os.path.join(ROOT, "oracle", x) for x in os.listdir(os.path.join(ROOT, "oracle")) if x.endswith(".h")):
            h.update(open(f, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"nb200_oracle_check_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.tmp{os.getpid()}"
            subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "oracle"), SRC, "-o", tmp], check=True)
            os.replace(tmp, so)
        _lib = C.CDLL(so)
        _lib.orc_check_constraints.restype = C.c_int
    return _lib


def n_constraints(words, comp):
    import nexus_zkvm_b200 as nb
    w = np.ascontiguousarray(words, dtype=np.uint32)
    h = C.c_void_p()
    assert nb.lib().nb200_air_load(None, w.ctypes.data_as(u32p), C.c_size_t(w.size), C.byref(h)) == 0
    nb.lib().nb200_air_n_constraints.restype = C.c_uint32
    n = int(nb.lib().nb200_air_n_constraints(h, C.c_uint32(comp)))
    nb.lib().nb200_air_free(h)
    return n


def check(words, comp, trees, params):
    """[(failing rows, first failing trace row or None)] per constraint of component `comp`; trees[t][col] = committed evaluations."""
    w = np.ascontiguousarray(words, dtype=np.uint32)
    n = n_constraints(w, comp)
    keep = [[np.ascontiguousarray(c, dtype=np.uint32) for c in t] for t in trees]
    arrs = [(u32p * max(len(t), 1))(*[c.ctypes.data_as(u32p) for c in t]) for t in keep]
    cols = (C.c_void_p * 3)(*[C.cast(a, C.c_void_p) for a in arrs])
    ncols = (C.c_size_t * 3)(*[len(t) for t in keep])
    prm = np.ascontiguousarray(np.array(params, dtype=np.uint32).reshape(-1, 4))
    nf, fr = np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.uint64)
    st = lib().orc_check_constraints(w.ctypes.data_as(u32p), C.c_size_t(w.size), C.c_uint32(comp), cols, ncols, prm.ctypes.data_as(u32p),
                                     C.c_size_t(prm.shape[0]), nf.ctypes.data_as(u64p), fr.ctypes.data_as(u64p), C.c_size_t(n))
    assert st == 0, "orc_check_constraints failed"
    return [(int(nf[k]), int(fr[k]) if nf[k] else None) for k in range(n)]


class _OracleCheckProver(_OracleProver):
    """The oracle prover that also keeps the committed evaluations, so that it can run the constraint check."""

    def __init__(self, words, config):
        super().__init__(words, config)
        self.words = words
        self.trees = []

    def commit(self, cols, ch, coset_order=False):
        flat = []
        for c in cols:
            a = np.asarray(c)
            flat += list(a) if a.ndim == 2 else [a]
        flat = [np.ascontiguousarray(c, dtype=np.uint32) for c in flat]
        self.trees.append([orc.finalize_column(c) for c in flat] if coset_order else flat)
        return super().commit(flat, ch, coset_order)

    def commit_interaction(self, inter, ch):
        self.trees.append([np.ascontiguousarray(c, dtype=np.uint32) for block in inter for c in block])
        return super().commit_interaction(inter, ch)

    def check_constraints(self, comp, params):
        import nexus_zkvm_b200 as nb
        res = check(self.words, comp, self.trees, params)
        deg = np.zeros(max(len(res), 1), np.uint32)
        w = np.ascontiguousarray(self.words, dtype=np.uint32)
        h = C.c_void_p()
        assert nb.lib().nb200_air_load(None, w.ctypes.data_as(u32p), C.c_size_t(w.size), C.byref(h)) == 0
        assert nb.lib().nb200_air_constraint_degrees(h, C.c_uint32(comp), deg.ctypes.data_as(u32p), C.c_size_t(len(res))) == 0
        nb.lib().nb200_air_free(h)
        return [(k, int(deg[k]), a, r) for k, (a, r) in enumerate(res) if a]


class OracleCheckBackend(OracleBackend):
    """OracleBackend whose prover also answers check_constraints (machine.check_constraints on the CPU oracle)."""

    def prover(self, words, config):
        return _OracleCheckProver(words, config)
