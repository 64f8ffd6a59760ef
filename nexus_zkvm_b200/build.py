"""In-tree build of libnexus_b200.so (hand-written CUDA for sm_90a + C++ host library, flat C ABI).

    python -m nexus_zkvm_b200.build [--force] [--verbose]

nvcc cross-compiles without a GPU.  The .so, the objects and jit_cache/ are build products (git-ignored).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libnexus_b200.so")
NVCC = os.environ.get("NB200_NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++",
          "-Xcudafe", "--diag_suppress=177", "--expt-relaxed-constexpr"]


def _sources():
    out = []
    for root, _, files in os.walk(CSRC):
        for f in sorted(files):
            if f.endswith((".cu", ".cc")):
                out.append(os.path.join(root, f))
    return sorted(out)


def _headers():
    out = [os.path.join(HERE, "..", "include", "nb200.h")]
    for root, _, files in os.walk(CSRC):
        for f in files:
            if f.endswith((".cuh", ".h")):
                out.append(os.path.join(root, f))
    return out


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    srcs = _sources()
    hdr_mtime = max(os.path.getmtime(h) for h in _headers())
    jobs = []
    objs = []
    for s in srcs:
        o = os.path.join(OBJ, os.path.relpath(s, CSRC).replace(os.sep, "_") + ".o")
        objs.append(o)
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hdr_mtime):
            cmd = [NVCC] + ARCH + CFLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-x", "cu", "-c", s, "-o", o]
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        return cmd, r

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for cmd, r in ex.map(run, jobs):
                if verbose or r.returncode != 0:
                    sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
                if r.returncode != 0:
                    raise RuntimeError("nvcc failed: " + " ".join(cmd))
    if jobs or force or not os.path.exists(LIB):
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-cudart", "static", "-ccbin", "/usr/bin/g++"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return LIB


# ---- cubin cache for the run-time specialised AIR kernels (csrc/jit.cu) ---------------------------------------------
JIT_CACHE = os.path.join(HERE, "jit_cache")
# (log_size, n_lanes, logup_in_pairs): bench.py / tools/prove_trace.py, __graft_entry__.smoke and the machines of tests/test_gpu_*.py
SHIPPED_MACHINES = [(20, 21, False), (22, 21, False), (16, 21, False), (8, 1, False), (8, 2, False), (8, 2, True), (8, 3, False), (9, 1, False), (9, 2, False),
                    (9, 2, True), (10, 1, False), (12, 3, False)] + [(ls, 1, False) for ls in range(16, 23)]   # the fused commit sizes


# prover2-shaped machines (machine.MultiMachine) of tests/test_gpu_prove_parity.py and bench.py --multi: component log sizes
SHIPPED_MULTI = [list(range(4, 12)), list(range(4, 18)), list(range(4, 22))]
# the reference's v1 main component as data (nexus_v1.NexusV1Machine): log sizes of the tests, bench.py (16 = CPU sample, 20, 22) and smoke()
SHIPPED_NEXUS_V1 = [8, 9, 12, 16, 18, 20, 22, 24]   # 18 / 24: the sharded large-proof test (default size / configs[3])
# the keccak precompile extension (keccak.KeccakMachine): log2 of the permutation count of tests/test_gpu_keccak.py (KeccakRound 0 at 2^10 and 2^12
# rows; 2^18 rows) and of tools/keccak_prove.py
SHIPPED_KECCAK = [6, 8, 14]


def kernel_sources(words, short_checks=False):
    """[(cache key, CUDA C source)] of the kernels the library specialises for an AIR (no GPU needed).  The constraint check (which = 3) is
    listed for the components whose constraint program is specialised; `short_checks` adds it for the short programs too (small table
    components, whose check kernel is often the same source in several machines)."""
    import ctypes as C
    import numpy as np
    L = C.CDLL(LIB)
    L.nb200_kernel_source_key.restype = C.c_uint64
    L.nb200_kernel_source_key.argtypes = [C.c_char_p]
    L.nb200_air_n_components.restype = C.c_uint32
    L.nb200_air_n_components.argtypes = [C.c_void_p]
    L.nb200_free.argtypes = [C.c_void_p]
    w = np.ascontiguousarray(words, dtype=np.uint32)
    air = C.c_void_p()
    if L.nb200_air_load(None, w.ctypes.data_as(C.POINTER(C.c_uint32)), C.c_size_t(w.size), C.byref(air)) != 0:
        raise RuntimeError("nb200_air_load failed")
    out = []
    for comp in range(L.nb200_air_n_components(air)):
        specialised = False
        for which in (0, 1, 2, 3):   # constraints, LogUp program, constraints of degree > 2 (the half coset D2), constraint check
            if which == 3 and not (specialised or short_checks):
                continue
            p = C.c_void_p()
            if L.nb200_air_kernel_source(air, C.c_uint32(comp), C.c_int(which), C.byref(p)) != 0 or not p:
                continue
            specialised = specialised or which == 0
            src = C.string_at(p)
            L.nb200_free(p)
            out.append((int(L.nb200_kernel_source_key(src)), src))
    L.nb200_air_free(air)
    return out


def precompile_kernels(machines=SHIPPED_MACHINES, verbose=False):
    """Compile the AIR kernels of the shipped machines with nvcc into jit_cache/<key>.cubin (what NVRTC would produce on
    first use): a fresh machine then neither pages in libnvrtc nor compiles."""
    from . import machine as M
    os.makedirs(JIT_CACHE, exist_ok=True)
    todo = {}
    ms = [M.AddMachine(log_size=log_size, n_lanes=lanes, logup_in_pairs=pairs) for log_size, lanes, pairs in machines]
    ms += [M.MultiMachine(sizes) for sizes in SHIPPED_MULTI]
    from .nexus_v1 import NexusV1Machine
    ms += [NexusV1Machine(ls) for ls in SHIPPED_NEXUS_V1]
    from .keccak import KeccakMachine
    ms += [KeccakMachine(lp) for lp in SHIPPED_KECCAK]
    for m in ms:
        for key, src in kernel_sources(m.words, short_checks=True):
            path = os.path.join(JIT_CACHE, f"{key:016x}.cubin")
            if not os.path.exists(path):
                todo[path] = src

    def run(item):
        path, src = item
        cu = path[:-6] + ".cu"
        with open(cu, "wb") as f:
            f.write(src)
        cmd = [NVCC] + ARCH + ["-O3", "-std=c++17", "-lineinfo", "-ccbin", "/usr/bin/g++", "-cubin", cu, "-o", path + ".tmp"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        os.remove(cu)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed on a generated kernel:\n" + r.stderr[-2000:])
        os.replace(path + ".tmp", path)
        return path

    if todo:
        with ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
            for path in ex.map(run, sorted(todo.items())):
                if verbose:
                    sys.stderr.write("cubin " + path + "\n")
    return len(todo)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
    if "--no-kernels" not in sys.argv:
        n = precompile_kernels(verbose="--verbose" in sys.argv)
        print(f"jit_cache: {n} kernel(s) compiled")
