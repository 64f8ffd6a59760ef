"""Time the table-multiplicity count (nb200_table_multiplicities) on one GPU.

    python tools/table_multiplicities_time.py [--v1-log-size 20] [--keccak-log-perms 14] [--whole-log-size 20 --whole-log-perms 12]
                                              [--reps 20] [--out FILE]

Two workloads, each timed `reps` times after a warm-up with CUDA events recorded on the library's stream (one call: scratch allocation, hash
build, probes, stores, and the two synchronisations of the call):
  * NexusV1Machine(v1_log_size), padding witness, trees 0 and 1 uploaded from host columns; next to it the host's numpy bincount over the
    same lookup columns (what fill_main_trace does for the Range256 / Range32 columns);
  * KeccakMachine(keccak_log_perms) from device_trees (the side-note fill); next to it, in the same run, the device time of the side-note
    fill's hand-written lookup histogram (keccak_round_count_kernel) and of the count's own kernels, both from torch.profiler;
  * with --whole-log-size, NexusV1KeccakMachine(whole_log_size, 2^whole_log_perms) from device_trees, counted by
    nb200_table_multiplicities_first_row (its Range8 table lists 0 nine times); next to it the device time of the first-row resolve's two
    kernels (table_first_row_claim_kernel, table_first_row_slot_kernel) and of all the count's kernels, from torch.profiler.
The one-time NVRTC compile time of every component's count kernel (nb200_air_count_kernel_source) is measured on its own, with libnvrtc and
the options the library compiles with.  The library's cubin cache points to an empty directory under the system's temporary directory, so
nothing is read from or written to the tree.  Prints one JSON line with the card name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return dict(zip(q.split(","), (x.strip() for x in r.stdout.strip().split(",")))) if r.returncode == 0 else {}


def nvrtc_compile_ms(words):
    """{component: ms} of one NVRTC compile of each component's count kernel (the options of csrc/jit.cu jit_compile)."""
    import ctypes as C
    import numpy as np

    import nexus_zkvm_b200 as nb
    nv = None
    for name in ("libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so.12"):
        try:
            nv = C.CDLL(name)
            break
        except OSError:
            pass
    assert nv is not None, "libnvrtc not found"
    w = np.ascontiguousarray(words, dtype=np.uint32)
    h = C.c_void_p()
    assert nb.lib().nb200_air_load(None, w.ctypes.data_as(C.POINTER(C.c_uint32)), C.c_size_t(w.size), C.byref(h)) == 0
    out = {}
    opts = (C.c_char_p * 3)(b"--gpu-architecture=sm_90a", b"--std=c++17", b"-lineinfo")
    for k in range(nb.lib().nb200_air_n_components(h)):
        p = C.c_void_p()
        if nb.lib().nb200_air_count_kernel_source(h, C.c_uint32(k), C.byref(p)) != 0:
            continue
        src = C.string_at(p)
        nb.lib().nb200_free(p)
        prog = C.c_void_p()
        assert nv.nvrtcCreateProgram(C.byref(prog), src, b"nb200_air.cu", 0, None, None) == 0
        t = time.perf_counter()
        st = nv.nvrtcCompileProgram(prog, 3, opts)
        out[k] = (time.perf_counter() - t) * 1e3
        nv.nvrtcDestroyProgram(C.byref(prog))
        assert st == 0, f"NVRTC failed on component {k}"
    nb.lib().nb200_air_free(h)
    return out


def kernel_ms(fn, names, reps):
    """Device time per call of fn() spent in kernels whose name contains one of `names` (torch.profiler, `reps` calls)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    tot = 0.0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and any(n in e.name for n in names):
            tot += e.device_time_total   # microseconds
    return tot / reps / 1e3


def timed(ctx, stream, air, tree0, tree1, reps, first_row=False):
    import torch
    call = lambda: ctx.table_multiplicities(air, tree0, tree1, first_row=first_row)
    call()                                                       # warm-up: loads (or compiles) every count kernel
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        n = call()[0]
        e1.record(stream)
        e1.synchronize()
        assert n == 0
        ms.append(e0.elapsed_time(e1))
    ms.sort()
    names = ("nbjit", "table_mult_store") + (("table_first_row",) if first_row else ())
    return {"ms_median": ms[len(ms) // 2], "ms_min": ms[0], "ms_max": ms[-1], "count_kernels_ms": kernel_ms(call, names, 5)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--v1-log-size", type=int, default=20)
    ap.add_argument("--keccak-log-perms", type=int, default=14)
    ap.add_argument("--whole-log-size", type=int, default=0, help="main component log size of the whole-machine workload (0: not run)")
    ap.add_argument("--whole-log-perms", type=int, default=12)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    os.environ["NB200_JIT_CACHE"] = tempfile.mkdtemp(prefix="nb200_count_jit_")
    import numpy as np
    import torch

    import nexus_zkvm_b200 as nb
    from nexus_zkvm_b200.keccak import KeccakMachine
    from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
    from nexus_zkvm_b200.prover import Air
    from tests import table_mult_ref as ref

    assert torch.cuda.is_available(), "needs a GPU"
    stream = torch.cuda.Stream()
    ctx = nb.Context(0, stream=stream.cuda_stream)
    res = {"what": "nb200_table_multiplicities", "reps": a.reps, "gpu": card()}

    m = NexusV1Machine(a.v1_log_size)
    t1 = ref.flat(m.fill_main_trace(seed=1))
    groups = []
    for cols in (ref.flat(m.preprocessed_columns()), t1):
        out, i = [], 0
        while i < len(cols):
            j = i
            while j < len(cols) and len(cols[j]) == len(cols[i]):
                j += 1
            out.append(ctx.upload(np.stack(cols[i:j]), coset_order=True))
            i = j
        groups.append(out)
    air = Air(ctx, m.words)
    v1 = timed(ctx, stream, air, groups[0], groups[1], a.reps)
    # the host's count of the same lookups: one bincount per looked-up column (Range256 / Range32), as fill_main_trace does
    comp = m.air.components[0]
    lk = [(ref._leaves(comp, comp.lookups[i][2][0]), 256 if rel.name == "Range256" else 32)
          for i, (kind, rel, _x) in enumerate(ref.classify(m.air)[0]) if kind == "lookup"]
    ts = []
    for _ in range(3):
        t = time.perf_counter()
        h = {256: np.zeros(256, np.int64), 32: np.zeros(32, np.int64)}
        for leaves, size in lk:
            (tree, col, _o), = leaves
            h[size] += np.bincount(t1[col], minlength=size)
        ts.append((time.perf_counter() - t) * 1e3)
    v1["host_bincount_ms"] = min(ts)
    v1["lookups"] = len(lk)
    res["v1"] = dict(log_size=a.v1_log_size, nvrtc_compile_ms=nvrtc_compile_ms(m.words), **v1)
    del groups, t1

    km = KeccakMachine(a.keccak_log_perms)
    tree0, tree1 = km.device_trees(ctx)
    res["keccak"] = dict(log_n_perms=a.keccak_log_perms, n_perms=km.n_perms, round_log_sizes=km.round_log_sizes,
                         **timed(ctx, stream, Air(ctx, km.words), tree0, tree1, a.reps))
    side_note = km.side_note()

    def fill():
        for b in ctx.keccak_main_trace(*side_note):
            b.free()
    fill()
    res["keccak"]["fill_round_count_kernel_ms"] = kernel_ms(fill, ("keccak_round_count_kernel",), 5)
    res["keccak"]["nvrtc_compile_ms"] = nvrtc_compile_ms(km.words)
    del tree0, tree1

    if a.whole_log_size:
        from nexus_zkvm_b200.whole_machine import NexusV1KeccakMachine
        wm = NexusV1KeccakMachine(a.whole_log_size, 1 << a.whole_log_perms)
        tree0, tree1 = wm.device_trees(ctx)
        air = Air(ctx, wm.words)
        n_repeated = ctx.table_multiplicities(air, tree0, tree1, first_row=True)[2]
        w = timed(ctx, stream, air, tree0, tree1, a.reps, first_row=True)
        w["resolve_kernels_ms"] = kernel_ms(lambda: ctx.table_multiplicities(air, tree0, tree1, first_row=True), ("table_first_row",), 5)
        w["resolve_share_of_call"] = w["resolve_kernels_ms"] / w["ms_median"]
        table_rows = sum(1 << wm.air.components[k].log_size for k, row in enumerate(ref.classify(wm.air)) for (kind, _r, _c) in row if kind == "table")
        res["whole"] = dict(what="nb200_table_multiplicities_first_row", log_size=a.whole_log_size, n_perms=wm.n_perms,
                            component_log_sizes=wm.log_sizes, table_rows=table_rows, n_repeated=n_repeated, **w)
        del tree0, tree1
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
