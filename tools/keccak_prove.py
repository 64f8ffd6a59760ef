"""Time whole GPU proofs of the keccak precompile extension (nexus_zkvm_b200/keccak.py: its six components, witness from Keccak-f[1600]).

    python tools/keccak_prove.py [--log-perms 14] [--steps 3] [--warmup 1] [--out-dir DIR] [--device-fill [--fill-calls 20]]

KeccakMachine(log_perms) holds 2^log_perms - 1 permutations: KeccakRound 0 has 2^(log_perms + 4) rows, KeccakRound 1 half of that, the memory
check 2^log_perms.  One step = machine.prove on the CUDA backend from the host trace (tree commits with their uploads, interaction trace, quotients,
FRI, decommitment), timed with a host clock that ends when the proof bytes are back on the host.  The witness is built once, before the timed
steps.  Device memory in use (cudaMemGetInfo, whole device) is sampled every 20 ms over the timed steps.  The last proof is checked by the
oracle's verifier.  Writes keccak_prove.json (also printed) to --out-dir (default: <temp dir>/keccak_prove) with the card's name, power limit and SM clock read in the same run.

--device-fill compares two arms in one run, alternating step by step after the warm-up: `host` proves from the host columns as above,
`device` from the side note (KeccakMachine.device_trees: tree 0 uploaded, tree 1 filled by nb200_keccak_main_trace, then machine.prove with
resident=), both timed from the start of the call to the proof bytes on the host.  The peak of each arm is the memory pool's used-memory
high-water mark over its steps (reset before each step; the library's columns, trees and temporaries; twiddles are not pool memory).  The
fill alone is timed with CUDA events on the library's stream (median of --fill-calls calls after one warm-up call; the side note's host
checks and copies included), and one fill runs under torch.profiler to split it by kernel.  The two arms' proof bytes must be equal.  Writes
keccak_fill.json."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return dict(zip(q.split(","), (x.strip() for x in r.stdout.strip().split(",")))) if r.returncode == 0 else {}


class MemSampler:
    """Largest device memory in use (total - free) seen by a polling thread."""

    def __init__(self, torch):
        self.torch, self.peak, self.stop = torch, 0, threading.Event()
        self.t = threading.Thread(target=self.run, daemon=True)

    def run(self):
        while not self.stop.is_set():
            free, total = self.torch.cuda.mem_get_info(0)
            self.peak = max(self.peak, total - free)
            time.sleep(0.02)

    def __enter__(self):
        self.t.start()
        return self

    def __exit__(self, *exc):
        self.stop.set()
        self.t.join()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-perms", type=int, default=14)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "keccak_prove"))
    ap.add_argument("--no-verify", action="store_true")
    ap.add_argument("--device-fill", action="store_true")
    ap.add_argument("--fill-calls", type=int, default=20)
    a = ap.parse_args()
    if a.device_fill:
        return device_fill(a)
    import torch

    import nexus_zkvm_b200 as nb
    from nexus_zkvm_b200 import keccak as K
    from nexus_zkvm_b200 import machine as M
    from nexus_zkvm_b200.prover import CudaBackend

    assert torch.cuda.is_available(), "needs a GPU"
    t0 = time.perf_counter()
    m = K.KeccakMachine(a.log_perms, seed=a.seed)
    cols = m.fill_main_trace()
    witness_s = time.perf_counter() - t0
    ctx = nb.Context(0)
    backend = CudaBackend(ctx)
    free0, total = torch.cuda.mem_get_info(0)
    for _ in range(a.warmup):
        M.prove(m, backend, cols, None)
    times = []
    with MemSampler(torch) as mem:
        for _ in range(a.steps):
            t = time.perf_counter()
            proof, claimed, aux = M.prove(m, backend, cols, None)
            times.append(time.perf_counter() - t)
    verified = None
    if not a.no_verify:
        from tests.oracle_backend import verify_with_replayed_transcript
        verify_with_replayed_transcript(m, proof, claimed, aux)
        verified = "accepted"
    ms = 1e3 * min(times)
    rounds = m.n_perms * K.ROUNDS
    out = {
        "workload": "KeccakMachine: PermutationMemoryCheck, KeccakRound 0 (16 rounds), KeccakRound 1 (8 rounds), XorTable, BitNotAndTable, BitRotateTable",
        "log_perms": a.log_perms, "permutations": m.n_perms, "component_log_sizes": m.log_sizes, "columns": m.air.n_columns(),
        "config": dict(pow_bits=5, log_blowup=1, log_last=0, n_queries=3),
        "steps": a.steps, "warmup": a.warmup, "ms_per_proof": round(ms, 2), "ms_all_steps": [round(1e3 * x, 2) for x in times],
        "permutations_per_s": round(m.n_perms / (ms / 1e3), 1), "keccak_rounds_per_s": round(rounds / (ms / 1e3), 1),
        "peak_device_memory_gb": round(mem.peak / 1e9, 2), "device_memory_in_use_before_gb": round((total - free0) / 1e9, 2),
        "proof_bytes": len(proof), "oracle_verifier": verified, "witness_build_s": round(witness_s, 2),
        "timing": "host clock around machine.prove from host columns to proof bytes on the host; minimum over the steps",
        "card": card(),
    }
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "keccak_prove.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))
    ctx.close()


class PoolHigh:
    """The device's default memory pool (where the library allocates): its used-memory high-water mark, resettable."""
    USED_MEM_HIGH = 8   # CU_MEMPOOL_ATTR_USED_MEM_HIGH

    def __init__(self, device=0):
        import ctypes as C
        self.C, self.cu = C, C.CDLL("libcuda.so.1")
        assert self.cu.cuInit(0) == 0
        dev = C.c_int()
        assert self.cu.cuDeviceGet(C.byref(dev), device) == 0
        self.pool = C.c_void_p()
        assert self.cu.cuDeviceGetDefaultMemPool(C.byref(self.pool), dev) == 0

    def reset(self):
        z = self.C.c_uint64(0)
        assert self.cu.cuMemPoolSetAttribute(self.pool, self.USED_MEM_HIGH, self.C.byref(z)) == 0

    def high(self):
        v = self.C.c_uint64()
        assert self.cu.cuMemPoolGetAttribute(self.pool, self.USED_MEM_HIGH, self.C.byref(v)) == 0
        return v.value


def device_fill(a):
    import statistics

    import torch

    import nexus_zkvm_b200 as nb
    from nexus_zkvm_b200 import keccak as K
    from nexus_zkvm_b200 import machine as M
    from nexus_zkvm_b200.prover import CudaBackend

    assert torch.cuda.is_available(), "needs a GPU"
    t0 = time.perf_counter()
    m = K.KeccakMachine(a.log_perms, seed=a.seed)
    cols = m.fill_main_trace()
    witness_s = time.perf_counter() - t0
    side_note = m.side_note()
    stream = torch.cuda.Stream()
    ctx = nb.Context(0, stream=stream.cuda_stream)   # the library's work on a stream the CUDA events can be recorded on
    backend = CudaBackend(ctx)
    pool = PoolHigh()

    def fill_once():
        for b in ctx.keccak_main_trace(*side_note):
            b.free()

    # the fill alone
    fill_once()
    ctx.sync()
    fill_ms = []
    for _ in range(a.fill_calls):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream)
        batches = ctx.keccak_main_trace(*side_note)
        ev1.record(stream)
        ev1.synchronize()
        fill_ms.append(ev0.elapsed_time(ev1))
        for b in batches:
            b.free()
    ctx.sync()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fill_once()
        ctx.sync()
    kernels = {}   # device time (ms) of the fill's kernels and copies, by kernel
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", None)
        us = getattr(e, "self_cuda_time_total", 0) if us is None else us
        if us and ("keccak" in e.key or "emcpy" in e.key or "emset" in e.key):
            name = next((k for k in ("mem_fill", "round_fill", "round_count", "mult_kernel") if k in e.key), e.key)
            kernels[name] = kernels.get(name, 0.0) + us / 1e3

    arms = {"host": lambda: M.prove(m, backend, cols, None),
            "device": lambda: M.prove(m, backend, None, None, resident=m.device_trees(ctx))}
    for _ in range(a.warmup):
        for run in arms.values():
            run()
    times, peaks, proofs = {k: [] for k in arms}, {k: 0 for k in arms}, {}
    for _ in range(a.steps):
        for name, run in arms.items():
            ctx.sync()
            pool.reset()
            t = time.perf_counter()
            proofs[name] = run()
            times[name].append(time.perf_counter() - t)
            peaks[name] = max(peaks[name], pool.high())
    assert proofs["host"][0] == proofs["device"][0], "the two arms' proof bytes differ"
    verified = None
    if not a.no_verify:
        from tests.oracle_backend import verify_with_replayed_transcript
        proof, claimed, aux = proofs["device"]
        verify_with_replayed_transcript(m, proof, claimed, aux)
        verified = "accepted"
    med = statistics.median(fill_ms)
    out = {
        "workload": "KeccakMachine tree 1 filled on the device from the side note (nb200_keccak_main_trace) vs uploaded from host columns",
        "log_perms": a.log_perms, "permutations": m.n_perms, "component_log_sizes": m.log_sizes, "columns": m.air.n_columns(),
        "config": dict(pow_bits=5, log_blowup=1, log_last=0, n_queries=3),
        "fill_ms_median": round(med, 3), "fill_ms_all": [round(x, 3) for x in fill_ms], "fill_calls": a.fill_calls,
        "fill_kernel_ms": {k: round(v, 3) for k, v in sorted(kernels.items())},
        "side_note_bytes": int(sum(x.nbytes for x in side_note)),
        "tree1_bytes_on_device": int(4 * sum(c * (1 << ls) for c, ls in ((2001, m.mem_log_size), (1705, m.round_log_sizes[0]),
                                                                           (1705, m.round_log_sizes[1]), (32, 12), (1, 11)))),
        "steps": a.steps, "warmup": a.warmup,
        "ms_per_proof": {k: round(1e3 * min(v), 2) for k, v in times.items()},
        "ms_all_steps": {k: [round(1e3 * x, 2) for x in v] for k, v in times.items()},
        "peak_pool_gb": {k: round(v / 1e9, 2) for k, v in peaks.items()},
        "proof_bytes": len(proofs["device"][0]), "arms_equal": True, "oracle_verifier": verified, "witness_build_s": round(witness_s, 2),
        "timing": "host clock from the call to the proof bytes on the host, minimum over the steps (arms alternate); the host arm's witness "
                  "(witness_build_s) is built before the steps, the device arm starts from the side note",
        "card": card(),
    }
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "keccak_fill.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))
    del proofs
    ctx.close()


if __name__ == "__main__":
    main()
