"""Time whole GPU proofs of the keccak precompile extension (nexus_zkvm_b200/keccak.py: its six components, witness from Keccak-f[1600]).

    python tools/keccak_prove.py [--log-perms 14] [--steps 3] [--warmup 1] [--out-dir DIR]

KeccakMachine(log_perms) holds 2^log_perms - 1 permutations: KeccakRound 0 has 2^(log_perms + 4) rows, KeccakRound 1 half of that, the memory
check 2^log_perms.  One step = machine.prove on the CUDA backend from the host trace (tree commits with their uploads, interaction trace, quotients,
FRI, decommitment), timed with a host clock that ends when the proof bytes are back on the host.  The witness is built once, before the timed
steps.  Device memory in use (cudaMemGetInfo, whole device) is sampled every 20 ms over the timed steps.  The last proof is checked by the
oracle's verifier.  Writes keccak_prove.json (also printed) to --out-dir (default: <temp dir>/keccak_prove) with the card's name, power limit and SM clock read in the same run."""
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
    a = ap.parse_args()
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


if __name__ == "__main__":
    main()
