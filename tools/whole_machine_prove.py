"""Time whole GPU proofs of the v1 main component, its eight base extensions and the keccak extension as one machine
(nexus_zkvm_b200/whole_machine.py), from host columns and from device-filled extension trees, and time RamInitFinal's device fill.

    python tools/whole_machine_prove.py [--log-size 20] [--log-perms 12] [--steps 3] [--warmup 1] [--fill-calls 20] [--out-dir DIR]

Two arms alternate step by step after the warm-up: `host` proves from the host columns (machine.prove with the tree-1 columns built on the
host, RamInitFinal and the keccak blocks included), `device` from NexusV1KeccakMachine.device_trees (tree 0 and the main component's,
FinalReg's and BitOpMultiplicity's columns uploaded, RamInitFinal filled by nb200_ram_init_final_trace, the keccak extension by
nb200_keccak_main_trace and every table column counted by nb200_table_multiplicities_first_row), both timed
with a host clock from the call to the proof bytes on the host.  The host arm's columns are built once, before the steps; the device arm
builds its main columns inside the timed call.  The two arms' proof bytes must be equal; the oracle's verifier checks the last one.  The peak
of each arm is the memory pool's used-memory high-water mark over its steps (reset before each step).  RamInitFinal's fill alone is timed with
CUDA events on the library's stream (median of --fill-calls calls after a warm-up call; the side note's host checks and copies and the one
device-to-host read of the address count included).  Writes whole_machine_prove.json (also printed) to --out-dir (default: <temp
dir>/whole_machine_prove) with the card's name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from keccak_prove import PoolHigh, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-size", type=int, default=20)
    ap.add_argument("--log-perms", type=int, default=12)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--fill-calls", type=int, default=20)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "whole_machine_prove"))
    ap.add_argument("--no-verify", action="store_true")
    a = ap.parse_args()
    import torch

    import nexus_zkvm_b200 as nb
    from nexus_zkvm_b200 import machine as M
    from nexus_zkvm_b200.prover import CudaBackend
    from nexus_zkvm_b200.whole_machine import NexusV1KeccakMachine

    assert torch.cuda.is_available(), "needs a GPU"
    t0 = time.perf_counter()
    m = NexusV1KeccakMachine(a.log_size, 1 << a.log_perms, seed=a.seed)
    cols = m.fill_main_trace()
    witness_s = time.perf_counter() - t0
    side_note, (ia, iv) = m.side_note(), m.initial_memory()
    stream = torch.cuda.Stream()
    ctx = nb.Context(0, stream=stream.cuda_stream)   # the library's work on a stream the CUDA events can be recorded on
    backend = CudaBackend(ctx)
    pool = PoolHigh()

    out_batch = ctx.alloc(10, m.ram_log_size)
    ctx.ram_init_final_trace(*side_note, ia, iv, m.ram_log_size, out=out_batch)
    ctx.sync()
    fill_ms = []
    for _ in range(a.fill_calls):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream)
        ctx.ram_init_final_trace(*side_note, ia, iv, m.ram_log_size, out=out_batch)
        ev1.record(stream)
        ev1.synchronize()
        fill_ms.append(ev0.elapsed_time(ev1))
    out_batch.free()

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
    proof, claimed, aux = proofs["device"]
    assert M.verify_claimed_sums(claimed), "the claimed sums do not cancel"
    verified = None
    if not a.no_verify:
        from tests.oracle_backend import verify_with_replayed_transcript
        verify_with_replayed_transcript(m, proof, claimed, aux)
        verified = "accepted"
    out = {
        "workload": "NexusV1KeccakMachine: v1 main component + the eight base extensions + the keccak extension, 15 components",
        "log_size": a.log_size, "permutations": m.n_perms, "buffers": m.n_buffers, "ram_addresses": int(ia.size),
        "component_log_sizes": m.log_sizes, "columns": m.air.n_columns(),
        "config": dict(pow_bits=5, log_blowup=1, log_last=0, n_queries=3),
        "ram_fill_ms_median": round(statistics.median(fill_ms), 3), "ram_fill_ms_all": [round(x, 3) for x in fill_ms],
        "fill_calls": a.fill_calls,
        "steps": a.steps, "warmup": a.warmup,
        "ms_per_proof": {k: round(1e3 * min(v), 2) for k, v in times.items()},
        "ms_all_steps": {k: [round(1e3 * x, 2) for x in v] for k, v in times.items()},
        "peak_pool_gb": {k: round(v / 1e9, 2) for k, v in peaks.items()},
        "proof_bytes": len(proof), "arms_equal": True, "claimed_sums_cancel": True, "oracle_verifier": verified,
        "witness_build_s": round(witness_s, 2),
        "timing": "host clock from the call to the proof bytes on the host, minimum over the steps (arms alternate); the host arm's columns "
                  "(witness_build_s) are built before the steps, the device arm starts from the side note and builds the main columns in the call",
        "card": card(),
    }
    os.makedirs(a.out_dir, exist_ok=True)
    with open(os.path.join(a.out_dir, "whole_machine_prove.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))
    del proofs
    ctx.close()


if __name__ == "__main__":
    main()
