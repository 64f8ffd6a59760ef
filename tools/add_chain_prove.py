"""Time GPU proofs of the reference's ADD-chain benchmark as an executing v1 trace (nexus_zkvm_b200/add_chain.py), from host columns and from
device-filled trees, and time the main trace's device fill (nb200_v1_main_trace).  `--program alu` does the same for add_chain.AluMachine, a
seeded program of RV32I's 19 ALU instructions (filled by nb200_v1_alu_trace), and writes alu_program_prove.json instead; `--program
control` for add_chain.ControlMachine, a seeded looping program that adds the branches, JAL, JALR, LUI and AUIPC (filled by
nb200_v1_control_trace), and writes control_program_prove.json.

    python tools/add_chain_prove.py [--program {add-chain,alu,control}] [--log-sizes 16 18 20] [--steps 3] [--warmup 1] [--fill-calls 20] [--out-dir DIR]

For each log size n: AddChainMachine(n), 2^n executed steps and no padding rows.  Two arms alternate step by step after the warm-up: `host`
proves from the host columns (machine.prove with tree 1 built on the host), `device` from AddChainMachine.device_trees (tree 0 and FinalReg
uploaded, the main component filled on the device from the step record, every table column counted on the device), both timed with a host
clock from the call to the proof bytes on the host.  The host arm's columns and the step record are built once, before the steps (their
build time is reported as witness_build_s).  Rate = executed steps / wall second of the fastest step, in kHz, the reference's metric
(benchmarks/src/runner.rs:276-284: total_steps / duration / 1000).  The two arms' proof bytes must be equal; the oracle's verifier checks the
last one.  The peak of each arm is the memory pool's used-memory high-water mark over its steps.  The fill alone is timed with CUDA events
on the library's stream (median of --fill-calls calls after a warm-up call; the step record's host checks and upload included).  Writes
add_chain_prove.json (also printed) to --out-dir (default: <temp dir>/add_chain_prove) with the card's name, power limit and SM clock."""
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


def one_size(a, log_size, ctx, backend, stream, pool):
    import torch

    from nexus_zkvm_b200 import machine as M
    from nexus_zkvm_b200.add_chain import AddChainMachine, AluMachine, ControlMachine

    t0 = time.perf_counter()
    m = {"alu": AluMachine, "control": ControlMachine, "add-chain": AddChainMachine}[a.program](log_size)
    cols = m.fill_main_trace()
    witness_s = time.perf_counter() - t0
    out_batch = ctx.alloc(347, log_size)
    m.device_fill(ctx, out=out_batch)
    ctx.sync()
    fill_ms = []
    for _ in range(a.fill_calls):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream)
        m.device_fill(ctx, out=out_batch)
        ev1.record(stream)
        ev1.synchronize()
        fill_ms.append(ev0.elapsed_time(ev1))
    arms = {"host": lambda: M.prove(m, backend, cols, None),
            "device": lambda: M.prove(m, backend, None, None, resident=m.device_trees(ctx, out=out_batch))}
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
    n_steps = m.n_steps
    res = {
        "log_size": log_size, "executed_steps": n_steps, "component_log_sizes": m.log_sizes, "columns": m.air.n_columns(),
        "fill_ms_median": round(statistics.median(fill_ms), 3), "fill_ms_all": [round(x, 3) for x in fill_ms],
        "ms_per_proof": {k: round(1e3 * min(v), 2) for k, v in times.items()},
        "ms_all_steps": {k: [round(1e3 * x, 2) for x in v] for k, v in times.items()},
        "khz": {k: round(n_steps / min(v) / 1e3, 1) for k, v in times.items()},
        "peak_pool_gb": {k: round(v / 1e9, 2) for k, v in peaks.items()},
        "proof_bytes": len(proof), "arms_equal": True, "claimed_sums_cancel": True, "oracle_verifier": verified,
        "witness_build_s": round(witness_s, 2),
    }
    del proofs
    out_batch.free()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--program", choices=["add-chain", "alu", "control"], default="add-chain")
    ap.add_argument("--log-sizes", type=int, nargs="+", default=[16, 18, 20])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--fill-calls", type=int, default=20)
    ap.add_argument("--out-dir", default=os.path.join(tempfile.gettempdir(), "add_chain_prove"))
    ap.add_argument("--no-verify", action="store_true")
    a = ap.parse_args()
    import torch

    import nexus_zkvm_b200 as nb
    from nexus_zkvm_b200.prover import CudaBackend

    assert torch.cuda.is_available(), "needs a GPU"
    stream = torch.cuda.Stream()
    ctx = nb.Context(0, stream=stream.cuda_stream)   # the library's work on a stream the CUDA events can be recorded on
    backend = CudaBackend(ctx)
    pool = PoolHigh()
    sizes = [one_size(a, ls, ctx, backend, stream, pool) for ls in a.log_sizes]
    workload = {"add-chain": "AddChainMachine: the reference's ADD-chain benchmark (addi x1,x0,1; add x_k,x_j,x_i), 2^n executed steps, v1 "
                             "main component with DecodingCheck R / I + the eight base extensions",
                "alu": "AluMachine: alu_program(n, seed=0), 2^n executed steps over RV32I's 19 ALU instructions (ADD ... SRAI), v1 main "
                       "component with DecodingCheck R / I and SltuChip, SltChip, SllChip, SrlChip, SraChip + the eight base extensions",
                "control": "ControlMachine: control_program(n, seed=0), a looping program over the 19 ALU instructions and RV32I's branches, "
                           "JAL, JALR, LUI and AUIPC, 2^n executed steps, v1 main component with DecodingCheck R / I / B / U / J, the ALU "
                           "chips and the ten control-flow chips + the eight base extensions"}
    out = {
        "workload": workload[a.program],
        "config": dict(pow_bits=5, log_blowup=1, log_last=0, n_queries=3),
        "steps": a.steps, "warmup": a.warmup, "fill_calls": a.fill_calls,
        "timing": "host clock from the call to the proof bytes on the host, minimum over the steps (arms alternate); kHz = executed steps / "
                  "that time / 1000; the host arm's columns are built before the steps (witness_build_s), the device arm fills the main trace "
                  "from the step record in the call",
        "sizes": sizes,
        "card": card(),
    }
    os.makedirs(a.out_dir, exist_ok=True)
    name = {"alu": "alu_program_prove.json", "control": "control_program_prove.json", "add-chain": "add_chain_prove.json"}[a.program]
    with open(os.path.join(a.out_dir, name), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
