"""Time one constraint check (nb200_check_constraints) of the v1 main component on one GPU.

    python tools/check_constraints_time.py [--log-size 20] [--reps 20] [--out FILE]

The three trees of NexusV1Machine(log_size) with its padding witness are committed as machine.prove commits them; then the check of
component 0 is run `reps` times after a warm-up (the generated kernel is loaded on first use), each bracketed by CUDA events recorded on
the library's stream.  One call is: parameter upload, two memsets, the check kernel, the copy back of the report.  Prints one JSON line
with the card name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return dict(zip(q.split(","), (x.strip() for x in r.stdout.strip().split(",")))) if r.returncode == 0 else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-size", type=int, default=20)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch

    import nexus_zkvm_b200 as nb
    from nexus_zkvm_b200 import machine as M
    from nexus_zkvm_b200.nexus_v1 import NexusV1Machine
    from nexus_zkvm_b200.prover import CudaBackend

    assert torch.cuda.is_available(), "needs a GPU"
    stream = torch.cuda.Stream()
    ctx = nb.Context(0, stream=stream.cuda_stream)
    m = NexusV1Machine(a.log_size)
    _ch, prover, params, claimed, _roots, _ls = M._commit_trees(m, CudaBackend(ctx), m.fill_main_trace(seed=1), None, None, b"", None)
    assert M.verify_claimed_sums(claimed)
    assert prover.check_constraints(0, params) == []          # warm-up; the padding witness satisfies every constraint
    ms = []
    for _ in range(a.reps):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        prover.check_constraints(0, params)
        t1.record(stream)
        t1.synchronize()
        ms.append(t0.elapsed_time(t1))
    ms.sort()
    res = {"what": "nb200_check_constraints, NexusV1Machine main component", "log_size": a.log_size, "reps": a.reps,
           "ms_median": ms[len(ms) // 2], "ms_min": ms[0], "ms_max": ms[-1], "gpu": card()}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
