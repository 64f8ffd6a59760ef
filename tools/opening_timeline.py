#!/usr/bin/env python
"""Where the GPU sits idle in the opening stages of one proof (composition commit to the proof bytes).

Runs one warmed-up whole proof the way bench.py builds it (nexus_v1, trees 0 and 1 resident in HBM) under torch.profiler with CUDA
activities, with NB200_TRACE=1 so that the library marks its stages (each mark drains the stream and prints the wall-clock time of the
mark). For every stage from `composition: coefficients + commit` to the end it reports the wall time, the busy time of the GPU (the union
of kernel, copy and memset intervals), their difference (idle time), and the kernel launches, copies and stream syncs issued in the stage.
The trace mark's own drain of the stream is not counted among the syncs.

    python tools/opening_timeline.py --out DIR [--log-rows 20] [--warmup 2]

DIR receives trace.json (Chrome trace), summary.json and summary.md.
"""
import argparse
import json
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

FIRST_STAGE = "composition: coefficients + commit"
MARK = re.compile(r"^\[nb200\] (.+?)\s+([0-9.]+) ms @(\d+)$")
LAUNCH = ("cudaLaunchKernel", "cuLaunchKernel", "cudaLaunchKernelExC", "cuLaunchKernelEx")
SYNC = ("cudaStreamSynchronize", "cudaDeviceSynchronize", "cuStreamSynchronize", "cuCtxSynchronize", "cudaEventSynchronize")
COPY = ("cudaMemcpyAsync", "cudaMemcpy", "cuMemcpyAsync", "cuMemcpyHtoDAsync_v2", "cuMemcpyDtoHAsync_v2")


def build_resident(m, be, ctx, np, log_rows, config):
    """Trees 0 and 1 uploaded once, in finalized (coset) order: the HBM-resident proof bench.py times."""
    import bench
    all_cols, _ = bench.fill_trace(m, 0)
    up = be.prover(m.words, config)
    pre_cols = []
    for c in m.preprocessed_columns():
        a = np.asarray(c)
        pre_cols += list(a.astype(np.uint32)) if a.ndim == 2 else [a]
    t0 = up._batches_from_host(pre_cols, True)
    wide = np.stack([np.asarray(c, dtype=np.uint32) for c in all_cols[:m.n_main]])
    t1 = [ctx.upload(wide, coset_order=True)] + [ctx.upload(np.asarray(c, dtype=np.uint32)[None, :], coset_order=True) for c in all_cols[m.n_main:]]
    return t0, t1


def union_ms(intervals, lo, hi):
    """Length (ms) of the union of [a, b) intervals (µs) clipped to [lo, hi)."""
    iv = sorted((max(a, lo), min(b, hi)) for a, b in intervals if b > lo and a < hi)
    tot, cur_a, cur_b = 0.0, None, None
    for a, b in iv:
        if cur_b is None or a > cur_b:
            if cur_b is not None:
                tot += cur_b - cur_a
            cur_a, cur_b = a, b
        else:
            cur_b = max(cur_b, b)
    if cur_b is not None:
        tot += cur_b - cur_a
    return tot / 1e3


def summarize(trace, marks):
    base_ns = int(trace.get("baseTimeNanoseconds", 0))
    evs = [e for e in trace["traceEvents"] if e.get("ph") == "X"]
    dev = [(float(e["ts"]), float(e["ts"]) + float(e.get("dur", 0))) for e in evs if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    rt = [(e["name"], float(e["ts"])) for e in evs if e.get("cat") in ("cuda_runtime", "cuda_driver")]
    rows, prev = [], None
    for name, wall_ms, t_ns in marks:
        t_us = (t_ns - base_ns) / 1e3
        if prev is not None and (rows or name == FIRST_STAGE):
            lo, hi = prev, t_us
            busy = union_ms(dev, lo, hi)
            in_win = [n for n, ts in rt if lo <= ts < hi]
            syncs = sum(1 for n in in_win if n in SYNC)
            rows.append({"stage": name, "wall_ms": wall_ms, "busy_ms": busy, "idle_ms": wall_ms - busy,
                         "launches": sum(1 for n in in_win if n in LAUNCH), "copies": sum(1 for n in in_win if n in COPY),
                         "syncs": max(syncs - 1, 0)})
        prev = t_us
    tot = {k: sum(r[k] for r in rows) for k in ("wall_ms", "busy_ms", "idle_ms", "launches", "copies", "syncs")}
    return rows, tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--log-rows", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    os.environ["NB200_TRACE"] = "1"          # read when the context is created
    import numpy as np
    import torch
    from torch.profiler import profile, ProfilerActivity
    import bench
    import nexus_zkvm_b200 as nb
    from nexus_zkvm_b200 import machine as M
    from nexus_zkvm_b200.prover import CudaBackend

    os.makedirs(a.out, exist_ok=True)
    bargs = bench.parse(["--log-rows", str(a.log_rows)])
    m = bench.make_machine(bargs)
    stream = torch.cuda.Stream()
    ctx = nb.Context(torch.cuda.current_device(), stream=stream.cuda_stream)
    be = CudaBackend(ctx)
    # the library prints its marks on file descriptor 2: send them to a file for the run, then read the profiled proof's lines back
    log = tempfile.TemporaryFile(mode="w+b")
    saved = os.dup(2)
    os.dup2(log.fileno(), 2)
    try:
        with torch.cuda.stream(stream):
            ctx.precompute_twiddles(a.log_rows + 3)
            res = build_resident(m, be, ctx, np, a.log_rows, bench.CONFIG)
            for _ in range(a.warmup):
                M.prove(m, be, None, None, config=bench.CONFIG, resident=res)
            torch.cuda.synchronize()
            sys.stderr.flush()
            start = log.tell()
            l0 = ctx.launches
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                proof, _claimed, _aux = M.prove(m, be, None, None, config=bench.CONFIG, resident=res)
                torch.cuda.synchronize()
            launches = ctx.launches - l0
    finally:
        os.dup2(saved, 2)
        os.close(saved)
    log.seek(start)
    marks = []
    for line in log.read().decode(errors="replace").splitlines():
        mm = MARK.match(line.strip())
        if mm:
            marks.append((mm.group(1), float(mm.group(2)), int(mm.group(3))))
    path = os.path.join(a.out, "trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        trace = json.load(f)
    rows, tot = summarize(trace, marks)
    meta = {"log_rows": a.log_rows, "machine": "nexus_v1", "gpu": torch.cuda.get_device_name(), "proof_bytes": len(proof),
            "gpu_launches_per_proof": launches, "note": "NB200_TRACE drains the stream at every mark: wall times are those of a traced proof"}
    with open(os.path.join(a.out, "summary.json"), "w") as f:
        json.dump({"meta": meta, "stages": rows, "total": tot}, f, indent=1)
    md = ["| stage | wall ms | busy ms | idle ms | launches | copies | syncs |", "|---|---|---|---|---|---|---|"]
    for r in rows + [dict(tot, stage="**sum**")]:
        md.append(f"| {r['stage']} | {r['wall_ms']:.2f} | {r['busy_ms']:.2f} | {r['idle_ms']:.2f} | {r['launches']} | {r['copies']} | {r['syncs']} |")
    text = "\n".join(md)
    with open(os.path.join(a.out, "summary.md"), "w") as f:
        f.write(json.dumps(meta) + "\n\n" + text + "\n")
    print(json.dumps(meta))
    print(text)


if __name__ == "__main__":
    main()
