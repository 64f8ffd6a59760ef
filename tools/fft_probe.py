"""Event-timed probe of the commit transforms (fused iFFT + LDE) for one batch, beside the per-transform passes.
    python tools/fft_probe.py [log_rows] [n_cols] [reps]"""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import nexus_zkvm_b200 as nb

log_rows = int(sys.argv[1]) if len(sys.argv) > 1 else 20
n_cols = int(sys.argv[2]) if len(sys.argv) > 2 else 1012
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 5
P = (1 << 31) - 1
dev = torch.device("cuda", 0)
stream = torch.cuda.Stream(device=dev)
ctx = nb.Context(0, stream=stream.cuda_stream)
with torch.cuda.stream(stream):
    ev_t = torch.randint(0, P, (n_cols, 1 << log_rows), device=dev, dtype=torch.int32)
    ev = ctx.wrap_device(ev_t.data_ptr(), n_cols, log_rows)
    ctx.precompute_twiddles(log_rows + 1)
    co, lde = ctx.interpolate_evaluate(ev, 1)
    times = []
    for _ in range(reps + 2):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        ctx.interpolate_evaluate(ev, 1, co, lde)
        b.record(stream)
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    t = sorted(times[2:])[len(times[2:]) // 2]
    # the per-transform passes (nb200_interpolate + nb200_evaluate) in the same process, for comparison
    tl = []
    tmp = torch.empty_like(ev_t)
    scw = ctx.wrap_device(tmp.data_ptr(), n_cols, log_rows)
    for _ in range(3):
        tmp.copy_(ev_t)
        a, b, c = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        a.record(stream); ctx.interpolate(scw); b.record(stream)
        ctx._chk(nb.lib().nb200_evaluate(ctx._h, scw._h, C.c_uint32(1), lde._h)); c.record(stream)
        torch.cuda.synchronize()
        tl.append((a.elapsed_time(b), b.elapsed_time(c)))
    elems = n_cols << log_rows
    print(json.dumps({"log_rows": log_rows, "n_cols": n_cols, "ms": round(t, 3), "GBps_12B": round(12.0 * elems / (t * 1e-3) / 1e9, 1), "all_ms": [round(x, 3) for x in times],
                      "legacy_ifft_ms": round(min(x[0] for x in tl), 3), "legacy_lde_ms": round(min(x[1] for x in tl), 3)}))
