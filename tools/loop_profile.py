#!/usr/bin/env python
"""Per-kernel device time of one device-resident ICP call under torch.profiler (CUDA activities).

    python tools/loop_profile.py OUT_DIR [N] [p2p|combined] [ITERS]

A warm-up call, then ONE estimate() of ITERS iterations (tol = 0, L2 flushed before every iteration, as bench.py times
it) inside the profiler. Writes OUT_DIR/loop_profile_<metric>_<n>.json: every kernel launch of that call in stream
order (name, start relative to the first launch, duration, both in microseconds), and per kernel name the count, total
and mean. Also prints the per-name table. The flush memsets are listed like any other launch.
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cilantro_b200 import capi, synth  # noqa: E402


def main():
    out_dir = sys.argv[1]
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 1_000_000
    metric = sys.argv[3] if len(sys.argv) > 3 else "p2p"
    iters = int(sys.argv[4]) if len(sys.argv) > 4 else 15
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    ctx = capi.Context(0)
    dst, src, nrm, _ = synth.icp_pair(n, seed=1, noise=0.001, with_normals=(metric == "combined"))
    icp = capi.Icp(ctx, capi.Cloud(ctx, dst, nrm), capi.Cloud(ctx, src))
    kw = dict(metric=metric, tol=0.0, max_d2=np.float32((0.02 if n <= 2_000_000 else 0.01) ** 2), max_iter=iters,
              timing=0, flush_l2=True)
    if metric == "combined":
        kw.update(w_pt=0.1, w_pl=1.0)
    icp.estimate(**kw)
    ctx.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        r = icp.estimate(**kw)
        ctx.synchronize()
    events = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    events.sort(key=lambda e: e.time_range.start)
    t0 = events[0].time_range.start if events else 0
    launches = [{"name": e.name, "start_us": float(e.time_range.start - t0),
                 "dur_us": float(e.time_range.end - e.time_range.start)} for e in events]
    per_name = {}
    for e in launches:
        s = per_name.setdefault(e["name"], {"count": 0, "total_us": 0.0})
        s["count"] += 1
        s["total_us"] += e["dur_us"]
    for s in per_name.values():
        s["mean_us"] = s["total_us"] / s["count"]
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, f"loop_profile_{metric}_{n}.json")
    with open(path, "w") as f:
        json.dump({"n": n, "metric": metric, "iterations": r["iterations"], "num_corr": r["num_corr"],
                   "kernel_launches": r["kernel_launches"], "device": torch.cuda.get_device_name(0),
                   "per_name": per_name, "launches": launches}, f, indent=1)
    for name, s in sorted(per_name.items(), key=lambda kv: -kv[1]["total_us"]):
        print(f"{s['count']:4d} x {s['mean_us']:9.2f} us = {s['total_us']:9.1f} us  {name}")
    print("wrote", path)
    ctx.close()


if __name__ == "__main__":
    main()
