"""Time of PointCloud.cluster_dbscan on a 2 M-point cloud, on cuda:0.

    python profiles/dbscan_time.py [--calls 5] [--out FILE]

The cloud is the target of tests/synth.make_icp_pair(2_000_000, seed=1) (a height field sampled every 0.02); "out"
is the same cloud with 1 % outliers added uniformly in a box 10 times its bounding box.  After one untimed call, --calls
whole cluster_dbscan calls run between CUDA events for each of eps 0.03 and 0.05 at min_points 10, on both clouds.
Each call's labels are checked against the CPU oracle (oracle/dbscan on every host thread), whose time is the CPU
baseline (kind "port": a restatement of upstream's algorithm, not upstream's own code).  A separate phase runs each
call once under torch.profiler for each kernel's device time.  The card's name, power limit and SM clock are read
before and after.  One JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import open3d_b200 as o3d  # noqa: E402
from oracle import dbscan as od  # noqa: E402
from tests.synth import make_icp_pair  # noqa: E402

N = 2_000_000
MIN_POINTS = 10


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    name, power, clock, max_clock = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": clock, "max_sm_clock": max_clock}


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def stats(ms):
    return {"median_ms": float(np.median(ms)), "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "dbscan_time.py measures on cuda:0"
    torch.cuda.set_device(0)
    res = {"card": card(), "points": N, "min_points": MIN_POINTS, "calls": args.calls, "times": {}, "clusters": {},
           "cpu_baseline": {"kind": "port", "impl": "oracle/dbscan, grid neighbour pass on every host thread and "
                                                     "upstream's sequential labelling", "threads": os.cpu_count()}}
    tgt = make_icp_pair(N, seed=1)[1]
    rng = np.random.default_rng(2)
    lo, hi = tgt.min(0), tgt.max(0)
    mid, ext = (lo + hi) / 2, hi - lo
    outl = rng.uniform(mid - 5 * ext, mid + 5 * ext, (N // 100, 3)).astype(np.float32)
    clouds = {"": tgt, "_out": np.concatenate([tgt, outl])}
    calls = {}
    for suffix, p in clouds.items():
        pc = o3d.t.geometry.PointCloud(p)
        for eps in (0.03, 0.05):
            calls[f"eps{eps}{suffix}"] = (p, eps, lambda pc=pc, eps=eps: pc.cluster_dbscan(eps, MIN_POINTS))
    for name, (p, eps, fn) in calls.items():
        got = fn().cpu().numpy()
        res["times"][name] = stats([event_ms(fn) for _ in range(args.calls)])
        t = time.perf_counter()
        want = od.cluster_dbscan(p, eps, MIN_POINTS)
        res["cpu_baseline"][name + "_ms"] = (time.perf_counter() - t) * 1e3
        res["clusters"][name] = {"points": len(p), "clusters": int(want.max()) + 1, "noise": int((want < 0).sum()),
                                 "equal_to_oracle": bool(np.array_equal(got, want))}

    from torch.profiler import ProfilerActivity, profile
    kernels = {}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _, _, fn in calls.values():
            fn()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and e.count:
            kernels[e.key] = {"count": e.count, "total_ms": e.device_time_total / 1e3,
                              "mean_ms": e.device_time_total / 1e3 / e.count}
    res["kernels"] = {k: v for k, v in sorted(kernels.items(), key=lambda kv: -kv[1]["total_ms"])[:25]}
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
