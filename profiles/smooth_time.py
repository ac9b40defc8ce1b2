"""Time of the four point-cloud smoothing calls on a 2 M-point cloud, on cuda:0.

    python profiles/smooth_time.py [--calls 5] [--out FILE]

The cloud is the target of tests/synth.make_icp_pair(2_000_000, seed=1), with its analytic normals.  After one untimed
call, --calls of each of the following run between CUDA events, whole public calls:
    laplacian         smooth_laplacian() at its defaults (10 passes, max_nn 20, neighbourhoods searched every pass)
    laplacian_fixed   the same with use_fixed_neighborhoods=True
    taubin            smooth_taubin() at its defaults (20 passes)
    taubin_fixed      the same with use_fixed_neighborhoods=True
    mls               smooth_mls() at its defaults (radius 0.05, max_nn 30) and at radius 0.08, max_nn 30
    bilateral         smooth_bilateral() at its defaults and at radius 0.08, max_nn 30
A separate phase runs each call once under torch.profiler for each kernel's device time.  The CPU baseline is the
oracle (oracle/smooth, all host threads) on neighbour lists from scipy.spatial.cKDTree(workers=-1), labelled as such:
one Laplacian pass and one MLS / bilateral call at radius 0.08, max_nn 30.  One JSON line.
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
from tests.synth import make_icp_pair  # noqa: E402

N = 2_000_000


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


def cpu_baseline(tgt, nrm):
    try:
        from scipy.spatial import cKDTree
    except ImportError:
        return None
    from oracle import smooth as osm
    out = {"label": "oracle/smooth on all host threads, neighbours from scipy cKDTree(workers=-1); not the reference",
           "threads": os.cpu_count()}
    t0 = time.perf_counter()
    tree = cKDTree(tgt)
    _, idx = tree.query(tgt, 21, workers=-1)
    t1 = time.perf_counter()
    osm.laplacian_pass(tgt, idx.astype(np.int32), 0.5)
    t2 = time.perf_counter()
    out["laplacian_pass_ms"] = {"search": 1e3 * (t1 - t0), "pass": 1e3 * (t2 - t1)}
    t0 = time.perf_counter()
    d, idx = tree.query(tgt, 30, distance_upper_bound=0.08, workers=-1)
    ok = np.isfinite(d)
    cnt = ok.sum(1).astype(np.int32)
    idx = np.where(ok, idx, -1).astype(np.int32)
    d2 = np.where(ok, d * d, 0).astype(np.float32)
    t1 = time.perf_counter()
    osm.smooth_mls(tgt, 0.08, 30, lists=(idx, d2, cnt, 30))
    t2 = time.perf_counter()
    osm.smooth_bilateral(tgt, nrm, 0.08, 30, 0.05, 0.05, lists=(idx, d2, cnt))
    t3 = time.perf_counter()
    out["radius_0.08_max_nn_30_ms"] = {"search": 1e3 * (t1 - t0), "mls": 1e3 * (t2 - t1), "bilateral": 1e3 * (t3 - t2)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    _, tgt, nrm, _ = make_icp_pair(N, seed=1)
    pc = o3d.t.geometry.PointCloud(tgt).set_point_normals(nrm)
    n = len(tgt)
    calls = {
        "laplacian": lambda: pc.smooth_laplacian(),
        "laplacian_fixed": lambda: pc.smooth_laplacian(use_fixed_neighborhoods=True),
        "taubin": lambda: pc.smooth_taubin(),
        "taubin_fixed": lambda: pc.smooth_taubin(use_fixed_neighborhoods=True),
        "mls": lambda: pc.smooth_mls(),
        "mls_r0.08": lambda: pc.smooth_mls(0.08, 30),
        "bilateral": lambda: pc.smooth_bilateral(),
        "bilateral_r0.08": lambda: pc.smooth_bilateral(0.08, 30),
    }
    res = {"card": card(), "points": n, "calls": args.calls, "times": {}}
    for name, fn in calls.items():
        fn()
        res["times"][name] = stats([event_ms(fn) for _ in range(args.calls)])

    from torch.profiler import ProfilerActivity, profile
    kernels = {}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fn in calls.values():
            fn()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and e.count:
            kernels[e.key] = {"count": e.count, "total_ms": e.device_time_total / 1e3,
                              "mean_ms": e.device_time_total / 1e3 / e.count}
    res["kernels"] = {k: v for k, v in sorted(kernels.items(), key=lambda kv: -kv[1]["total_ms"])[:25]}
    res["cpu_baseline"] = cpu_baseline(tgt, nrm)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
