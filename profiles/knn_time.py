"""Time of the exact k-nearest-neighbour search and its two consumers on a 2 M-point cloud, on cuda:0.

    python profiles/knn_time.py [--calls 20] [--out FILE]

The cloud is the target of tests/synth.make_icp_pair(2_000_000, seed=1); "source" is that pair's source.  After 3
untimed calls, --calls of each of the following run between CUDA events:
    index      o3db_knn_create on the target (o3db_knn_destroy is outside the events)
    knn30      o3db_knn_search of the target on itself, k = 30, into preallocated buffers
    hybrid     o3db_nns_hybrid_search of the target on itself, radius 0.08, max_nn 30, alternated call by call with knn30
    knn1       o3db_knn_search of the source in the target, k = 1
    metrics    a whole PointCloud.compute_metrics(source, target) call (Chamfer, Hausdorff, F-score at 0.01)
    outliers   a whole PointCloud.remove_statistical_outliers(20, 2.0) call
    knn30_out  knn30 on the target with 1 % outliers added uniformly in a box 10 times its bounding box
A separate phase runs 3 index builds and searches under torch.profiler for each kernel's device time.  When scipy
imports, scipy.spatial.cKDTree(workers=-1) building and querying k = 30 on the target is the CPU baseline.  The index's
cell size, cells and blocks, and its mean occupancy (points per occupied cell) are reported.  One JSON line.
"""
import argparse
import ctypes as C
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
from open3d_b200 import _lib as L  # noqa: E402
from tests.synth import make_icp_pair  # noqa: E402

N = 2_000_000


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    name, power, clock, max_clock = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": clock, "max_sm_clock": max_clock}


def stream():
    return int(torch.cuda.current_stream().cuda_stream)


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def stats(ms):
    return {"median_ms": float(np.median(ms)), "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms))}


def knn_create(p):
    h = C.c_void_p()
    L.check(L.lib.o3db_knn_create(p.data_ptr(), int(p.shape[0]), stream(), C.byref(h)))
    return h


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    src, tgt, _, _ = make_icp_pair(N, seed=1)
    p, s = torch.from_numpy(tgt).cuda(), torch.from_numpy(src).cuda()
    rng = np.random.default_rng(2)
    lo, hi = tgt.min(0), tgt.max(0)
    mid, ext = (lo + hi) / 2, hi - lo
    outl = rng.uniform(mid - 5 * ext, mid + 5 * ext, (N // 100, 3)).astype(np.float32)
    po = torch.from_numpy(np.concatenate([tgt, outl])).cuda()
    n = N
    idx = torch.empty((len(po), 30), dtype=torch.int32, device="cuda")
    d2 = torch.empty((len(po), 30), dtype=torch.float32, device="cuda")
    hcnt = torch.empty((n,), dtype=torch.int32, device="cuda")
    geo = o3d.t.geometry
    pc_t, pc_s = geo.PointCloud(p), geo.PointCloud(s)

    h = knn_create(p)
    ho = knn_create(po)
    nns = C.c_void_p()
    L.check(L.lib.o3db_nns_create(p.data_ptr(), n, 0.08, stream(), C.byref(nns)))
    cell, ncell, nblk = C.c_double(), C.c_int64(), C.c_int64()
    L.check(L.lib.o3db_knn_index_stats(h, C.byref(cell), C.byref(ncell), C.byref(nblk)))

    def knn30():
        L.check(L.lib.o3db_knn_search(h, p.data_ptr(), n, 30, L.INDEX_INT32, idx.data_ptr(), d2.data_ptr(), stream()))

    def hybrid():
        L.check(L.lib.o3db_nns_hybrid_search(nns, p.data_ptr(), n, 0.08, 30, idx.data_ptr(), d2.data_ptr(),
                                             hcnt.data_ptr(), stream()))

    def knn1():
        L.check(L.lib.o3db_knn_search(h, s.data_ptr(), n, 1, L.INDEX_INT32, idx.data_ptr(), d2.data_ptr(), stream()))

    def knn30_out():
        L.check(L.lib.o3db_knn_search(ho, po.data_ptr(), len(po), 30, L.INDEX_INT32, idx.data_ptr(), d2.data_ptr(),
                                      stream()))

    def metrics():
        pc_s.compute_metrics(pc_t, (geo.Metric.ChamferDistance, geo.Metric.HausdorffDistance, geo.Metric.FScore))

    def outliers():
        pc_t.remove_statistical_outliers(20, 2.0)

    def index():
        nonlocal_h.append(knn_create(p))

    nonlocal_h = []
    # points per occupied cell: the distinct cells of the index's cell size that the points fall in (binned here in
    # f64 from the bounding box, as the index bins in f32)
    c = cell.value
    g = np.floor((tgt - lo) / c).astype(np.int64)
    occupied = len(np.unique(g[:, 0] * (1 << 42) + g[:, 1] * (1 << 21) + g[:, 2]))
    for fn in (knn30, hybrid, knn1, knn30_out, metrics, outliers):
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    res = {k: [] for k in ("index", "knn30", "hybrid", "knn1", "knn30_out", "metrics", "outliers")}
    for _ in range(args.calls):
        res["index"].append(event_ms(index))
        L.lib.o3db_knn_destroy(nonlocal_h.pop())
        res["knn30"].append(event_ms(knn30))
        res["hybrid"].append(event_ms(hybrid))
        res["knn1"].append(event_ms(knn1))
        res["knn30_out"].append(event_ms(knn30_out))
        res["metrics"].append(event_ms(metrics))
        res["outliers"].append(event_ms(outliers))
    out = {"workload": "make_icp_pair(2_000_000, seed=1)", "card": card(), "calls": args.calls,
           "times": {k: stats(v) for k, v in res.items()},
           "index": {"cell_size": c, "cells": ncell.value, "blocks": nblk.value, "occupied_cells": occupied,
                     "points_per_occupied_cell": n / occupied}}

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            index()
            L.lib.o3db_knn_destroy(nonlocal_h.pop())
            knn30()
            hybrid()
            knn1()
            knn30_out()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and e.count:
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            kern[e.key[:80]] = {"count": e.count, "avg_us": t / e.count}
    out["kernels"] = dict(sorted(kern.items(), key=lambda kv: -kv[1]["avg_us"] * kv[1]["count"])[:20])
    try:
        from scipy.spatial import cKDTree
        t0 = time.perf_counter()
        tree = cKDTree(tgt)
        t1 = time.perf_counter()
        tree.query(tgt, k=30, workers=-1)
        t2 = time.perf_counter()
        out["cpu_baseline_scipy_ckdtree"] = {"build_ms": (t1 - t0) * 1e3, "query_k30_ms": (t2 - t1) * 1e3,
                                             "host_threads": os.cpu_count()}
    except ImportError:
        out["cpu_baseline_scipy_ckdtree"] = None
    L.lib.o3db_knn_destroy(h)
    L.lib.o3db_knn_destroy(ho)
    L.lib.o3db_nns_destroy(nns)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
