"""Times registration.compute_fpfh_feature and correspondences_from_features on the GPU and writes one JSON file
(default profiles/h100_fpfh.json).  Whole calls: medians of CUDA-event timings after warm-up.  Per-kernel times (wide
search, SPFH, FPFH, feature 1-NN): torch.profiler in a separate pass.  The card name, power limit and SM clock are read
in the same run.  Beside them, the CPU oracle's and the reference's FPFH pass (oracle/_ref/libo3dref_fpfh.so) on 8 host
threads, over the library's own hybrid lists at max_nn 30 (the public hybrid search stops at 32)."""
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

reg = o3d.t.pipelines.registration


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def timed(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def kernel_ms(fn, names):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in names}
    for e in prof.events():
        for k in names:
            if k in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
                out[k] += e.device_time_total / 1000.0 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
    return out


def host_passes(pts, nrm, radius):
    """The oracle's and the reference's FPFH pass over the library's hybrid lists (max_nn 30), 8 host threads."""
    from oracle import fpfh as of
    os.environ["OMP_NUM_THREADS"] = "8"
    n = len(pts)
    p = torch.from_numpy(pts).cuda()
    nns = C.c_void_p()
    L.check(L.lib.o3db_nns_create(p.data_ptr(), n, radius, None, C.byref(nns)))
    hi = torch.empty((n, 30), dtype=torch.int32, device="cuda")
    hd = torch.empty((n, 30), dtype=torch.float32, device="cuda")
    hc = torch.empty((n,), dtype=torch.int32, device="cuda")
    L.check(L.lib.o3db_nns_hybrid_search(nns, p.data_ptr(), n, radius, 30, hi.data_ptr(), hd.data_ptr(), hc.data_ptr(),
                                         None))
    torch.cuda.synchronize()
    L.lib.o3db_nns_destroy(nns)
    idx, d2, cnt = hi.cpu().numpy(), hd.cpu().numpy(), hc.cpu().numpy()
    t0 = time.perf_counter()
    want = of.fpfh_from_lists(pts, nrm, idx, d2, cnt)
    res = {"oracle_ms": (time.perf_counter() - t0) * 1e3}
    ref = os.path.join(ROOT, "oracle", "_ref", "libo3dref_fpfh.so")
    if os.path.exists(ref):
        R = C.CDLL(ref)
        R.ref_compute_fpfh_feature_f32.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                                   C.c_int64, C.c_void_p, C.c_void_p]
        out = np.zeros((n, 33), np.float32)
        t0 = time.perf_counter()
        R.ref_compute_fpfh_feature_f32(pts.ctypes.data, nrm.ctypes.data, n, idx.ctypes.data, d2.ctypes.data, 30,
                                       cnt.ctypes.data, out.ctypes.data)
        res["reference_ms"] = (time.perf_counter() - t0) * 1e3
        res["reference_equals_oracle"] = bool(np.array_equal(out.view(np.int32), want.view(np.int32)))
    got = reg.compute_fpfh_feature(o3d.t.geometry.PointCloud(pts).set_point_normals(nrm), 30, radius)
    res["library_equals_oracle"] = bool(np.array_equal(got.cpu().numpy().view(np.int32), want.view(np.int32)))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_fpfh.json"))
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    info = gpu_info()
    res = {"gpu": info, "fpfh": [], "correspondences": [], "host": {}}
    clouds = {}
    _, tgt, nrm, _ = make_icp_pair(200_000, seed=2, spacing=0.005)
    clouds["scan_200k"] = (tgt, nrm, 5 * 0.005)
    _, tgt, nrm, _ = make_icp_pair(2_000_000, seed=3)
    clouds["scan_2m"] = (tgt, nrm, 5 * 0.02)
    kernels = ("knn_lists_kernel", "knn_probe", "fpfh_spfh_kernel", "fpfh_kernel")
    for name, (pts, nrm, radius) in clouds.items():
        cloud = o3d.t.geometry.PointCloud(pts).set_point_normals(nrm)
        for max_nn in (30, 100):
            fn = lambda: reg.compute_fpfh_feature(cloud, max_nn, radius)  # noqa: E731
            row = {"cloud": name, "n": len(pts), "radius": radius, "max_nn": max_nn, "whole_call_ms": timed(fn, args.reps)}
            row["kernel_ms"] = kernel_ms(fn, kernels)
            res["fpfh"].append(row)
            print(json.dumps(row), flush=True)
    feats = reg.compute_fpfh_feature(o3d.t.geometry.PointCloud(clouds["scan_200k"][0]).set_point_normals(
        clouds["scan_200k"][1]), 100, clouds["scan_200k"][2])
    for n in (50_000, 200_000):
        s = feats[:n].contiguous()
        t = feats[torch.randperm(feats.shape[0], generator=torch.Generator().manual_seed(0))[:n].cuda()].contiguous()
        for mutual in (False, True):
            fn = lambda: reg.correspondences_from_features(s, t, mutual)  # noqa: E731
            row = {"n": n, "m": n, "dim": 33, "mutual_filter": mutual, "whole_call_ms": timed(fn, 3),
                   "kernel_ms": kernel_ms(fn, ("feature_nn_kernel",))}
            res["correspondences"].append(row)
            print(json.dumps(row), flush=True)
    pts, nrm, radius = clouds["scan_200k"]
    res["host"] = {"cloud": "scan_200k", "max_nn": 30, "radius": radius, "threads": 8, **host_passes(pts, nrm, radius)}
    print(json.dumps(res["host"]), flush=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
