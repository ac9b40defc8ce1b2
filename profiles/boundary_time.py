"""Time of boundary detection (o3db_compute_boundary_points, PointCloud.compute_boundary_points) on cuda:0.
    python profiles/boundary_time.py [--calls 30] [--out FILE]
Clouds, both with max_nn 30 and their analytic normals: the target of tests/synth.make_icp_pair(2_000_000, seed=1) at
radius 0.08, and that of make_icp_pair(200_000, seed=2, spacing=0.005), a ~200 k-point scan 5 mm apart, at radius
0.02.  After 5 untimed calls, CUDA events around --calls each of: the index build (o3db_nns_create), the hybrid
search, the whole C ABI call and the whole PointCloud.compute_boundary_points call.  A separate torch.profiler phase gives each kernel's device time, and
the boundary kernel's byte model is set beside it.  Every GPU mask and max_gap is checked against the CPU oracle's f64
mode.  On the host, on the same neighbour lists: the oracle (OpenMP, all host threads) and, where
oracle/_ref/libo3dref_boundary.so was built, the reference's own ComputeBoundaryPointsCPU (its ParallelFor on OpenMP,
all host threads).  The card's name, power limit and SM clock are read before and after.  One JSON line.
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

MAX_NN = 30
ANGLE = 90.0
HBM_BYTES_PER_S = 3.35e12
REF = os.path.join(ROOT, "oracle", "_ref", "libo3dref_boundary.so")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    name, power, clock, max_clock = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": clock, "max_sm_clock": max_clock}


def stream():
    return int(torch.cuda.current_stream().cuda_stream)


def timed(fn, calls, after=None):
    ms = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
        if after:
            after(out)
    ms = np.array(ms)
    return {"ms_median": round(float(np.median(ms)), 4), "ms_p10": round(float(np.percentile(ms, 10)), 4),
            "ms_p90": round(float(np.percentile(ms, 90)), 4), "ms_min": round(float(ms.min()), 4)}


def host_ms(fn, reps=3):
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return round(1e3 * float(np.median(times)), 2)


def measure(pts, nrm_np, radius, calls):
    import oracle
    from oracle import boundary as ob
    n = len(pts)
    p = torch.from_numpy(pts).cuda()
    q = torch.from_numpy(nrm_np).cuda()
    mask = torch.empty(n, dtype=torch.uint8, device="cuda")
    gap = torch.empty(n, dtype=torch.float32, device="cuda")
    idx = torch.empty((n, MAX_NN), dtype=torch.int32, device="cuda")
    cnt = torch.empty(n, dtype=torch.int32, device="cuda")
    pc = o3d.t.geometry.PointCloud(p).set_point_normals(q)

    def call():
        L.check(L.lib.o3db_compute_boundary_points(p.data_ptr(), q.data_ptr(), n, radius, MAX_NN, ANGLE,
                                                   mask.data_ptr(), None, stream()))

    def index():
        h = C.c_void_p()
        L.check(L.lib.o3db_nns_create(p.data_ptr(), n, radius, stream(), C.byref(h)))
        return h

    for _ in range(5):
        call()
    torch.cuda.synchronize()
    t_call = timed(call, calls)
    t_python = timed(lambda: pc.compute_boundary_points(radius, MAX_NN, ANGLE), calls)
    t_index = timed(index, calls, after=L.lib.o3db_nns_destroy)
    h = index()

    def search():
        L.check(L.lib.o3db_nns_hybrid_search(h, p.data_ptr(), n, radius, MAX_NN, idx.data_ptr(), None, cnt.data_ptr(),
                                             stream()))

    for _ in range(3):
        search()
    t_search = timed(search, calls)
    torch.cuda.synchronize()
    L.lib.o3db_nns_destroy(h)
    mean_kept = float((cnt.double() - 1).clamp(min=0).mean())

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            call()
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        if e.device_time_total > 0 and "Memset" not in e.key and "Memcpy" not in e.key:
            kernels[e.key.split("(")[0].replace("o3db::", "").replace("void ", "")] = round(e.device_time_total / 5, 1)
    k_us = next((v for k, v in kernels.items() if k.startswith("boundary_kernel")), None)
    # compulsory bytes: per point the count, the kept row entries, the point's position and normal, the mask; every
    # gathered neighbour position is counted once (its line is shared with the neighbours' own reads)
    model_bytes = int(n * (4 + 4 * mean_kept + 12 + 12 + 1))

    L.check(L.lib.o3db_compute_boundary_points(p.data_ptr(), q.data_ptr(), n, radius, MAX_NN, ANGLE, mask.data_ptr(),
                                               gap.data_ptr(), stream()))
    torch.cuda.synchronize()
    threads = oracle.set_num_threads(oracle.host_cores())
    o_idx, _, o_cnt = oracle.hybrid_search(pts, pts, radius, MAX_NN)
    want, wgap = ob.compute_boundary_points_lists(pts, nrm_np, o_idx, o_cnt, ANGLE, mode="f64")
    got = mask.cpu().numpy().astype(bool)
    equal = bool(np.array_equal(got, want) and np.array_equal(gap.cpu().numpy().view(np.uint32), wgap.view(np.uint32)))
    res = {
        "points": n, "radius": radius, "max_nn": MAX_NN, "angle_threshold": ANGLE,
        "mean_kept_neighbours": round(mean_kept, 3), "boundary_points": int(got.sum()),
        "equal_to_f64_oracle": equal,
        "index": t_index, "search": t_search, "boundary_call": t_call, "python_call": t_python,
        "kernel_us_per_call": kernels, "boundary_kernel_us": k_us,
        "boundary_kernel_byte_model": {
            "bytes": model_bytes,
            "per": "4 B count + 4 B per kept row entry + 12 B position + 12 B normal + 1 B mask, per point",
            "bound_us": round(model_bytes / HBM_BYTES_PER_S * 1e6, 1),
            "fraction_of_3.35TBps": None if k_us is None else round(model_bytes / (k_us * 1e-6) / HBM_BYTES_PER_S, 3)},
        "host_threads": threads,
        "oracle_search_ms": host_ms(lambda: oracle.hybrid_search(pts, pts, radius, MAX_NN)),
        "oracle_boundary_ms": host_ms(lambda: ob.compute_boundary_points_lists(pts, nrm_np, o_idx, o_cnt, ANGLE,
                                                                               mode="libm")),
    }
    if os.path.exists(REF):
        R = C.CDLL(REF)
        R.ref_compute_boundary_points_f32.restype = None
        R.ref_compute_boundary_points_f32.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                                      C.c_void_p, C.c_void_p, C.c_double]
        rmask = np.zeros(n, np.uint8)

        def ref():
            rmask[:] = 0
            R.ref_compute_boundary_points_f32(pts.ctypes.data, nrm_np.ctypes.data, n, o_idx.ctypes.data, MAX_NN,
                                              o_cnt.ctypes.data, rmask.ctypes.data, ANGLE)

        res["reference_boundary_ms"] = host_ms(ref)
        libm, _ = ob.compute_boundary_points_lists(pts, nrm_np, o_idx, o_cnt, ANGLE, mode="libm")
        res["reference_equal_to_libm_oracle"] = bool(np.array_equal(rmask.astype(bool), libm))
        res["gpu_differs_from_reference"] = int(np.count_nonzero(rmask.astype(bool) != got))
    else:
        res["reference_boundary_ms"] = "not measured (oracle/_ref/libo3dref_boundary.so not built)"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("boundary_time.py needs a CUDA device")
    torch.cuda.set_device(0)
    line = {"workload": f"compute_boundary_points(radius, max_nn={MAX_NN}, angle_threshold={ANGLE})",
            "card": card(), "calls": args.calls, "cases": {}}
    for name, n, seed, spacing, radius in (("target_2M", 2_000_000, 1, 0.02, 0.08),
                                           ("scan_200k", 200_000, 2, 0.005, 0.02)):
        _, tgt, nrm, _ = make_icp_pair(n, seed=seed, spacing=spacing)
        line["cases"][name] = measure(np.ascontiguousarray(tgt, np.float32), np.ascontiguousarray(nrm, np.float32),
                                      radius, args.calls)
        torch.cuda.empty_cache()
    line["card_after"] = card()
    out = json.dumps(line)
    print(out)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(out + "\n")


if __name__ == "__main__":
    main()
