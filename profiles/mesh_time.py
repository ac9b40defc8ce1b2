"""Time of VoxelBlockGrid.extract_triangle_mesh on the volume of bench.py's TSDF workload, on cuda:0.

    python profiles/mesh_time.py [--calls 60] [--out FILE]

The 1000 synthetic room frames of bench.py (tests/synth.py, colour) are integrated into a slam.Model(0.008, 16, 40000),
then extract_triangle_mesh() (weight_threshold 3) is called 5 times untimed and --calls times between CUDA events: the
whole call, i.e. the nine passes (twelve launches) of o3db_vbg_extract_triangle_mesh, its one read-back of the two
counts, and the copies into the returned TriangleMesh.  A second, separate phase runs 5 calls under torch.profiler for
the device time of each kernel.  When oracle/_ref is built, the reference's own ExtractTriangleMeshCPU (with its
neighbour table) runs on the same volume on all host threads as the CPU baseline.

Byte model: every voxel's tsdf and weight must be read (6 B), each vertex written once (36 B with colour) and each
triangle (12 B); the bound is those bytes over the 3.35 TB/s of the H100 SXM data sheet.  One JSON line.
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
from tests.synth import PRIMESENSE_K, camera_pose, render_depth  # noqa: E402

FRAMES = 1000
VOXEL, RES, CAP, THRESHOLD = 0.008, 16, 40000, 3.0
HBM_BYTES_PER_S = 3.35e12


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    name, power, clock, max_clock = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": clock, "max_sm_clock": max_clock}


def build_volume():
    slam = o3d.t.pipelines.slam
    model = slam.Model(VOXEL, RES, CAP)
    for i in range(FRAMES):
        T = camera_pose(i, n_frames=FRAMES)
        d, c = render_depth(T, device="cuda", with_color=True)
        frame = slam.Frame(480, 640, PRIMESENSE_K)
        frame.set_data("depth", d)
        frame.set_data("color", c)
        model.update_frame_pose(i, T)
        model.integrate(frame)
    torch.cuda.synchronize()
    return model


def kernel_times(model, calls=5):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            model.voxel_grid.extract_triangle_mesh(THRESHOLD)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if any(k in e.key for k in ("extract_", "mesh_", "scan_")):
            out[e.key.split("(")[0].replace("o3db::", "")] = round(e.device_time_total / calls, 1)   # us per call
    return out


def cpu_reference(model, n_vertices, n_triangles):
    ref = os.path.join(ROOT, "oracle", "_ref", "libo3dref_mesh.so")
    if not os.path.exists(ref):
        return None
    import oracle
    threads = oracle.host_cores()
    vbg = model.voxel_grid
    n = vbg.hashmap().size()
    keys = vbg.hashmap().key_tensor()[:n].cpu().numpy()
    tsdf = vbg.attribute("tsdf")[:n].reshape(n, -1).cpu().numpy()
    wt = vbg.attribute("weight")[:n].reshape(n, -1).cpu().numpy()
    col = vbg.attribute("color")[:n].reshape(n, -1, 3).cpu().numpy()
    L = C.CDLL(ref)
    vp = C.c_void_p
    L.ref_extract_triangle_mesh.restype = C.c_int64
    L.ref_extract_triangle_mesh.argtypes = [vp, C.c_int64, vp, vp, vp, C.c_int, C.c_float, C.c_float, C.c_int,
                                            C.c_int64, C.c_int64, vp, vp, vp, vp, C.POINTER(C.c_int64)]
    out = [np.empty((n_vertices, 3), np.float32) for _ in range(3)] + [np.empty((n_triangles, 3), np.int32)]
    times, nt = [], C.c_int64(0)
    for _ in range(3):
        t0 = time.perf_counter()
        total = L.ref_extract_triangle_mesh(keys.ctypes.data, n, tsdf.ctypes.data, wt.ctypes.data, col.ctypes.data,
                                            RES, VOXEL, THRESHOLD, threads, n_vertices, n_triangles,
                                            *[o.ctypes.data for o in out], C.byref(nt))
        times.append(time.perf_counter() - t0)
    assert (total, nt.value) == (n_vertices, n_triangles), (total, nt.value, n_vertices, n_triangles)
    return {"impl": "reference ExtractTriangleMeshCPU<float,u16,u16> + neighbour table, OpenMP", "threads": threads,
            "ms_median": round(1e3 * float(np.median(times)), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=60)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_time.py needs a CUDA device")
    torch.cuda.set_device(0)
    model = build_volume()
    blocks = model.get_hashmap().size()
    for _ in range(5):
        mesh = model.voxel_grid.extract_triangle_mesh(THRESHOLD)
    vertices = int(mesh.vertex["positions"].shape[0])
    triangles = int(mesh.triangle["indices"].shape[0])
    ms, wall = [], []
    for _ in range(args.calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        a.record()
        model.voxel_grid.extract_triangle_mesh(THRESHOLD)
        b.record()
        b.synchronize()
        wall.append(1e3 * (time.perf_counter() - t0))
        ms.append(a.elapsed_time(b))
    ms = np.array(ms)
    med = float(np.median(ms))
    voxels = blocks * RES ** 3
    model_bytes = 6 * voxels + 36 * vertices + 12 * triangles
    line = {
        "workload": f"extract_triangle_mesh(weight_threshold={THRESHOLD}) of bench.py's {FRAMES}-frame colour volume",
        "card": card(), "blocks": blocks, "vertices": vertices, "triangles": triangles, "calls": args.calls,
        "ms_median": round(med, 4), "ms_p10": round(float(np.percentile(ms, 10)), 4),
        "ms_p90": round(float(np.percentile(ms, 90)), 4), "ms_min": round(float(ms.min()), 4),
        "ms_max": round(float(ms.max()), 4), "host_wall_ms_median": round(float(np.median(wall)), 4),
        "byte_model": {"bytes": model_bytes, "per": "6 B per voxel (tsdf + weight) + 36 B per vertex + 12 B per triangle written",
                       "bandwidth_TBps": round(model_bytes / (med * 1e-3) / 1e12, 3),
                       "fraction_of_3.35TBps": round(model_bytes / (med * 1e-3) / HBM_BYTES_PER_S, 3),
                       "bound_ms": round(model_bytes / HBM_BYTES_PER_S * 1e3, 4)},
        "kernel_us_per_call": kernel_times(model),
    }
    base = cpu_reference(model, vertices, triangles)
    if base is not None:
        line["cpu_baseline"] = base
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
