"""Time of PointCloud.create_from_rgbd_image and project_to_rgbd_image on cuda:0.

    python profiles/projection_time.py [--calls 50] [--out FILE]

Workloads:
    unproject_vga   create_from_rgbd_image of a 640x480 u16 depth + u8 colour frame of the synthetic room
                    (tests/synth.render_depth(camera_pose(100)), PRIMESENSE_K), stride 1, a world pose
    unproject_hd    the same at 1280x720 (tests/camera_cases.HD_K)
    project_2m      project_to_rgbd_image of make_icp_pair(2_000_000, seed=3)'s target with colours into 640x480,
                    from 6 m below the cloud (depth_max 10)
After 5 untimed calls, --calls calls of each run between CUDA events; each Python call includes its output allocations
and, for create_from_rgbd_image, the one host synchronisation that reads the point count.  A separate phase runs 5
calls of each under torch.profiler for the device time of each kernel.  The CPU oracle (oracle/projection, one host
thread) runs the same workloads as the CPU figure beside each.  One JSON line.
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
import oracle  # noqa: E402
from oracle import projection  # noqa: E402
from tests.camera_cases import HD_K  # noqa: E402
from tests.synth import PRIMESENSE_K, camera_pose, make_icp_pair, render_depth  # noqa: E402
from tests.projection_cases import _above, indexed_colors  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    name, power, clock, max_clock = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": clock, "max_sm_clock": max_clock}


def timed(fn, calls):
    ms = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    ms = np.array(ms)
    return {"ms_median": round(float(np.median(ms)), 4), "ms_p10": round(float(np.percentile(ms, 10)), 4),
            "ms_p90": round(float(np.percentile(ms, 90)), 4), "ms_min": round(float(ms.min()), 4)}


def cpu_ms(fn, reps=3):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return round(1e3 * float(np.median(t)), 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("projection_time.py needs a CUDA device")
    torch.cuda.set_device(0)
    G = o3d.t.geometry
    T = camera_pose(100)
    E = oracle.inverse_transformation(T)
    work = {}
    for name, K, w, h in (("unproject_vga", PRIMESENSE_K, 640, 480), ("unproject_hd", HD_K, 1280, 720)):
        depth, color = render_depth(T, K=K, width=w, height=h, with_color=True)
        rgbd = G.RGBDImage(color.cuda(), depth.cuda())
        dn, cn = depth.numpy(), color.numpy()
        n = len(G.PointCloud.create_from_rgbd_image(rgbd, K, E).point["positions"])
        work[name] = (lambda rgbd=rgbd, K=K: G.PointCloud.create_from_rgbd_image(rgbd, K, E),
                      lambda dn=dn, cn=cn, K=K: projection.unproject(dn, K, E, color=cn),
                      {"image": f"{w}x{h}", "points": n})
    _, tgt, _, _ = make_icp_pair(2_000_000, seed=3)
    cols = indexed_colors(tgt)
    Ep = _above(tgt, 6.0)
    pcd = G.PointCloud(torch.from_numpy(tgt).cuda()).set_point_colors(torch.from_numpy(cols).cuda())
    work["project_2m"] = (lambda: pcd.project_to_rgbd_image(640, 480, PRIMESENSE_K, Ep, 1000.0, 10.0),
                          lambda: projection.project(tgt, PRIMESENSE_K, Ep, 640, 480, 1000.0, 10.0, cols),
                          {"image": "640x480", "points": len(tgt)})

    out = {}
    for name, (gpu, cpu, info) in work.items():
        for _ in range(5):
            gpu()
        torch.cuda.synchronize()
        out[name] = dict(info, gpu=timed(gpu, args.calls), cpu_oracle_ms_median=cpu_ms(cpu))

    from torch.profiler import ProfilerActivity, profile
    for name, (gpu, _, _) in work.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                gpu()
            torch.cuda.synchronize()
        kernels = {}
        for e in prof.key_averages():
            if e.device_time_total > 0 and "Memcpy" not in e.key:
                kernels[e.key.split("(")[0].replace("o3db::", "").replace("void ", "")] = round(
                    e.device_time_total / 5, 1)
        out[name]["device_us_per_call"] = kernels

    line = {"workload": "create_from_rgbd_image 640x480 and 1280x720; project_to_rgbd_image 2 M points -> 640x480",
            "card": card(), "calls": args.calls, **out,
            "cpu_oracle": "oracle/projection (C, one host thread)"}
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
