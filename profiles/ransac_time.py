"""Time of RANSAC registration (o3db_registration_ransac, registration_ransac_based_on_*) on cuda:0.
    python profiles/ransac_time.py [--calls 5] [--out FILE]
Workloads:
  pipeline_20k / pipeline_200k  tests/ransac_cases.overlap_pair of a scene of 22 500 / 202 500 points (noise a tenth
                of the spacing), each part voxel-down-sampled at 2.5 lattice spacings and sorted, normals (max_nn 30,
                radius 2 voxels), FPFH (max_nn 100, radius 5 voxels), correspondences without the mutual filter, then
                RANSAC with the tutorial settings: ransac_n 3, edge length 0.9, distance 1.5 voxels,
                RANSACConvergenceCriteria(100000, 0.999);
  fixed_100 / fixed_1000 / fixed_10000  the 20 k pair's correspondences without checkers and with confidence 1, so
                that exactly 100 / 1 000 / 10 000 hypotheses are drawn and every one is validated.
For each, after one untimed call, --calls C ABI calls run between CUDA events, each after the same seed.  Reported:
time per call, per validated hypothesis (null when none was validated), the host's share (drawing the same number of
ints from the engine, timed on its own, and the call's synchronise count), and the CPU oracle (oracle/ransac, OpenMP
over source points on all host threads) on the fixed 100-hypothesis case, checked for equality.  The card's name, power limit and SM clock are read
before and after.  One JSON line.
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
from open3d_b200 import _lib  # noqa: E402
from oracle import ransac as orc  # noqa: E402
from tests import ransac_cases as rc  # noqa: E402

SEED = 1


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


def prepare(n_side, spacing, voxel):
    reg = o3d.t.pipelines.registration
    src, tgt, _ = rc.overlap_pair(rc.scene(n_side, spacing, 1), 2, noise=spacing / 10)
    out = []
    for p in (src, tgt):
        q = o3d.t.geometry.PointCloud(torch.from_numpy(p.astype(np.float32)).cuda()).voxel_down_sample(voxel)
        q = q.point["positions"].cpu().numpy()
        q = np.ascontiguousarray(q[np.lexsort((q[:, 2], q[:, 1], q[:, 0]))])
        pc = o3d.t.geometry.PointCloud(torch.from_numpy(q).cuda())
        pc.estimate_normals(30, 2 * voxel)
        out.append((pc, reg.compute_fpfh_feature(pc, 100, 5 * voxel)))
    (s, fs), (t, ft) = out
    return s, t, reg.correspondences_from_features(fs, ft, False)


def cabi(s, t, c, dist, max_it, conf, ck):
    o3d.utility.random.seed(SEED)
    sp, tp = s.point["positions"], t.point["positions"]
    T = np.zeros(16)
    st = _lib.RansacStats()
    out = torch.empty(sp.shape[0], dtype=torch.int64, device="cuda")
    rc_ = _lib.lib.o3db_registration_ransac(sp.data_ptr(), None, sp.shape[0], tp.data_ptr(), None, tp.shape[0],
                                            c.data_ptr(), c.shape[0], dist, 3, max_it, conf, C.byref(ck),
                                            T.ctypes.data, out.data_ptr(), C.byref(st),
                                            int(torch.cuda.current_stream().cuda_stream))
    assert rc_ == 0, _lib.last_error()
    return T, out, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "ransac_time.py measures on cuda:0"
    torch.cuda.set_device(0)
    res = {"card": card(), "calls": args.calls, "host_threads": os.cpu_count(), "cases": {}}
    work = []
    for name, side, spacing in (("20k", 150, 0.02), ("200k", 450, 0.02 / 3)):
        voxel = 2.5 * spacing
        s, t, c = prepare(side, spacing, voxel)
        ck = _lib.RansacCheckers(1, 1, 0, 0.9, 1.5 * voxel, 0.0)
        work.append((f"pipeline_{name}", s, t, c, 1.5 * voxel, 100000, 0.999, ck))
        if name == "20k":
            none = _lib.RansacCheckers(0, 0, 0, 0.0, 0.0, 0.0)
            work += [(f"fixed_{h}", s, t, c, 1.5 * voxel, h, 1.0, none) for h in (100, 1000, 10000)]
    for cname, s, t, c, dist, max_it, conf, ck in work:
        T, out, st = cabi(s, t, c, dist, max_it, conf, ck)
        ms = [event_ms(lambda: cabi(s, t, c, dist, max_it, conf, ck)) for _ in range(args.calls)]
        draws = np.zeros(max(st.drawn * 3, 1), np.int32)
        t0 = time.perf_counter()
        _lib.check(_lib.lib.o3db_random_uniform_ints(0, int(c.shape[0]) - 1, st.drawn * 3, draws.ctypes.data))
        draw_ms = (time.perf_counter() - t0) * 1e3
        batches = -(-st.drawn // orc.BATCH)
        med = float(np.median(ms))
        case = {"source_points": int(s.point["positions"].shape[0]), "target_points": int(t.point["positions"].shape[0]),
                "correspondences": int(c.shape[0]), "max_iteration": max_it, "confidence": conf,
                "drawn": int(st.drawn), "validated": int(st.validated), "best_index": int(st.best_index),
                "fitness": st.fitness, "inlier_rmse": st.inlier_rmse,
                "median_ms": med, "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms)),
                "ms_per_validated": med / int(st.validated) if st.validated > 0 else None, "host_draw_ms": draw_ms,
                "host_syncs": 2 + 2 * batches}
        if cname == "fixed_100":
            sp, tp = s.point["positions"].cpu().numpy(), t.point["positions"].cpu().numpy()
            o3d.utility.random.seed(SEED)
            d = np.zeros(max_it * 3, np.int32)
            _lib.check(_lib.lib.o3db_random_uniform_ints(0, int(c.shape[0]) - 1, d.size, d.ctypes.data))
            t0 = time.perf_counter()
            want = orc.ransac(sp, tp, c.cpu().numpy(), d, dist, 3, max_it, conf,
                              orc.Checkers())
            case["oracle_all_threads_ms"] = (time.perf_counter() - t0) * 1e3
            case["equal_to_oracle"] = bool(np.array_equal(T.reshape(4, 4), want.transformation) and
                                           np.array_equal(out.cpu().numpy(), want.correspondence_set) and
                                           st.fitness == want.fitness and st.inlier_rmse == want.rmse)
        res["cases"][cname] = case
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
