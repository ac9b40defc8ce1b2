"""Time of Fast Global Registration (o3db_registration_fgr, registration_fgr_based_on_feature_matching) on cuda:0.
    python profiles/fgr_time.py [--calls 10] [--out FILE]
Workloads: the clouds of profiles/ransac_time.py's pipeline cases (tests/ransac_cases.overlap_pair of a scene of
22 500 / 202 500 points, each part voxel-down-sampled at 2.5 lattice spacings and sorted, normals with max_nn 30 and
radius 2 voxels, FPFH with max_nn 100 and radius 5 voxels), registered from their features with
FastGlobalRegistrationOption(maximum_correspondence_distance = 0.5 voxel), as upstream's tutorial does, with the tuple
test on and off.
For each, after one untimed call, --calls C ABI calls run between CUDA events, each after the same seed.  Reported:
the median, min and max time per call; the split: the feature matching alone (o3db_correspondences_from_features with
the mutual filter, between events), the host's draws (the same number of ints from the engine, timed on its own),
and per-kernel device times from a separate torch.profiler phase, grouped into normalisation, matching, scan (the
shared u32 scan of the matching's mutual filter and of the tuple test), tuple test, optimisation and evaluation; the
cudaStreamSynchronize calls per call counted in the same trace, beside the count the
code's structure gives (3, one per batch of 16 384 trials, two in the matching); the result checked against the CPU oracle (oracle/fgr) on the same draws, and the
compiled reference (oracle/_ref/libo3dref_fgr.so, one host thread, with the shim's brute-force searches) timed beside
it on the 20 k case where it was built.  The card's
name, power limit and SM clock are read before and after.  One JSON line.
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
from oracle import fgr as orc  # noqa: E402
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
        out.append((pc.point["positions"], reg.compute_fpfh_feature(pc, 100, 5 * voxel)))
    return out


def cabi(s, t, fs, ft, opt):
    o3d.utility.random.seed(SEED)
    T = np.zeros(16)
    st = _lib.FgrStats()
    out = torch.empty(s.shape[0], dtype=torch.int64, device="cuda")
    rc_ = _lib.lib.o3db_registration_fgr(s.data_ptr(), s.shape[0], t.data_ptr(), t.shape[0], None, 0, fs.data_ptr(),
                                         ft.data_ptr(), fs.shape[1], C.byref(opt), T.ctypes.data, out.data_ptr(),
                                         C.byref(st), int(torch.cuda.current_stream().cuda_stream))
    assert rc_ == 0, _lib.last_error()
    return T, out, st


def matching(fs, ft, swapped):
    q, t = (ft, fs) if swapped else (fs, ft)
    out = torch.empty((q.shape[0], 2), dtype=torch.int64, device="cuda")
    k, mutual = C.c_int64(0), C.c_int64(0)
    _lib.check(_lib.lib.o3db_correspondences_from_features(q.data_ptr(), q.shape[0], t.data_ptr(), t.shape[0],
                                                           q.shape[1], 1, -1.0, out.data_ptr(), C.byref(k),
                                                           C.byref(mutual), int(torch.cuda.current_stream().cuda_stream)))


def group(name):
    if name.startswith("fgr_optimize"):
        return "optimise"
    if name.startswith(("fgr_tuple", "fgr_stop")):
        return "tuple_test"
    if "scan" in name:   # the shared u32 scan: the matching's mutual filter and the tuple test's counts
        return "scan"
    if name.startswith(("fgr_check", "fgr_mean", "fgr_scale")):
        return "normalise"
    if name.startswith(("feature_nn", "mutual_flag", "corres_write")):
        return "matching"
    return "evaluation"


def kernel_times(fn, reps):
    """Per-kernel and per-group device ms per call, and the cudaStreamSynchronize calls per call as the CUDA runtime
    trace counts them (None when the trace has no runtime calls)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
    per = {}
    syncs = 0
    runtime_seen = False
    for e in prof.key_averages():
        if e.key.startswith("cuda") and e.device_type.name == "CPU":
            runtime_seen = True
            if e.key == "cudaStreamSynchronize":
                syncs += e.count
            continue
        if e.device_type.name != "CUDA" or "Memcpy" in e.key or "Memset" in e.key:
            continue
        name = e.key.split("(")[0].split("::")[-1].split("<")[0].strip()
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        per[name] = per.get(name, 0.0) + t / 1e3 / reps
    groups = {}
    for k, v in per.items():
        groups[group(k)] = groups.get(group(k), 0.0) + v
    return per, groups, (syncs / reps if runtime_seen else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "fgr_time.py measures on cuda:0"
    torch.cuda.set_device(0)
    res = {"card": card(), "calls": args.calls, "cases": {}}
    for name, side, spacing in (("20k", 150, 0.02), ("200k", 450, 0.02 / 3)):
        voxel = 2.5 * spacing
        (s, fs), (t, ft) = prepare(side, spacing, voxel)
        for tuple_test in (True, False):
            opt = _lib.FgrOption(1.4, 0, 0, 0.5 * voxel, 64, 0.95, 1000, int(tuple_test))
            T, out, st = cabi(s, t, fs, ft, opt)
            ms = [event_ms(lambda: cabi(s, t, fs, ft, opt)) for _ in range(args.calls)]
            swapped = tuple_test and s.shape[0] < t.shape[0]
            matching(fs, ft, swapped)
            match_ms = [event_ms(lambda: matching(fs, ft, swapped)) for _ in range(args.calls)]
            draws = np.zeros(max(st.trials * 3, 1), np.int32)
            t0 = time.perf_counter()
            if st.trials:
                _lib.check(_lib.lib.o3db_random_uniform_ints(0, int(st.cross) - 1, st.trials * 3, draws.ctypes.data))
            draw_ms = (time.perf_counter() - t0) * 1e3
            per, groups, syncs = kernel_times(lambda: cabi(s, t, fs, ft, opt), 3)
            batches = -(-st.trials // orc.BATCH)
            sp, tp = s.cpu().numpy(), t.cpu().numpy()
            fsn, ftn = fs.cpu().numpy(), ft.cpu().numpy()
            K = int(st.cross)
            o3d.utility.random.seed(SEED)
            d = np.zeros(max(300 * K, 1), np.int32)
            if tuple_test and K > 2:
                _lib.check(_lib.lib.o3db_random_uniform_ints(0, K - 1, d.size, d.ctypes.data))
            want, _ = orc.fgr_features(sp, tp, fsn, ftn, d, orc.option(
                maximum_correspondence_distance=0.5 * voxel, tuple_test=tuple_test))
            med = float(np.median(ms))
            case = {"source_points": int(s.shape[0]), "target_points": int(t.shape[0]), "mutual_pairs": K,
                    "tuples": int(st.tuples), "trials": int(st.trials), "pairs_optimised": int(st.pairs),
                    "fitness": st.fitness, "inlier_rmse": st.inlier_rmse,
                    "median_ms": med, "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms)),
                    "matching_median_ms": float(np.median(match_ms)), "host_draw_ms": draw_ms,
                    "device_ms_by_group": groups, "device_ms_by_kernel": per,
                    "optimise_us_per_iteration": groups.get("optimise", 0.0) * 1e3 / 64 if st.pairs >= 10 else None,
                    "host_syncs_counted": syncs,
                    "host_syncs_expected": 3 + batches + 2,   # 3, one per batch of trials, two in the matching
                    "equal_to_oracle": bool(np.array_equal(T.reshape(4, 4), want.transformation) and
                                            np.array_equal(out.cpu().numpy(), want.correspondence_set) and
                                            st.fitness == want.fitness and st.inlier_rmse == want.rmse)}
            if orc.ref() is not None and name == "20k":   # its brute-force feature search is quadratic
                orc.ref_seed(SEED)
                t0 = time.perf_counter()
                r = orc.ref_fgr(sp, tp, orc.option(maximum_correspondence_distance=0.5 * voxel,
                                                   tuple_test=tuple_test), source_feature=fsn, target_feature=ftn)
                case["reference_one_thread_ms"] = (time.perf_counter() - t0) * 1e3
                case["reference_fitness"] = r.fitness
            res["cases"][f"pipeline_{name}_{'tuples' if tuple_test else 'no_tuples'}"] = case
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
