"""Device time per iteration of a Doppler and a point-to-plane registration of the same clouds (bench.py's 2 M-point
pair, r = 0.05, 30 iterations, criteria that never trigger), alternated in one process on cuda:0.  The source's
directions and Doppler values are tests/doppler_cases.py's (its mounted sensor, period 0.1 s, 5 % dynamic points); the
Doppler estimator rejects dynamic outliers from iteration 2 on.

    python profiles/icp_doppler_times.py [--reps 5] [--out FILE]

Measured as profiles/icp_iter_times.py does: every registration starts from o3db_icp_reset with the L2 flushed (a
256 MiB write), one o3db_icp_iterate(h, 1) runs between each pair of CUDA events, and o3db_icp_finish between the last
two.  Two untimed registrations per estimator warm up; then --reps rounds time one registration of each estimator, in
turn.  The result is one JSON object (printed, and written to --out) with, per estimator, the median over the rounds of
the first iteration, of the aligned iterations (from the 6th on) and of the evaluation pass, the byte model's bytes per
iteration and per query with the rate they are streamed at in the aligned iterations, and the card's name, power limit and maximum SM clock read in the same run; and, per estimator, the
iterations each needs to converge under the default criteria (relative fitness and rmse 1e-6, at most 30) with the
distance of that result from the true motion.  Needs a CUDA device.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from open3d_b200 import _lib as L  # noqa: E402
from tests.doppler_cases import CALIB, make_doppler_pair  # noqa: E402

ITERS = 30


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    name, power, clock = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def model_bytes(n, m, doppler):
    """DESIGN.md 4.1: source record read + written (20 B per point; the Doppler record is read with its 16 B of
    directions and Doppler values, which are never written), target points and normals, original indices, CSR offsets,
    seeds."""
    h = min(max(m // 32, 1), 1 << 25)
    return (56 if doppler else 40) * n + 12 * m + 12 * m + 4 * m + 4 * (h + 1) + 4 * n


def timed_registration(h, stream, flush):
    res = L.IcpResult()
    L.check(L.lib.o3db_icp_reset(h, stream))
    flush.fill_(1)
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(ITERS + 2)]
    evs[0].record()
    for k in range(ITERS):
        L.check(L.lib.o3db_icp_iterate(h, 1, stream))
        evs[k + 1].record()
    L.check(L.lib.o3db_icp_finish(h, C.byref(res), None, None, stream))
    evs[ITERS + 1].record()
    torch.cuda.synchronize()
    return [1e3 * evs[k].elapsed_time(evs[k + 1]) for k in range(ITERS + 1)], res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("icp_doppler_times.py needs a CUDA device")
    torch.cuda.set_device(0)
    stream = int(torch.cuda.current_stream().cuda_stream)
    src, dops, dirs, tgt, nrm, T_gt, _ = make_doppler_pair(2_000_000, seed=2, dynamic=0.05)
    d = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (src, tgt, nrm, dops, dirs)]
    opt = L.IcpOptions()
    opt.max_correspondence_distance, opt.max_iteration = 0.05, ITERS
    opt.relative_fitness = opt.relative_rmse = 0.0
    opt.kernel = L.RobustKernel(0, 1.0, 1.0)
    from open3d_b200.t.pipelines.registration import TransformationEstimationForDopplerICP
    params = TransformationEstimationForDopplerICP(reject_dynamic_outliers=True, transform_vehicle_to_sensor=CALIB)._params()
    handles = {"doppler": C.c_void_p(), "point_to_plane": C.c_void_p()}
    L.check(L.lib.o3db_icp_create_doppler(d[0].data_ptr(), d[3].data_ptr(), d[4].data_ptr(), len(src), d[1].data_ptr(),
                                          d[2].data_ptr(), len(tgt), L.dptr(np.eye(4)), C.byref(opt), C.byref(params),
                                          None, stream, C.byref(handles["doppler"])))
    L.check(L.lib.o3db_icp_create(d[0].data_ptr(), len(src), d[1].data_ptr(), d[2].data_ptr(), len(tgt),
                                  L.dptr(np.eye(4)), C.byref(opt), None, stream, C.byref(handles["point_to_plane"])))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    times = {k: [] for k in handles}
    last = {}
    for rep in range(2 + args.reps):
        for name, h in handles.items():
            t, last[name] = timed_registration(h, stream, flush)
            if rep >= 2:
                times[name].append(t)
    for h in handles.values():
        L.lib.o3db_icp_destroy(h)
    converge = {}
    copt = L.IcpOptions()
    copt.max_correspondence_distance, copt.max_iteration = 0.05, ITERS
    copt.relative_fitness = copt.relative_rmse = 1e-6
    copt.kernel = L.RobustKernel(0, 1.0, 1.0)
    for name in handles:
        res = L.IcpResult()
        if name == "doppler":
            L.check(L.lib.o3db_icp_doppler(d[0].data_ptr(), d[3].data_ptr(), d[4].data_ptr(), len(src), d[1].data_ptr(),
                                           d[2].data_ptr(), len(tgt), L.dptr(np.eye(4)), C.byref(copt), C.byref(params),
                                           C.byref(res), None, None, stream))
        else:
            L.check(L.lib.o3db_icp_point_to_plane(d[0].data_ptr(), len(src), d[1].data_ptr(), d[2].data_ptr(), len(tgt),
                                                  L.dptr(np.eye(4)), C.byref(copt), C.byref(res), None, None, stream))
        converge[name] = {"converged": bool(res.converged), "iterations": int(res.num_iterations),
                          "transformation_error_vs_ground_truth":
                              float(np.abs(np.array(res.transformation).reshape(4, 4) - T_gt).max())}
    out = {"workload": f"{len(src)} source / {len(tgt)} target points, r = 0.05, {ITERS} iterations, L2 flushed per "
                       "registration, one launch per CUDA-event pair",
           "card": card(), "reps": args.reps}
    for name, rows in times.items():
        t = np.array(rows)
        med = np.median(t, axis=0)
        res = last[name]
        out[name] = {
            "first_iteration_us_median": round(float(med[0]), 1),
            "aligned_iteration_us_median": round(float(med[5:ITERS].mean()), 1),
            "aligned_iteration_us_min_max_over_reps": [round(float(t[:, 5:ITERS].mean(axis=1).min()), 1),
                                                       round(float(t[:, 5:ITERS].mean(axis=1).max()), 1)],
            "mean_iteration_us_median": round(float(np.median(t[:, :ITERS].mean(axis=1))), 1),
            "evaluate_us_median": round(float(med[ITERS]), 1),
            "iteration_us_median": [round(float(x), 1) for x in med[:ITERS]],
            "model_bytes_per_iteration": model_bytes(len(src), len(tgt), name == "doppler"),
            "model_bytes_per_query": round(model_bytes(len(src), len(tgt), name == "doppler") / len(src), 1),
            "aligned_model_GB_per_s": round(model_bytes(len(src), len(tgt), name == "doppler") /
                                            float(med[5:ITERS].mean()) / 1e3, 1),
            "fitness": res.fitness, "inlier_rmse": res.inlier_rmse,
            "transformation_error_vs_ground_truth": float(np.abs(np.array(res.transformation).reshape(4, 4) - T_gt).max()),
            "default_criteria": converge[name],
        }
    text = json.dumps(out, indent=1)
    print(text, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
