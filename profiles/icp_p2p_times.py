"""Device time per iteration of a point-to-point and a point-to-plane registration of the same clouds (bench.py's
2 M-point pair, r = 0.05, 30 iterations, criteria that never trigger), alternated in one process on cuda:0.

    python profiles/icp_p2p_times.py [--reps 5] [--out FILE]

Measured as profiles/icp_iter_times.py does: every registration starts from o3db_icp_reset with the L2 flushed (a
256 MiB write), one o3db_icp_iterate(h, 1) runs between each pair of CUDA events, and o3db_icp_finish between the last
two.  Two untimed registrations per estimator warm up; then --reps rounds time one registration of each estimator, in
turn.  The result is one JSON object (printed, and written to --out) with, per estimator, the median over the rounds of
the first iteration, of the aligned iterations (from the 6th on) and of the evaluation pass, the byte model's bytes per
iteration, and the card's name, power limit and maximum SM clock read in the same run.  Needs a CUDA device.
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
from tests.synth import make_icp_pair  # noqa: E402

ITERS = 30


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    name, power, clock = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def model_bytes(n, m, normals):
    """DESIGN.md 4.1: source read + written, target points (+ normals), original indices, CSR offsets, seeds."""
    h = min(max(m // 32, 1), 1 << 25)
    return 12 * n + 12 * n + 12 * m + (12 * m if normals else 0) + 4 * m + 4 * (h + 1) + 4 * n


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
        raise SystemExit("icp_p2p_times.py needs a CUDA device")
    torch.cuda.set_device(0)
    stream = int(torch.cuda.current_stream().cuda_stream)
    src, tgt, nrm, T_gt = make_icp_pair(2_000_000, seed=2)
    d = [torch.from_numpy(a).cuda() for a in (src, tgt, nrm)]
    opt = L.IcpOptions()
    opt.max_correspondence_distance, opt.max_iteration = 0.05, ITERS
    opt.relative_fitness = opt.relative_rmse = 0.0
    opt.kernel = L.RobustKernel(0, 1.0, 1.0)
    handles = {"point_to_point": C.c_void_p(), "point_to_plane": C.c_void_p()}
    L.check(L.lib.o3db_icp_create_point_to_point(d[0].data_ptr(), len(src), d[1].data_ptr(), len(tgt), L.dptr(np.eye(4)),
                                                 C.byref(opt), None, stream, C.byref(handles["point_to_point"])))
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
            "model_bytes_per_iteration": model_bytes(len(src), len(tgt), name == "point_to_plane"),
            "fitness": res.fitness, "inlier_rmse": res.inlier_rmse,
            "transformation_error_vs_ground_truth": float(np.abs(np.array(res.transformation).reshape(4, 4) - T_gt).max()),
        }
    text = json.dumps(out, indent=1)
    print(text, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
