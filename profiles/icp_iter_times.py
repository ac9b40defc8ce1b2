"""Device time of every iteration of bench.py's ICP registration (point-to-plane, 2 M-point clouds, r = 0.05, 30
iterations), and of the final evaluation pass, on cuda:0.

    python profiles/icp_iter_times.py [--reps 5] [--label NAME]

Each registration starts from o3db_icp_reset with the L2 flushed (a 256 MiB write), as a bench.py step does; then one
o3db_icp_iterate(h, 1) runs between each pair of CUDA events, and o3db_icp_finish (the evaluation kernel plus the
read-back of the result) between the last two.  The events between the launches also stop one iteration's kernel
from starting during the previous one's tail (programmatic dependent launch), so the sum of the per-iteration times
is a little above bench.py's loop time.  Two untimed registrations warm up; the result is one JSON line with the
median and minimum over --reps registrations of every interval, and the card's name, power limit and maximum SM clock
read in the same run.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--label", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("icp_iter_times.py needs a CUDA device")
    torch.cuda.set_device(0)
    stream = int(torch.cuda.current_stream().cuda_stream)
    src, tgt, nrm, T_gt = make_icp_pair(2_000_000, seed=2)
    d = [torch.from_numpy(a).cuda() for a in (src, tgt, nrm)]
    opt = L.IcpOptions()
    opt.max_correspondence_distance, opt.max_iteration = 0.05, ITERS
    opt.relative_fitness = opt.relative_rmse = 0.0
    opt.kernel = L.RobustKernel(0, 1.0, 1.0)
    h = C.c_void_p()
    L.check(L.lib.o3db_icp_create(d[0].data_ptr(), len(src), d[1].data_ptr(), d[2].data_ptr(), len(tgt),
                                  L.dptr(np.eye(4)), C.byref(opt), None, stream, C.byref(h)))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = L.IcpResult()
    times = []
    for rep in range(2 + args.reps):
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
        if rep >= 2:
            times.append([1e3 * evs[k].elapsed_time(evs[k + 1]) for k in range(ITERS + 1)])
    L.lib.o3db_icp_destroy(h)
    t = np.array(times)
    med, mn = np.median(t, axis=0), t.min(axis=0)
    print(json.dumps({
        "label": args.label, "card": card(), "reps": args.reps,
        "iteration_us_median": [round(float(x), 1) for x in med[:ITERS]],
        "iteration_us_min": [round(float(x), 1) for x in mn[:ITERS]],
        "evaluate_us_median": round(float(med[ITERS]), 1),
        "sum_of_iterations_ms_median": round(float(np.median(t[:, :ITERS].sum(axis=1))) / 1e3, 4),
        "mean_iteration_us_after_5": round(float(med[5:ITERS].mean()), 1),
        "fitness": res.fitness, "inlier_rmse": res.inlier_rmse,
        "transformation_error_vs_ground_truth": float(np.abs(np.array(res.transformation).reshape(4, 4) - T_gt).max()),
    }), flush=True)


if __name__ == "__main__":
    main()
