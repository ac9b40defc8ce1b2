"""Device time of one 30-iteration point-to-plane registration on bench.py's 2 M-point clouds, per ICP search variant.

    python profiles/icp_ab.py [--variants 1 2] [--rounds 12]

Variant 1 = direct loads, 2 = staged (TMA bulk copies + cp.async ring, the default).  The variants run alternately
(the order flips every round), the L2 is flushed before each registration, the first two rounds are warm-up, and the
result is one JSON line with the median / min / max milliseconds per variant.  To compare a compile-time knob (e.g.
-DICP_STAGED_THREADS=512), build a copy of the tree with O3DB_NVCC_EXTRA set and run this script from each copy.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from open3d_b200 import _lib as L  # noqa: E402
from tests.synth import make_icp_pair  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--variants", type=int, nargs="+", default=[1, 2], choices=[1, 2])
ap.add_argument("--rounds", type=int, default=12)
args = ap.parse_args()

stream = int(torch.cuda.current_stream().cuda_stream)
src, tgt, nrm, _ = make_icp_pair(2_000_000, seed=2)
d = [torch.from_numpy(a).cuda() for a in (src, tgt, nrm)]
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
handles, times, results = {}, {v: [] for v in args.variants}, {}
for v in args.variants:
    opt = L.IcpOptions()
    opt.max_correspondence_distance, opt.max_iteration = 0.05, 30
    opt.kernel = L.RobustKernel(0, 1.0, 1.0)
    opt.search_variant = v
    h = C.c_void_p()
    L.check(L.lib.o3db_icp_create(d[0].data_ptr(), len(src), d[1].data_ptr(), d[2].data_ptr(), len(tgt),
                                  L.dptr(np.eye(4)), C.byref(opt), None, stream, C.byref(h)))
    handles[v] = h
for rnd in range(args.rounds):
    for v in (args.variants if rnd % 2 == 0 else args.variants[::-1]):
        L.check(L.lib.o3db_icp_reset(handles[v], stream))
        flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        L.check(L.lib.o3db_icp_iterate(handles[v], 30, stream))
        b.record()
        r = L.IcpResult()
        L.check(L.lib.o3db_icp_finish(handles[v], C.byref(r), None, None, stream))
        torch.cuda.synchronize()
        if rnd >= 2:
            times[v].append(a.elapsed_time(b))
        results[v] = [r.fitness, r.inlier_rmse]
for h in handles.values():
    L.lib.o3db_icp_destroy(h)
print(json.dumps({"device": torch.cuda.get_device_name(), "nvcc_extra": os.environ.get("O3DB_NVCC_EXTRA", ""),
                  "ms_per_30_iterations": {v: {"median": float(np.median(t)), "min": float(np.min(t)),
                                               "max": float(np.max(t)), "n": len(t)} for v, t in times.items()},
                  "fitness_rmse": results}))
