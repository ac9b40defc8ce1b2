"""Time of PointCloud.estimate_normals(max_nn=30, radius=0.08) on a 2 M-point cloud, on cuda:0.

    python profiles/normals_time.py [--calls 30] [--out FILE]

The cloud is the target of tests/synth.make_icp_pair(2_000_000, seed=1).  After 5 untimed calls, --calls of each of
the following run between CUDA events:
    index   o3db_nns_create (the cell-sorted copy of the cloud; o3db_nns_destroy is outside the events)
    search  o3db_nns_hybrid_search of the cloud on itself, max_nn 30, into preallocated index / count buffers
    call    the whole o3db_estimate_normals call: index, search, normals kernel, frees, one stream synchronise
A separate phase runs 5 whole calls under torch.profiler for the device time of each kernel; normals_kernel's is the
"normals kernel" time.  The CPU oracle (oracle/normals, the same two steps with the hybrid search of oracle/) runs on
all host threads as the CPU baseline.

Byte model of the normals kernel: each point's count and neighbour indices (4 B + 4 B per neighbour), its own position
read once from DRAM (12 B; the neighbours' positions are the same rows, met again in L1 / L2) and its normal written
(12 B); the bound is those bytes over the 3.35 TB/s of the H100 SXM data sheet.  One JSON line.
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
import open3d_b200 as o3d  # noqa: E402,F401
from open3d_b200 import _lib as L  # noqa: E402
from tests.synth import make_icp_pair  # noqa: E402

N, RADIUS, MAX_NN = 2_000_000, 0.08, 30
HBM_BYTES_PER_S = 3.35e12


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("normals_time.py needs a CUDA device")
    torch.cuda.set_device(0)
    _, tgt, _, _ = make_icp_pair(N, seed=1)
    n = len(tgt)
    p = torch.from_numpy(tgt).cuda()
    nrm = torch.empty_like(p)
    idx = torch.empty((n, MAX_NN), dtype=torch.int32, device="cuda")
    cnt = torch.empty(n, dtype=torch.int32, device="cuda")

    def call():
        L.check(L.lib.o3db_estimate_normals(p.data_ptr(), n, RADIUS, MAX_NN, 0, nrm.data_ptr(), None, stream()))

    def index():
        h = C.c_void_p()
        L.check(L.lib.o3db_nns_create(p.data_ptr(), n, RADIUS, stream(), C.byref(h)))
        return h

    for _ in range(5):
        call()
    torch.cuda.synchronize()
    t_call = timed(call, args.calls)
    t_index = timed(index, args.calls, after=L.lib.o3db_nns_destroy)
    h = index()

    def search():
        L.check(L.lib.o3db_nns_hybrid_search(h, p.data_ptr(), n, RADIUS, MAX_NN, idx.data_ptr(), None, cnt.data_ptr(),
                                             stream()))

    for _ in range(3):
        search()
    t_search = timed(search, args.calls)
    torch.cuda.synchronize()
    L.lib.o3db_nns_destroy(h)
    mean_count = float(cnt.double().mean())

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            call()
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        if e.device_time_total > 0 and "Memset" not in e.key and "Memcpy" not in e.key:
            kernels[e.key.split("(")[0].replace("o3db::", "").replace("void ", "")] = round(e.device_time_total / 5, 1)
    k_us = next((v for k, v in kernels.items() if "normals_kernel" in k), None)
    model_bytes = int(n * (4 + 4 * mean_count + 12 + 12))

    import oracle
    from oracle import normals as on
    threads = oracle.set_num_threads(oracle.host_cores())
    times = []
    for _ in range(3):
        t0 = time.perf_counter()
        on.estimate_normals(tgt, RADIUS, MAX_NN)
        times.append(time.perf_counter() - t0)

    line = {
        "workload": f"estimate_normals(max_nn={MAX_NN}, radius={RADIUS}) of make_icp_pair({N}, seed=1)'s target",
        "card": card(), "points": n, "mean_neighbours": round(mean_count, 3), "calls": args.calls,
        "index": t_index, "search": t_search, "call": t_call,
        "kernel_us_per_call": kernels, "normals_kernel_us": k_us,
        "normals_kernel_byte_model": {
            "bytes": model_bytes, "per": "4 B count + 4 B per neighbour index + 12 B position + 12 B normal, per point",
            "bound_us": round(model_bytes / HBM_BYTES_PER_S * 1e6, 1),
            "fraction_of_3.35TBps": None if k_us is None else round(model_bytes / (k_us * 1e-6) / HBM_BYTES_PER_S, 3)},
        "cpu_baseline": {"impl": "oracle/normals (hybrid search + covariance + fast eigen), OpenMP", "threads": threads,
                         "ms_median": round(1e3 * float(np.median(times)), 1)},
    }
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
