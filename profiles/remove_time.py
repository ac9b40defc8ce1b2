"""Time of the clean-up filters (PointCloud.remove_radius_outliers, remove_duplicated_points, remove_non_finite_points)
on cuda:0.

    python profiles/remove_time.py [--calls 30] [--out FILE]

Cloud: the target of tests/synth.make_icp_pair(2_000_000, seed=3), about 2 M points of a smooth height field 0.02 apart
(tests/remove_cases.scan_2m).  The radius count runs at radius 0.02 and 0.05 with nb_points 16 and 64; the duplicate
removal on the same cloud with 10 % of its points overwritten by copies of others; the non-finite removal on the cloud
with 1 % of its points given a NaN or infinite coordinate.  After 5 untimed calls, CUDA events around --calls of each
C ABI call and each Python call.  A separate torch.profiler phase gives each kernel's device time.  Every mask is
checked against the CPU oracle (oracle/remove), whose time on all host threads is set beside it.  The card's name,
power limit and SM clock are read in the same run.  One JSON line.
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
from open3d_b200 import _lib as L  # noqa: E402
from tests import remove_cases as rc  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                         text=True, timeout=30).stdout.strip()
    name, power, clock, max_clock = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit": power, "sm_clock": clock, "max_sm_clock": max_clock}


def stream():
    return int(torch.cuda.current_stream().cuda_stream)


def timed(fn, calls):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
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


def host_ms(fn, reps=3):
    times = []
    out = None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        times.append(time.perf_counter() - t0)
    return round(1e3 * float(np.median(times)), 2), out


def kernels_us(fn, reps=5):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_time_total > 0 and "Memcpy" not in e.key:
            out[e.key.split("(")[0].replace("o3db::", "").replace("void ", "")] = round(e.device_time_total / reps, 1)
    return out


def measure(name, pts, abi, python, oracle_fn, calls):
    n = len(pts)
    p = torch.from_numpy(pts).cuda()
    mask = torch.empty(n, dtype=torch.uint8, device="cuda")
    pc = o3d.t.geometry.PointCloud(p)

    def call():
        L.check(abi(p, n, mask))

    t_call = timed(call, calls)
    t_python = timed(lambda: python(pc), calls)
    k = kernels_us(call)
    call()
    torch.cuda.synchronize()
    got = mask.cpu().numpy().astype(bool)
    o_ms, want = host_ms(lambda: oracle_fn(pts))
    return {"case": name, "points": n, "kept": int(got.sum()), "equal_to_oracle": bool(np.array_equal(got, want)),
            "abi_call": t_call, "python_call": t_python, "kernel_us_per_call": k, "oracle_host_ms": o_ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "remove_time.py measures on cuda:0"
    import oracle
    from oracle import remove as orm
    threads = oracle.set_num_threads(oracle.host_cores())
    before = card()
    scan = rc.scan_2m()
    rows = []
    for r in (0.02, 0.05):
        for nb in (16, 64):
            rows.append(measure(
                f"radius_outliers r={r} nb_points={nb}", scan,
                lambda p, n, m, r=r, nb=nb: L.lib.o3db_remove_radius_outliers(p.data_ptr(), n, nb, r, m.data_ptr(),
                                                                              stream()),
                lambda pc, r=r, nb=nb: pc.remove_radius_outliers(nb, r),
                lambda a, r=r, nb=nb: orm.remove_radius_outliers(a, nb, r, "cuda"), args.calls))
    dup = rc.duplicated_2m()
    rows.append(measure(
        "duplicated_points 10 %", dup,
        lambda p, n, m: L.lib.o3db_remove_duplicated_points(p.data_ptr(), n, m.data_ptr(), stream()),
        lambda pc: pc.remove_duplicated_points(), orm.remove_duplicated_points, args.calls))
    bad = scan.copy()
    rng = np.random.default_rng(7)
    idx = rng.choice(len(bad), len(bad) // 100, replace=False)
    bad[idx, rng.integers(0, 3, len(idx))] = np.float32([np.nan, np.inf, -np.inf])[rng.integers(0, 3, len(idx))]
    rows.append(measure(
        "non_finite_points 1 %", bad,
        lambda p, n, m: L.lib.o3db_remove_non_finite_points(p.data_ptr(), n, 1, 1, m.data_ptr(), stream()),
        lambda pc: pc.remove_non_finite_points(), orm.remove_non_finite_points, args.calls))
    line = json.dumps({"card_before": before, "card_after": card(), "oracle_host_threads": threads,
                       "torch": torch.__version__, "rows": rows})
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
