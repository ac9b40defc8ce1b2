"""Time of RANSAC plane segmentation (o3db_segment_plane, PointCloud.segment_plane) on cuda:0.
    python profiles/segment_plane_time.py [--calls 5] [--out FILE]
Clouds: 100 k and 2 M points of tests/segment_cases.scene (a height field, a floor plane and uniform outliers).  For
100 and 1000 hypotheses (ransac_n 3, probability 1, so no early stop and every hypothesis is scored), after one
untimed call, --calls C ABI calls (sampling on the host, every launch and the call's one stream synchronise) and
--calls whole PointCloud.segment_plane calls run between CUDA events, each after the same seed.  Every case is
checked against the CPU oracle (oracle/segment) on the same samples.
For comparison on the host: the oracle (OpenMP over the hypotheses of a wave, all host threads) and, where
oracle/_ref/libo3dref_segment.so was built, the reference's own SegmentPlane, whose tbb::parallel_for the shim runs on
one thread.  The card's name, power limit and SM clock are read before and after.  One JSON line.
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
from oracle import segment as sg  # noqa: E402
from tests import segment_cases as sc  # noqa: E402

HYPOTHESES = (100, 1000)
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


def stats(ms):
    return {"median_ms": float(np.median(ms)), "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms))}


def cabi(d, plane, inl, h):
    o3d.utility.random.seed(SEED)
    k = C.c_int64()
    rc = _lib.lib.o3db_segment_plane(d.data_ptr(), d.shape[0], sc.THRESHOLD, 3, h, 1.0, plane.data_ptr(),
                                     inl.data_ptr(), C.byref(k), None, int(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, _lib.last_error()
    return k.value


def python_call(pc, h):
    o3d.utility.random.seed(SEED)
    return pc.segment_plane(sc.THRESHOLD, 3, h, 1.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "segment_plane_time.py measures on cuda:0"
    torch.cuda.set_device(0)
    res = {"card": card(), "calls": args.calls, "host_threads": os.cpu_count(), "cases": {}}
    for cname, n in (("scene_100k", 100_000), ("scene_2M", 2_000_000)):
        p = sc.scene(n, 7)
        d = torch.from_numpy(p).cuda()
        pc = o3d.t.geometry.PointCloud(d)
        plane = torch.empty(4, dtype=torch.float64, device="cuda")
        inl = torch.empty(n, dtype=torch.int64, device="cuda")
        for h in HYPOTHESES:
            k = cabi(d, plane, inl, h)
            o3d.utility.random.seed(SEED)
            s = np.zeros((h, 3), np.int64)
            _lib.check(_lib.lib.o3db_random_sample_indices(n, 3, h, s.ctypes.data))
            t0 = time.perf_counter()
            want = sg.segment_plane(p, s, sc.THRESHOLD, 1.0)
            oracle_ms = (time.perf_counter() - t0) * 1e3
            case = {"points": n, "hypotheses": h, "inliers": k,
                    "equal_to_oracle": bool(np.array_equal(inl[:k].cpu().numpy(), want.inliers)
                                            and plane.cpu().numpy().tobytes() == want.plane.tobytes()),
                    "cabi": stats([event_ms(lambda: cabi(d, plane, inl, h)) for _ in range(args.calls)])}
            python_call(pc, h)
            case["python_call"] = stats([event_ms(lambda: python_call(pc, h)) for _ in range(args.calls)])
            case["oracle_all_threads_ms"] = oracle_ms
            if sg.ref() is not None:
                sg.ref_seed(SEED)
                t0 = time.perf_counter()
                r = sg.ref_segment_plane(p, sc.THRESHOLD, 3, h, 1.0)
                case["reference_one_thread_ms"] = (time.perf_counter() - t0) * 1e3
                case["reference_same_inliers"] = bool(np.array_equal(r.inliers, want.inliers))
            res["cases"][f"{cname}_{h}"] = case
        del d, pc, inl
        torch.cuda.empty_cache()
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
