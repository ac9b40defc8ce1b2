"""Time of farthest-point down-sampling (o3db_farthest_point_down_sample, PointCloud.farthest_point_down_sample) on
cuda:0.

    python profiles/fps_time.py [--calls 5] [--torch-samples 512] [--out FILE]

Clouds: 100 k points uniform in the unit cube (tests/knn_cases.uniform), the target of
tests/synth.make_icp_pair(2_000_000, seed=1), and 4 M uniform points, above the kernel's on-chip capacity of
18432 points per SM.  For 1 k and 8 k samples, after one untimed call, --calls C ABI calls (the one cooperative launch
and the call's one stream synchronise) and --calls whole PointCloud.farthest_point_down_sample calls (with the sort and
the gather of the result) run between CUDA events; the per-round time is the C ABI call's over num_samples - 1.  The
100 k selections are checked against the CPU oracle (oracle/fps).

For comparison, upstream's device loop (t/geometry/PointCloud.cpp:633-645) restated as torch ops on the same GPU: per
sample the mask write, subtract, multiply, sum, minimum and argmax, and an .item(); timed at --torch-samples samples
because it is slow, and reported per round.  The card's name, power limit and SM clock are read before and after.  One
JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import open3d_b200 as o3d  # noqa: E402
from open3d_b200 import _lib  # noqa: E402
from oracle import fps as of  # noqa: E402
from tests import knn_cases as kc  # noqa: E402
from tests.synth import make_icp_pair  # noqa: E402

SAMPLES = (1000, 8000)


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


def cabi(d, out, m):
    rc = _lib.lib.o3db_farthest_point_down_sample(d.data_ptr(), d.shape[0], m, 0, out.data_ptr(),
                                                  int(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, _lib.last_error()


def torch_loop(pos, m):
    """upstream's tensor loop, op for op"""
    n = pos.shape[0]
    mask = torch.zeros(n, dtype=torch.bool, device=pos.device)
    dist = torch.full((n,), float("inf"), dtype=pos.dtype, device=pos.device)
    f = 0
    for _ in range(m):
        mask[f] = True
        diff = pos - pos[f]
        dist = torch.minimum((diff * diff).sum(1), dist)
        f = int(dist.argmax(0).item())
    return mask


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--torch-samples", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "fps_time.py measures on cuda:0"
    torch.cuda.set_device(0)
    res = {"card": card(), "calls": args.calls, "cases": {}, "torch_loop": {"samples": args.torch_samples}}
    clouds = {"uniform_100k": kc.uniform(100_000, seed=1), "icp_target_2M": make_icp_pair(2_000_000, seed=1)[1],
              "uniform_4M": kc.uniform(4_000_000, seed=2)}
    for cname, p in clouds.items():
        d = torch.from_numpy(p).cuda()
        pc = o3d.t.geometry.PointCloud(p)
        for m in SAMPLES:
            out = torch.empty(m, dtype=torch.int32, device="cuda")
            cabi(d, out, m)
            case = {"points": len(p), "num_samples": m}
            if len(p) <= 100_000:
                case["equal_to_oracle"] = bool(np.array_equal(out.cpu().numpy(), of.farthest_point_down_sample(p, m)))
            t = stats([event_ms(lambda: cabi(d, out, m)) for _ in range(args.calls)])
            case["cabi"] = t
            case["per_round_us"] = t["median_ms"] * 1e3 / (m - 1)
            pc.farthest_point_down_sample(m)
            case["python_call"] = stats([event_ms(lambda: pc.farthest_point_down_sample(m)) for _ in range(args.calls)])
            res["cases"][f"{cname}_{m}"] = case
        torch_loop(d, 8)
        ms = event_ms(lambda: torch_loop(d, args.torch_samples))
        res["torch_loop"][cname] = {"points": len(p), "ms": ms, "per_round_us": ms * 1e3 / args.torch_samples}
        del d, pc
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
