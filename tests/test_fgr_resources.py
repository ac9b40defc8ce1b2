"""Resources of the Fast Global Registration kernels (fgr.cu), read from the in-tree libo3db200.so with cuobjdump,
and its entry point's failure without a device; no GPU needed.  No kernel uses stack or local memory: the 6x6 solve
works in shared memory and the search's best match stays in registers."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

KERNELS = ("fgr_check_kernel", "fgr_mean_kernel", "fgr_scale_kernel", "fgr_tuple_kernel", "fgr_stop_kernel",
           "fgr_tuple_compact_kernel", "fgr_optimize_kernel", "fgr_transform_kernel", "fgr_eval_kernel",
           "fgr_sum_kernel", "fgr_finite_kernel")


def _cuobjdump():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return tool


def test_fgr_kernels_have_no_stack():
    from open3d_b200 import _lib
    out = subprocess.run([_cuobjdump(), "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    res = {k: (int(s), int(l)) for k, s, l in
           re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)}
    for kernel in KERNELS:
        hits = [v for k, v in res.items() if f"{kernel}E" in k]
        assert len(hits) == 1, (kernel, hits)
        assert hits[0] == (0, 0), (kernel, hits[0])


def test_fgr_kernels_have_no_local_accesses():
    from open3d_b200 import _lib
    sass = subprocess.run([_cuobjdump(), "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    current, hits, seen = None, 0, set()
    for line in sass.splitlines():
        if "Function :" in line:
            current = line.split("Function :")[1].strip()
            if "fgr_" in current:
                seen.add(current)
        elif current is not None and "fgr_" in current and re.search(r"\b(STL|LDL)\b", line):
            hits += 1
    assert len(seen) == len(KERNELS), sorted(seen)
    assert hits == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="exercises the no-GPU failure path")
def test_no_cpu_fallback():
    from open3d_b200 import _lib as L
    p = np.random.default_rng(0).uniform(-1, 1, (16, 3)).astype(np.float32)
    c = np.stack([np.arange(16), np.arange(16)], 1).astype(np.int64)
    T = np.zeros(16)
    out = np.zeros(16, np.int64)
    opt = L.FgrOption(1.4, 0, 0, 0.025, 64, 0.95, 1000, 1)
    rc = L.lib.o3db_registration_fgr(p.ctypes.data, 16, p.ctypes.data, 16, c.ctypes.data, 16, None, None, 0,
                                     C.byref(opt), T.ctypes.data, out.ctypes.data, None, None)
    assert rc == L.ERR_CUDA and "cuda" in L.last_error().lower(), (rc, L.last_error())
