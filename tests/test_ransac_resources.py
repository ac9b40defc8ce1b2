"""Resources of the RANSAC registration kernels (ransac.cu), read from the in-tree libo3db200.so with
cuobjdump, and its entry point's failure without a device; no GPU needed.  No kernel uses stack or local memory: the
hypothesis's estimate and the search's best match stay in registers."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

KERNELS = ("ransac_hypothesis_kernel", "ransac_compact_kernel", "ransac_validate_kernel", "ransac_select_kernel",
           "ransac_emit_kernel", "ransac_check_kernel", "ransac_finite_kernel")


def _cuobjdump():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return tool


def test_ransac_kernels_have_no_stack():
    from open3d_b200 import _lib
    out = subprocess.run([_cuobjdump(), "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    res = {k: (int(s), int(l)) for k, s, l in
           re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)}
    for kernel in KERNELS:
        hits = [v for k, v in res.items() if kernel in k]
        assert len(hits) == 1, (kernel, hits)
        assert hits[0] == (0, 0), (kernel, hits[0])


def test_ransac_kernels_have_no_local_accesses():
    from open3d_b200 import _lib
    sass = subprocess.run([_cuobjdump(), "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    current, hits, seen = None, 0, set()
    for line in sass.splitlines():
        if "Function :" in line:
            current = line.split("Function :")[1].strip()
            if "ransac_" in current:
                seen.add(current)
        elif current is not None and "ransac_" in current and re.search(r"\b(STL|LDL)\b", line):
            hits += 1
    assert len(seen) == len(KERNELS), sorted(seen)
    assert hits == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="exercises the no-GPU failure path")
def test_no_cpu_fallback():
    from open3d_b200 import _lib as L
    p = np.zeros((16, 3), np.float32)
    c = np.stack([np.arange(16), np.arange(16)], 1).astype(np.int64)
    T = np.zeros(16)
    out = np.zeros(16, np.int64)
    rc = L.lib.o3db_registration_ransac(p.ctypes.data, None, 16, p.ctypes.data, None, 16, c.ctypes.data, 16, 0.1, 3,
                                        10, 0.999, None, T.ctypes.data, out.ctypes.data, None, None)
    assert rc == L.ERR_CUDA and "cuda" in L.last_error().lower(), (rc, L.last_error())
