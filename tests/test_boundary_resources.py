"""Resources of the boundary-detection kernels (boundary.cu), read from the in-tree libo3db200.so with cuobjdump, and
its entry point's failure without a device; no GPU needed.  The boundary kernel keeps each neighbour's angle in its
lane's registers and sorts them with warp shuffles, so neither kernel uses stack or local memory."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

KERNELS = ("boundary_kernel", "boundary_check_kernel")


def _cuobjdump():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return tool


def _name(mangled):
    m = re.search(r"o3db\d+(\w+?)E", mangled)
    return m.group(1) if m else None


def test_boundary_kernels_have_no_stack():
    from open3d_b200 import _lib
    out = subprocess.run([_cuobjdump(), "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    res = {k: (int(s), int(l)) for k, s, l in
           re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)}
    for kernel in KERNELS:
        hits = [v for k, v in res.items() if _name(k) == kernel]
        assert len(hits) == 1, (kernel, hits)
        assert hits[0] == (0, 0), (kernel, hits[0])


def test_boundary_kernels_have_no_local_accesses():
    from open3d_b200 import _lib
    sass = subprocess.run([_cuobjdump(), "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    current, hits, seen = None, 0, set()
    for line in sass.splitlines():
        if "Function :" in line:
            current = _name(line.split("Function :")[1].strip())
            if current in KERNELS:
                seen.add(current)
        elif current in KERNELS and re.search(r"\b(STL|LDL)\b", line):
            hits += 1
    assert seen == set(KERNELS), sorted(seen)
    assert hits == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="exercises the no-GPU failure path")
def test_no_cpu_fallback():
    from open3d_b200 import _lib as L
    p = np.zeros((16, 3), np.float32)
    q = np.zeros((16, 3), np.float32)
    mask = np.zeros(16, np.uint8)
    rc = L.lib.o3db_compute_boundary_points(p.ctypes.data, q.ctypes.data, 16, 0.05, 30, 90.0, mask.ctypes.data, None,
                                            None)
    assert rc == L.ERR_CUDA and "cuda" in L.last_error().lower(), (rc, L.last_error())
