"""Resources of the clean-up filter kernels (remove.cu), read from the in-tree libo3db200.so with cuobjdump, and the
entry points' failure without a device; no GPU needed.  Every kernel keeps its state in registers: none uses stack
or local memory."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

KERNELS = ("remove_radius_kernel", "remove_finite_kernel", "remove_dup_claim_kernel", "remove_dup_first_kernel",
           "remove_dup_mask_kernel", "remove_non_finite_kernel")


def _cuobjdump():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return tool


def _name(mangled):
    m = re.search(r"o3db\d+(\w+?)E", mangled)
    return m.group(1) if m else None


def test_remove_kernels_have_no_stack():
    from open3d_b200 import _lib
    out = subprocess.run([_cuobjdump(), "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    res = {k: (int(s), int(l)) for k, s, l in
           re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)}
    for kernel in KERNELS:
        hits = [v for k, v in res.items() if _name(k) == kernel]
        assert len(hits) == 1, (kernel, hits)
        assert hits[0] == (0, 0), (kernel, hits[0])


def test_remove_kernels_have_no_local_accesses():
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


def test_argument_errors_before_any_cuda_call():
    from open3d_b200 import _lib as L
    p = np.zeros((4, 3), np.float32)
    mask = np.zeros(4, np.uint8)
    for nb, r in ((0, 0.1), (3, 0.0), (3, -1.0)):
        rc = L.lib.o3db_remove_radius_outliers(p.ctypes.data, 4, nb, r, mask.ctypes.data, None)
        assert rc == L.ERR_INVALID and "number of points and radius must be positive" in L.last_error()
    for r in (float("nan"), float("inf")):
        rc = L.lib.o3db_remove_radius_outliers(p.ctypes.data, 4, 3, r, mask.ctypes.data, None)
        assert rc == L.ERR_INVALID and "finite" in L.last_error(), L.last_error()
    assert L.lib.o3db_remove_radius_outliers(None, 4, 3, 0.1, mask.ctypes.data, None) == L.ERR_INVALID
    assert L.lib.o3db_remove_duplicated_points(p.ctypes.data, -1, mask.ctypes.data, None) == L.ERR_INVALID
    assert L.lib.o3db_remove_non_finite_points(p.ctypes.data, 4, 1, 1, None, None) == L.ERR_INVALID


@pytest.mark.skipif(torch.cuda.is_available(), reason="exercises the no-GPU failure path")
def test_no_cpu_fallback():
    from open3d_b200 import _lib as L
    p = np.zeros((16, 3), np.float32)
    mask = np.zeros(16, np.uint8)
    for rc in (L.lib.o3db_remove_radius_outliers(p.ctypes.data, 16, 2, 0.05, mask.ctypes.data, None),
               L.lib.o3db_remove_duplicated_points(p.ctypes.data, 16, mask.ctypes.data, None),
               L.lib.o3db_remove_non_finite_points(p.ctypes.data, 16, 1, 1, mask.ctypes.data, None)):
        assert rc == L.ERR_CUDA and "cuda" in L.last_error().lower(), (rc, L.last_error())
