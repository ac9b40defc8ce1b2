"""Resources of the smoothing kernels (smooth.cu), read from the in-tree libo3db200.so with cuobjdump; no GPU needed.

The Laplacian pass and the bilateral kernel use no stack and no local memory.  The MLS kernel's only frame is that of
the eigen solve it shares with normals_kernel (eigen3x3.cuh): the slow-path argument reduction of the f64 cos, which the
solve's arguments in [0, pi] never take, so the MLS kernel's frame must equal normals_kernel's.  The KNN search keeps its two
instantiations."""
import os
import re
import shutil
import subprocess

import pytest

KERNELS = ("smooth_gather_pass_kernel", "smooth_bilateral_kernel")


def _cuobjdump():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return tool


def _resources():
    from open3d_b200 import _lib
    out = subprocess.run([_cuobjdump(), "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    return {k: (int(r), int(s), int(l)) for k, r, s, l in
            re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)}


def _one(res, name):
    hits = [v for k, v in res.items() if name in k]
    assert len(hits) == 1, (name, sorted(k for k in res if name in k))
    return hits[0]


def test_smoothing_kernels_have_no_stack():
    res = _resources()
    for name in KERNELS:
        reg, stack, local = _one(res, name)
        assert stack == 0 and local == 0, (name, reg, stack, local)
    assert _one(res, "smooth_mls_kernel")[1:] == _one(res, "4o3db14normals_kernel")[1:]
    assert sum("knn_search_kernel" in k for k in res) == 2


def test_smoothing_kernels_have_no_local_accesses():
    from open3d_b200 import _lib
    sass = subprocess.run([_cuobjdump(), "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    current, hits, seen = None, {}, set()
    for line in sass.splitlines():
        if "Function :" in line:
            current = line.split("Function :")[1].strip()
            if any(k in current for k in KERNELS):
                seen.add(current)
        elif current is not None and any(k in current for k in KERNELS) and re.search(r"\b(STL|LDL)\b", line):
            hits[current] = hits.get(current, 0) + 1
    assert len(seen) == len(KERNELS), sorted(seen)
    assert not hits, hits
