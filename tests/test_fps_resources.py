"""Resources of the farthest-point down-sampling kernel (fps.cu), read from the in-tree libo3db200.so with cuobjdump,
and its entry point's failure without a device; no GPU needed.  The kernel uses no stack and no local memory: its
running minima must stay in registers."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

KERNEL = "fps_kernel"


def _cuobjdump():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return tool


def test_fps_kernel_has_no_stack():
    from open3d_b200 import _lib
    out = subprocess.run([_cuobjdump(), "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    res = {k: (int(s), int(l)) for k, s, l in
           re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)}
    hits = [v for k, v in res.items() if KERNEL in k]
    assert len(hits) == 1, hits
    assert hits[0] == (0, 0), hits[0]


def test_fps_kernel_has_no_local_accesses():
    from open3d_b200 import _lib
    sass = subprocess.run([_cuobjdump(), "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    current, hits, seen = None, 0, set()
    for line in sass.splitlines():
        if "Function :" in line:
            current = line.split("Function :")[1].strip()
            if KERNEL in current:
                seen.add(current)
        elif current is not None and KERNEL in current and re.search(r"\b(STL|LDL)\b", line):
            hits += 1
    assert len(seen) == 1, sorted(seen)
    assert hits == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="exercises the no-GPU failure path")
def test_no_cpu_fallback():
    from open3d_b200 import _lib as L
    p = np.zeros((16, 3), np.float32)
    sel = np.zeros(4, np.int32)
    rc = L.lib.o3db_farthest_point_down_sample(p.ctypes.data, 16, 4, 0, sel.ctypes.data, None)
    assert rc == L.ERR_CUDA and "cuda" in L.last_error().lower(), (rc, L.last_error())
