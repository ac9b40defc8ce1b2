"""Resources of the triangle-mesh extraction kernels (extract.cu), read from the in-tree libo3db200.so with cuobjdump; no GPU needed.
Every kernel uses no stack and no local memory."""
import os
import re
import shutil
import subprocess

import pytest

KERNELS = ("mesh_classify_kernel", "mesh_count_kernel", "mesh_triangle_kernel")


def _cuobjdump():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return tool


def test_mesh_kernels_have_no_stack():
    from open3d_b200 import _lib
    out = subprocess.run([_cuobjdump(), "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    res = {k: (int(s), int(l)) for k, s, l in
           re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)}
    for name in KERNELS:
        hits = [v for k, v in res.items() if name in k]
        assert len(hits) == 1, (name, hits)
        assert hits[0] == (0, 0), (name, hits[0])


def test_mesh_kernels_have_no_local_accesses():
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
