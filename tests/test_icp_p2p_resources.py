"""The point-to-point iteration kernel keeps its term array and the Kabsch step's matrices in registers: no stack
frame, no local loads or stores, and the 80 registers that 768 threads per SM allow.  Reads the in-tree
libo3db200.so with cuobjdump; needs no GPU (tests/test_local_memory.py does the same for the other instantiations)."""
import os
import re
import shutil
import subprocess

import pytest

KERNEL = "icp_point_iteration_kernel"


def test_point_iteration_kernel_uses_no_stack():
    from open3d_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    usage = [(int(r), int(s)) for k, r, s in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", out) if KERNEL in k]
    assert len(usage) == 1, usage
    assert usage[0][0] <= 80 and usage[0][1] == 0, usage
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    body = [part for part in sass.split("Function :")[1:] if KERNEL in part.splitlines()[0]]
    assert len(body) == 1
    assert "UBLKCP" in body[0] and "LDGSTS" in body[0] and not re.search(r"\b(STL|LDL)\b", body[0])
