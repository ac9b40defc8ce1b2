"""The symmetric iteration kernels keep their term arrays, the recentring and the half-angle step in registers: no
stack frame, no local loads or stores, and the 80 registers that 768 threads per SM allow.  Reads the in-tree
libo3db200.so with cuobjdump; needs no GPU (tests/test_local_memory.py does the same for the other instantiations)."""
import os
import re
import shutil
import subprocess

import pytest

KERNEL = "icp_symmetric_iteration_kernel"


def test_symmetric_iteration_kernels_use_no_stack():
    from open3d_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    usage = [(int(r), int(s)) for k, r, s in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", out) if KERNEL in k]
    assert len(usage) == 3, usage   # iteration <L2>, iteration <robust>, evaluation pass
    assert all(r <= 80 and s == 0 for r, s in usage), usage
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    bodies = [part for part in sass.split("Function :")[1:] if KERNEL in part.splitlines()[0]]
    assert len(bodies) == 3
    for body in bodies:
        assert "UBLKCP" in body and "LDGSTS" in body and not re.search(r"\b(STL|LDL)\b", body)
