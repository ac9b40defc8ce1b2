"""The k-nearest-neighbour search kernel keeps its running list in registers: no stack frame, no local loads or
stores, and at most the 80 registers that three 256-thread CTAs per SM allow.  Reads the in-tree libo3db200.so with
cuobjdump; needs no GPU."""
import os
import re
import shutil
import subprocess

import pytest

KERNEL = "knn_search_kernel"


def test_knn_search_kernel_uses_no_local_memory():
    from open3d_b200 import _lib
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([tool, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    usage = [(int(r), int(s)) for k, r, s in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", out) if KERNEL in k]
    assert len(usage) == 2, usage   # Int32 and Int64 indices
    assert all(r <= 80 and s == 0 for r, s in usage), usage
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    bodies = [part for part in sass.split("Function :")[1:] if KERNEL in part.splitlines()[0]]
    assert len(bodies) == 2
    for body in bodies:
        assert not re.search(r"\b(STL|LDL)\b", body)
