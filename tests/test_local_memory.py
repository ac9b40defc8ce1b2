"""The per-query partial sums of the fused ICP and odometry kernels stay in registers.

Each lane of icp_iteration_kernel and odometry_level_kernel keeps a 32-float term array and sums it over the warp with
the transposed reduction of reduce.cuh.  If ptxas places that array in local memory, every 32-query chunk stores and
reloads it through L1 / L2: the port of the same source from sm_100a to sm_90a did exactly that (176 B of stack per
thread, STL.128 / LDL.128 in the loop) and lost 4.7x of ICP speed with no test noticing, because the results do not
change.  This reads the resource usage and the SASS of the in-tree libo3db200.so and needs no GPU."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = ("icp_iteration_kernel", "odometry_level_kernel")
MAX_STACK = 128   # bytes: one 32-float array


def _cuobjdump():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return tool


def _ours(name):
    return any(k in name for k in KERNELS)


def test_fused_kernels_keep_their_term_arrays_off_the_stack():
    from open3d_b200 import _lib
    out = subprocess.run([_cuobjdump(), "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    stacks = dict(re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)", out))
    ours = {k: int(v) for k, v in stacks.items() if _ours(k)}
    assert sum("icp_iteration_kernel" in k for k in ours) == 5 and sum("odometry_level_kernel" in k for k in ours) == 1, ours
    big = {k: v for k, v in ours.items() if v >= MAX_STACK}
    assert not big, f"stack frames of {MAX_STACK} B or more (a per-lane array in local memory): {big}"


def test_fused_kernels_have_no_vector_local_accesses():
    from open3d_b200 import _lib
    sass = subprocess.run([_cuobjdump(), "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    current, hits, seen = None, {}, set()
    for line in sass.splitlines():
        if "Function :" in line:
            current = line.split("Function :")[1].strip()
            if _ours(current):
                seen.add(current)
        elif current is not None and _ours(current):
            m = re.search(r"\b(STL|LDL)\.128\b", line)
            if m:
                hits[current] = hits.get(current, 0) + 1
    assert len(seen) == 6, sorted(seen)
    assert not hits, f"128-bit local loads / stores (a per-lane array in local memory): {hits}"
