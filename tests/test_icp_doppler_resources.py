"""The Doppler iteration kernels keep their term arrays in registers: no spills, no local loads or stores in the
per-query loop, and at most the 80 registers that 768 threads per SM allow.  The only stack frame is the 40 bytes of
the f64 cos / sin slow path in the Gauss-Newton step they share with the point-to-plane iteration kernels, and its
local accesses are that path's.  Reads the in-tree libo3db200.so with cuobjdump; needs no GPU."""
import os
import re
import shutil
import subprocess

import pytest

KERNEL = "icp_doppler_iteration_kernel"
PLANE_L2 = "_ZN4o3db20icp_iteration_kernelILb1ELi0ELb0EEEvNS_7IcpArgsE"


def _tool():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return tool


def test_doppler_iteration_kernels_use_registers_only():
    from open3d_b200 import _lib
    tool = _tool()
    out = subprocess.run([tool, "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    usage = dict((k, (int(r), int(s))) for k, r, s in re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", out))
    ours = {k: v for k, v in usage.items() if KERNEL in k}
    assert len(ours) == 3, ours   # iteration <L2>, iteration <robust>, evaluation pass
    plane_stack = usage[PLANE_L2][1]
    assert all(r <= 80 and s <= plane_stack for r, s in ours.values()), (ours, plane_stack)
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    bodies = {part.splitlines()[0].strip(): part for part in sass.split("Function :")[1:]}
    local = lambda body: len(re.findall(r"\b(STL|LDL)\b", body))   # noqa: E731
    for name, body in bodies.items():
        if KERNEL not in name:
            continue
        assert "UBLKCP" in body and "LDGSTS" in body
        # as many local accesses as the point-to-plane kernel's Gauss-Newton step (0 for the evaluation pass)
        assert local(body) == (0 if "Li1E" in name else local(bodies[PLANE_L2])), name
