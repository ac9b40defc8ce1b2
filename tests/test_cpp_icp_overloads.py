"""The argument checks of the five registration::ICP overloads of the C++ mirror (include/open3d_b200.hpp): exact
messages, in order, on the host (tests/cpp/icp_overload_checks.cpp).  The program is compiled into a temporary
directory, so the test writes nothing into the tree; it needs nvcc, not a GPU."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "icp_overload_checks.cpp")
LIBDIR = os.path.join(ROOT, "open3d_b200")


def test_icp_overloads_reject_bad_arguments(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "icp_overload_checks")
    build = subprocess.run([nvcc, "-std=c++17", "-O1", "-o", exe, SRC, f"-I{os.path.join(ROOT, 'include')}",
                            f"-L{LIBDIR}", "-lo3db200", "-Xlinker", f"-rpath,{LIBDIR}"],
                           capture_output=True, text=True, timeout=300)
    assert build.returncode == 0, build.stdout + build.stderr
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "icp overload checks ok" in out.stdout, out.stdout + out.stderr
