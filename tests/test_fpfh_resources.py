"""Resources of the FPFH kernels (fpfh.cu) and of the wide KNN walk that gives them their lists (knn.cu's
knn_lists_kernel), read from the in-tree libo3db200.so with cuobjdump; no GPU needed.  The wide walk keeps its four
keys per lane in registers; no kernel uses stack or local memory."""
import os
import re
import shutil
import subprocess

import pytest

KERNELS = ("knn_lists_kernel", "knn_finite_kernel", "fpfh_check_kernel", "fpfh_select_kernel", "fpfh_compact_kernel", "fpfh_gather_kernel",
           "fpfh_mark_kernel", "fpfh_spfh_kernel", "fpfh_kernel", "feature_nn_kernel", "mutual_flag_kernel",
           "corres_write_kernel")


def _cuobjdump():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not available")
    return tool


def _name(mangled):
    m = re.search(r"o3db\d+(\w+?)E", mangled)
    return m.group(1) if m else None


def test_fpfh_kernels_have_no_stack():
    from open3d_b200 import _lib
    out = subprocess.run([_cuobjdump(), "-res-usage", _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    res = {k: (int(r), int(s), int(l)) for k, r, s, l in
           re.findall(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", out)}
    for kernel in KERNELS:
        hits = [v for k, v in res.items() if _name(k) == kernel]
        assert len(hits) == 1, (kernel, hits)
        assert hits[0][1:] == (0, 0), (kernel, hits[0])
    wide = [v for k, v in res.items() if _name(k) == "knn_lists_kernel"][0]
    assert wide[0] <= 80, wide   # three 256-thread CTAs per SM, as knn_search_kernel


def test_fpfh_kernels_have_no_local_accesses():
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
