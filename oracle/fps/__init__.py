"""ctypes front-end of the CPU oracle of farthest-point down-sampling, PointCloud::FarthestPointDownSample
(fps_oracle.c).

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle``: importable from tests/ and profiles/, never from
``open3d_b200``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libfps_oracle.so")
_lib = None


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "fps_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-B", "-C", _HERE, "libfps_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        L.orc_fps.restype = C.c_int
        L.orc_fps.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p]
        _lib = L
    return _lib


def farthest_point_down_sample(points, num_samples, start_index=0):
    """-> [num_samples] int32: the selected indices in selection order (sort them for upstream's output order)."""
    p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    out = np.empty(int(num_samples), np.int32)
    rc = lib().orc_fps(p.ctypes.data, p.shape[0], int(num_samples), int(start_index), out.ctypes.data)
    if rc == -2:
        raise MemoryError("orc_fps: out of memory")
    if rc:
        raise ValueError(f"orc_fps: bad arguments (n={p.shape[0]}, num_samples={num_samples}, "
                         f"start_index={start_index})")
    return out
