"""ctypes front-end of the CPU oracle of DBSCAN clustering, PointCloud::ClusterDBSCAN (dbscan_oracle.c).

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle``: importable from tests/ and profiles/, never from
``open3d_b200``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libdbscan_oracle.so")
_lib = None

_vp = C.c_void_p


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "dbscan_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-B", "-C", _HERE, "libdbscan_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        L.orc_dbscan.restype = C.c_int64
        L.orc_dbscan.argtypes = [_vp, C.c_int64, C.c_double, C.c_int64, C.c_int, _vp, _vp]
        L.orc_dbscan_core.restype = C.c_int
        L.orc_dbscan_core.argtypes = [_vp, C.c_int64, C.c_double, C.c_int64, C.c_int, _vp]
        _lib = L
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, np.float32).reshape(-1, 3)


def cluster_dbscan(points, eps, min_points, bruteforce=False, return_core=False):
    """PointCloud::ClusterDBSCAN(eps, min_points) -> labels [n] int32 (-1 noise), and the core flags [n] bool with
    return_core.  bruteforce: neighbours by a scan of every point instead of the grid."""
    p = _f32(points)
    n = p.shape[0]
    labels = np.empty(n, np.int32)
    core = np.empty(n, np.uint8)
    rc = lib().orc_dbscan(p.ctypes.data, n, float(eps), int(min_points), int(bool(bruteforce)), labels.ctypes.data,
                          core.ctypes.data)
    if rc < 0:
        raise MemoryError("orc_dbscan: out of memory")
    return (labels, core.astype(bool)) if return_core else labels


def core_points(points, eps, min_points, bruteforce=False):
    """-> [n] bool: the points with at least min_points neighbours (d2 < eps^2), themselves included."""
    p = _f32(points)
    core = np.empty(p.shape[0], np.uint8)
    if lib().orc_dbscan_core(p.ctypes.data, p.shape[0], float(eps), int(min_points), int(bool(bruteforce)),
                             core.ctypes.data):
        raise MemoryError("orc_dbscan_core: out of memory")
    return core.astype(bool)
