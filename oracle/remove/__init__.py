"""ctypes front-end of the CPU oracle of PointCloud::RemoveRadiusOutliers, RemoveDuplicatedPoints and
RemoveNonFinitePoints (remove_oracle.c).

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle``: importable from tests/ and profiles/, never from
``open3d_b200``.

mode "cuda" is upstream's CUDA distance test as nvcc contracts it, mode "plain" the same expression uncontracted.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libremove_oracle.so")
_lib = None

_vp = C.c_void_p
_i64 = C.c_int64
MODES = {"cuda": 0, "plain": 1}


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "remove_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-B", "-C", _HERE, "libremove_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        for name, res, args in (("orc_radius_counts_brute", None, [_vp, _i64, C.c_double, C.c_int, _i64, _vp]),
                                ("orc_radius_counts_grid", C.c_int, [_vp, _i64, C.c_double, C.c_int, _i64, _vp]),
                                ("orc_remove_duplicated_points", C.c_int, [_vp, _i64, _vp]),
                                ("orc_remove_non_finite_points", None, [_vp, _i64, C.c_int, C.c_int, _vp])):
            getattr(L, name).restype = res
            getattr(L, name).argtypes = args
        _lib = L
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, np.float32).reshape(-1, 3)


def radius_counts(points, radius, mode="cuda", cap=0, brute=False):
    """int64 [n]: the number of points within radius of each point, itself included, stopping at cap (0: no cap).
    brute=True compares all pairs; otherwise a grid, which needs finite coordinates."""
    p = _f32(points)
    n = p.shape[0]
    counts = np.zeros(n, np.int64)
    if brute:
        lib().orc_radius_counts_brute(p.ctypes.data, n, float(radius), MODES[mode], int(cap), counts.ctypes.data)
    elif lib().orc_radius_counts_grid(p.ctypes.data, n, float(radius), MODES[mode], int(cap), counts.ctypes.data):
        raise ValueError("radius_counts: non-finite coordinates (or out of memory)")
    return counts


def remove_radius_outliers(points, nb_points, search_radius, mode="cuda", brute=False):
    """RemoveRadiusOutliers' mask, bool [n]: at least nb_points points within search_radius."""
    return radius_counts(points, search_radius, mode, int(nb_points), brute) >= int(nb_points)


def remove_duplicated_points(points):
    """RemoveDuplicatedPoints' mask, bool [n]: the first occurrence of every bit pattern of the coordinates."""
    p = _f32(points)
    mask = np.zeros(p.shape[0], np.uint8)
    if lib().orc_remove_duplicated_points(p.ctypes.data, p.shape[0], mask.ctypes.data):
        raise MemoryError("remove_duplicated_points")
    return mask.astype(bool)


def remove_non_finite_points(points, remove_nan=True, remove_inf=True):
    """RemoveNonFinitePoints' mask, bool [n]."""
    p = _f32(points)
    mask = np.zeros(p.shape[0], np.uint8)
    lib().orc_remove_non_finite_points(p.ctypes.data, p.shape[0], int(bool(remove_nan)), int(bool(remove_inf)),
                                       mask.ctypes.data)
    return mask.astype(bool)
