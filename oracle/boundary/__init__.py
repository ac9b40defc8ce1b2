"""ctypes front-end of the CPU oracle of PointCloud::ComputeBoundaryPoints (boundary_oracle.c).

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle``: importable from tests/ and profiles/, never from
``open3d_b200``.

mode "libm" calls libm's atan2f, as the reference does; mode "f64" rounds an f64 atan2 to f32, as the device does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libboundary_oracle.so")
_lib = None

_vp = C.c_void_p
MODES = {"libm": 0, "f64": 1}


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "boundary_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-B", "-C", _HERE, "libboundary_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        for name, res, args in (("orc_boundary_frame_f32", None, [_vp, _vp, _vp]),
                                ("orc_is_boundary_f32", C.c_int, [_vp, C.c_int, C.c_double, _vp]),
                                ("orc_compute_boundary_points_f32", None,
                                 [_vp, _vp, C.c_int64, _vp, C.c_int, _vp, C.c_double, C.c_int, _vp, _vp])):
            getattr(L, name).restype = res
            getattr(L, name).argtypes = args
        _lib = L
    return _lib


def _f32(a, cols):
    return np.ascontiguousarray(a, np.float32).reshape(-1, cols)


def compute_boundary_points_lists(points, normals, idx, cnt, angle_threshold=90.0, mode="f64"):
    """ComputeBoundaryPoints over given neighbour lists idx [n, nn_size] and counts [n] -> (mask bool [n],
    max_gap f32 [n])."""
    p, nrm = _f32(points, 3), _f32(normals, 3)
    idx = np.ascontiguousarray(idx, np.int32)
    cnt = np.ascontiguousarray(cnt, np.int32)
    n = p.shape[0]
    mask = np.zeros(n, np.uint8)
    gap = np.zeros(n, np.float32)
    if n:
        lib().orc_compute_boundary_points_f32(p.ctypes.data, nrm.ctypes.data, n, idx.ctypes.data, idx.shape[1],
                                              cnt.ctypes.data, float(angle_threshold), MODES[mode], mask.ctypes.data,
                                              gap.ctypes.data)
    return mask.astype(bool), gap


def compute_boundary_points(points, normals, radius, max_nn=30, angle_threshold=90.0, mode="f64"):
    """PointCloud::ComputeBoundaryPoints(radius, max_nn, angle_threshold) with the oracle's hybrid search ->
    (mask bool [n], max_gap f32 [n])."""
    p = _f32(points, 3)
    if p.shape[0] == 0:
        return np.zeros(0, bool), np.zeros(0, np.float32)
    idx, _, cnt = oracle.hybrid_search(p, p, radius, int(max_nn))
    return compute_boundary_points_lists(p, normals, idx, cnt, angle_threshold, mode)


def frame(normal):
    """GetCoordinateSystemOnPlane<float> -> (u [3], v [3])."""
    nrm = np.ascontiguousarray(normal, np.float32).reshape(3)
    u = np.zeros(3, np.float32)
    v = np.zeros(3, np.float32)
    lib().orc_boundary_frame_f32(nrm.ctypes.data, u.ctypes.data, v.ctypes.data)
    return u, v


def is_boundary(sorted_angles, angle_threshold):
    """IsBoundaryPoints<float> over sorted angles (at least one) -> (bool, max_gap)."""
    a = np.ascontiguousarray(sorted_angles, np.float32).reshape(-1)
    gap = np.zeros(1, np.float32)
    r = lib().orc_is_boundary_f32(a.ctypes.data, len(a), float(angle_threshold), gap.ctypes.data)
    return bool(r), gap[0]
