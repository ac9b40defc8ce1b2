"""ctypes front-end of the CPU oracle of the point-cloud <-> image projection (projection_oracle.c).

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle``: importable from tests/ and profiles/, never from
``open3d_b200``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libprojection_oracle.so")
_lib = None

_vp = C.c_void_p


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "projection_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-B", "-C", _HERE, "libprojection_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        L.orc_unproject.restype = C.c_int64
        L.orc_unproject.argtypes = [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int, _vp, _vp, C.c_float, C.c_float,
                                    C.c_int, _vp, _vp]
        L.orc_project.restype = C.c_int
        L.orc_project.argtypes = [_vp, _vp, C.c_int64, _vp, _vp, C.c_float, C.c_float, C.c_int, C.c_int, _vp, _vp]
        _lib = L
    return _lib


def _f64(a, shape):
    return np.ascontiguousarray(np.asarray(a, np.float64).reshape(shape))


def unproject(depth, K, extrinsic=None, depth_scale=1000.0, depth_max=3.0, stride=1, color=None):
    """kernel::pointcloud::Unproject -> points [N,3] f32, or (points, colors) with a colour image.  depth: [H,W] (or
    [H,W,1]) u16 / f32; color: [H,W,3] u8 / f32, copied as f32 without scaling.  Rows row-major over the strided
    grid."""
    d = np.ascontiguousarray(depth)
    assert d.dtype in (np.uint16, np.float32), d.dtype
    rows, cols = d.shape[0], d.shape[1]
    c = None if color is None else np.ascontiguousarray(color)
    if c is not None:
        assert c.dtype in (np.uint8, np.float32) and c.shape[:2] == (rows, cols) and c.shape[-1] == 3
    E = np.eye(4) if extrinsic is None else extrinsic
    pose = _f64(oracle.inverse_transformation(_f64(E, (4, 4))), 16)
    cap = (rows // stride) * (cols // stride)
    pts = np.zeros((cap, 3), np.float32)
    col = np.zeros((cap, 3), np.float32) if c is not None else None
    n = lib().orc_unproject(d.ctypes.data, int(d.dtype == np.float32), rows, cols,
                            None if c is None else c.ctypes.data, int(c is not None and c.dtype == np.float32),
                            _f64(K, 9).ctypes.data, pose.ctypes.data, float(depth_scale), float(depth_max), int(stride),
                            pts.ctypes.data, None if col is None else col.ctypes.data)
    if c is None:
        return pts[:n].copy()
    return pts[:n].copy(), col[:n].copy()


def project(points, K, extrinsic=None, width=640, height=480, depth_scale=1000.0, depth_max=3.0, colors=None):
    """kernel::pointcloud::Project with the packed (depth bits, index) minimum per pixel -> depth [H,W,1] f32, or
    (depth, color [H,W,3] f32) when colors is given."""
    p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    c = None if colors is None else np.ascontiguousarray(colors, np.float32).reshape(-1, 3)
    E = np.eye(4) if extrinsic is None else extrinsic
    depth = np.zeros((height, width, 1), np.float32)
    color = np.zeros((height, width, 3), np.float32) if c is not None else None
    rc = lib().orc_project(p.ctypes.data, None if c is None else c.ctypes.data, p.shape[0], _f64(K, 9).ctypes.data,
                           _f64(E, 16).ctypes.data, float(depth_scale), float(depth_max), int(height), int(width),
                           depth.ctypes.data, None if color is None else color.ctypes.data)
    assert rc == 0, "orc_project: out of memory"
    return depth if c is None else (depth, color)
