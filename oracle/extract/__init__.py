"""ctypes front-end of the CPU oracle of VoxelBlockGrid::ExtractPointCloud (extract_oracle.c).

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle``: importable from tests/ and profiles/, never from
``open3d_b200``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libextract_oracle.so")
_lib = None


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "extract_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-B", "-C", _HERE, "libextract_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_extract_point_cloud.restype = C.c_int64
        _lib.orc_extract_point_cloud.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                                 C.c_float, C.c_float, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]
    return _lib


def extract_point_cloud(table_keys, size, tsdf, weight, color_buf=None, resolution=16, voxel_size=0.008,
                        weight_threshold=3.0) -> dict:
    """VoxelBlockGrid::ExtractPointCloud on host buffers (slots 0..size-1) -> {"positions", "normals"
    [, "colors"]: [N, 3] f32}, rows in orc_extract_point_cloud's order: slot, linear voxel index, axis."""
    keys = np.ascontiguousarray(table_keys, np.int32).reshape(-1, 3)
    tsdf = np.ascontiguousarray(tsdf, np.float32)
    weight = np.ascontiguousarray(weight, np.uint16)
    col = None if color_buf is None else np.ascontiguousarray(color_buf, np.uint16)
    args = (keys.ctypes.data, int(size), tsdf.ctypes.data, weight.ctypes.data, None if col is None else col.ctypes.data,
            int(resolution), float(voxel_size), float(weight_threshold))
    n = lib().orc_extract_point_cloud(*args, 0, None, None, None)
    out = {"positions": np.zeros((n, 3), np.float32), "normals": np.zeros((n, 3), np.float32)}
    if col is not None:
        out["colors"] = np.zeros((n, 3), np.float32)
    lib().orc_extract_point_cloud(*args, n, out["positions"].ctypes.data, out["normals"].ctypes.data,
                                  out["colors"].ctypes.data if col is not None else None)
    return out
