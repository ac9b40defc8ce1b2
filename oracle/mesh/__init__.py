"""ctypes front-end of the CPU oracle of VoxelBlockGrid::ExtractTriangleMesh (mesh_oracle.c).

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle``: importable from tests/ and profiles/, never from
``open3d_b200``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libmesh_oracle.so")
_lib = None


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its sources."""
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "mesh_oracle.c"), os.path.join(_HERE, "..", "extract", "extract_oracle.c")]
        if not os.path.exists(_LIB_PATH) or max(map(os.path.getmtime, srcs)) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-B", "-C", _HERE, "libmesh_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        _lib = C.CDLL(_LIB_PATH)
        vp = C.c_void_p
        _lib.orc_extract_triangle_mesh.restype = C.c_int64
        _lib.orc_extract_triangle_mesh.argtypes = [vp, C.c_int64, vp, vp, vp, C.c_int, C.c_float, C.c_float, C.c_int64,
                                                   C.c_int64, vp, vp, vp, vp, C.POINTER(C.c_int64)]
        _lib.orc_mc_table_row.restype = C.c_int
        _lib.orc_mc_table_row.argtypes = [C.c_int, vp, C.POINTER(C.c_int32)]
    return _lib


def table_row(c):
    """Case c of the oracle's generated table -> ([T, 3] int edge triples before the reversal, edge mask)."""
    tri = np.zeros(15, np.int32)
    mask = C.c_int32(0)
    n = lib().orc_mc_table_row(int(c), tri.ctypes.data, C.byref(mask))
    return tri[: 3 * n].reshape(n, 3), int(mask.value)


def extract_triangle_mesh(table_keys, size, tsdf, weight, color_buf=None, resolution=16, voxel_size=0.008,
                          weight_threshold=3.0) -> dict:
    """VoxelBlockGrid::ExtractTriangleMesh on host buffers (slots 0..size-1) -> {"positions", "normals"
    [, "colors"]: [N, 3] f32, "indices": [T, 3] int32}, in orc_extract_triangle_mesh's order."""
    keys = np.ascontiguousarray(table_keys, np.int32).reshape(-1, 3)
    tsdf = np.ascontiguousarray(tsdf, np.float32)
    weight = np.ascontiguousarray(weight, np.uint16)
    col = None if color_buf is None else np.ascontiguousarray(color_buf, np.uint16)
    args = (keys.ctypes.data, int(size), tsdf.ctypes.data, weight.ctypes.data, None if col is None else col.ctypes.data,
            int(resolution), float(voxel_size), float(weight_threshold))
    nt = C.c_int64(0)
    nv = lib().orc_extract_triangle_mesh(*args, 0, 0, None, None, None, None, C.byref(nt))
    out = {"positions": np.zeros((nv, 3), np.float32), "normals": np.zeros((nv, 3), np.float32)}
    if col is not None:
        out["colors"] = np.zeros((nv, 3), np.float32)
    out["indices"] = np.zeros((nt.value, 3), np.int32)
    lib().orc_extract_triangle_mesh(*args, nv, nt.value, out["positions"].ctypes.data, out["normals"].ctypes.data,
                                    out["colors"].ctypes.data if col is not None else None,
                                    out["indices"].ctypes.data, C.byref(nt))
    return out
