"""ctypes front-end of the CPU oracle of PointCloud::EstimateNormals and the OrientNormals* calls (normals_oracle.c).

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
_LIB_PATH = os.path.join(_HERE, "libnormals_oracle.so")
_lib = None

_vp = C.c_void_p


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "normals_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-B", "-C", _HERE, "libnormals_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        for name, args in (("orc_covariance_point_f32", [_vp, _vp, C.c_int, _vp]),
                           ("orc_normal_from_covariance_f32", [_vp, _vp]),
                           ("orc_normals_from_covariances_f32", [_vp, C.c_int64, C.c_int, _vp]),
                           ("orc_estimate_normals_f32", [_vp, C.c_int64, _vp, C.c_int, _vp, C.c_int, _vp, _vp]),
                           ("orc_orient_normals_to_align_with_direction_f32", [_vp, C.c_int64, _vp]),
                           ("orc_orient_normals_towards_camera_location_f32", [_vp, _vp, C.c_int64, _vp])):
            getattr(L, name).restype = None
            getattr(L, name).argtypes = args
        _lib = L
    return _lib


def _f32(a, cols):
    return np.ascontiguousarray(a, np.float32).reshape(-1, cols)


def estimate_normals(points, radius, max_nn=30, prior_normals=None):
    """PointCloud::EstimateNormals(max_nn, radius) -> (normals [n,3], covariances [n,9], neighbour counts [n]).
    prior_normals: the cloud's existing normals, which orient the result as upstream does when the cloud has
    normals."""
    p = _f32(points, 3)
    n = p.shape[0]
    nrm = _f32(prior_normals, 3).copy() if prior_normals is not None else np.zeros((n, 3), np.float32)
    cov = np.zeros((n, 9), np.float32)
    if n == 0:
        return nrm, cov, np.zeros(0, np.int32)
    idx, _, cnt = oracle.hybrid_search(p, p, radius, int(max_nn))
    lib().orc_estimate_normals_f32(p.ctypes.data, n, idx.ctypes.data, int(max_nn), cnt.ctypes.data,
                                   int(prior_normals is not None), nrm.ctypes.data, cov.ctypes.data)
    return nrm, cov, cnt


def covariance_point(points, indices, count) -> np.ndarray:
    """EstimatePointWiseRobustNormalizedCovarianceKernel<float> over the first `count` of `indices` -> [9]."""
    p = _f32(points, 3)
    idx = np.ascontiguousarray(indices, np.int32).reshape(-1)
    out = np.zeros(9, np.float32)
    lib().orc_covariance_point_f32(p.ctypes.data, idx.ctypes.data, int(count), out.ctypes.data)
    return out


def normals_from_covariances(covariances, prior_normals=None) -> np.ndarray:
    """EstimateNormalsFromCovariances<float> on [n,9] covariances, oriented against prior_normals when given."""
    c = _f32(covariances, 9)
    out = _f32(prior_normals, 3).copy() if prior_normals is not None else np.zeros((c.shape[0], 3), np.float32)
    lib().orc_normals_from_covariances_f32(c.ctypes.data, c.shape[0], int(prior_normals is not None), out.ctypes.data)
    return out


def normal_from_covariance(covariance) -> np.ndarray:
    """EstimatePointWiseNormalsWithFastEigen3x3<float> alone, before any orientation -> [3]."""
    c = _f32(covariance, 9)
    out = np.zeros(3, np.float32)
    lib().orc_normal_from_covariance_f32(c.ctypes.data, out.ctypes.data)
    return out


def orient_normals_to_align_with_direction(normals, direction=(0.0, 0.0, 1.0)) -> np.ndarray:
    out = _f32(normals, 3).copy()
    d = np.ascontiguousarray(direction, np.float32).reshape(3)
    lib().orc_orient_normals_to_align_with_direction_f32(out.ctypes.data, out.shape[0], d.ctypes.data)
    return out


def orient_normals_towards_camera_location(points, normals, camera=(0.0, 0.0, 0.0)) -> np.ndarray:
    p = _f32(points, 3)
    out = _f32(normals, 3).copy()
    c = np.ascontiguousarray(camera, np.float32).reshape(3)
    lib().orc_orient_normals_towards_camera_location_f32(p.ctypes.data, out.ctypes.data, out.shape[0], c.ctypes.data)
    return out
