"""ctypes front-end of the CPU oracle of the exact k-nearest-neighbour search, PointCloud::RemoveStatisticalOutliers
and PointCloud::ComputeMetrics (knn_oracle.c).

TEST INFRASTRUCTURE ONLY, like the rest of ``oracle``: importable from tests/ and profiles/, never from
``open3d_b200``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libknn_oracle.so")
_lib = None

_vp = C.c_void_p

CHAMFER, HAUSDORFF, FSCORE = 0, 1, 2


def lib() -> C.CDLL:
    """The oracle library, compiled with the committed Makefile if missing or older than its source."""
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "knn_oracle.c")
        if not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
            subprocess.run(["make", "-B", "-C", _HERE, "libknn_oracle.so"], check=True,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        L = C.CDLL(_LIB_PATH)
        for name, res, args in (
                ("orc_knn_f32", None, [_vp, C.c_int64, _vp, C.c_int64, C.c_int, _vp, _vp]),
                ("orc_fixed_order_sum", C.c_double, [_vp, C.c_int64]),
                ("orc_statistical_outliers_f32", None, [_vp, C.c_int64, C.c_int, C.c_double, _vp, _vp, _vp]),
                ("orc_metrics_f32", None, [_vp, C.c_int64, _vp, C.c_int64, _vp, C.c_int, _vp, C.c_int, _vp])):
            getattr(L, name).restype = res
            getattr(L, name).argtypes = args
        _lib = L
    return _lib


def _f32(a, cols):
    return np.ascontiguousarray(a, np.float32).reshape(-1, cols)


def knn(points, queries, k):
    """-> (idx [N, k'] int32, dist2 [N, k'] f32), k' = min(k, M): brute force, ascending by (dist^2, index)."""
    p, q = _f32(points, 3), _f32(queries, 3)
    kp = min(int(k), p.shape[0])
    idx = np.empty((q.shape[0], kp), np.int32)
    d2 = np.empty((q.shape[0], kp), np.float32)
    lib().orc_knn_f32(p.ctypes.data, p.shape[0], q.ctypes.data, q.shape[0], int(k), idx.ctypes.data, d2.ctypes.data)
    return idx, d2


def fixed_order_sum(values) -> float:
    v = np.ascontiguousarray(values, np.float64).reshape(-1)
    return float(lib().orc_fixed_order_sum(v.ctypes.data, v.shape[0]))


def statistical_outliers_from_dist2(d2, std_ratio):
    """-> (avg [n] f32, mask [n] bool, (cloud_mean, std, thr)) from the [n, k'] neighbour dist^2."""
    d2 = np.ascontiguousarray(d2, np.float32)
    n, kp = d2.shape
    avg = np.empty(n, np.float32)
    mask = np.empty(n, np.uint8)
    stats = np.zeros(3)
    lib().orc_statistical_outliers_f32(d2.ctypes.data, n, kp, float(std_ratio), avg.ctypes.data, mask.ctypes.data,
                                       stats.ctypes.data)
    return avg, mask.astype(bool), tuple(stats)


def remove_statistical_outliers(points, nb_neighbors, std_ratio):
    """PointCloud::RemoveStatisticalOutliers(nb_neighbors, std_ratio) -> (avg, mask, (cloud_mean, std, thr))."""
    p = _f32(points, 3)
    _, d2 = knn(p, p, nb_neighbors)
    return statistical_outliers_from_dist2(d2, std_ratio)


def compute_metrics(points1, points2, metrics, fscore_radius=(0.01,)):
    """PointCloud::ComputeMetrics -> [values] f32 in the order of `metrics` (FScore: one value per radius)."""
    p1, p2 = _f32(points1, 3), _f32(points2, 3)
    _, d12 = knn(p2, p1, 1)
    _, d21 = knn(p1, p2, 1)
    m = np.ascontiguousarray(metrics, np.int32)
    r = np.ascontiguousarray(fscore_radius, np.float32)
    out = np.zeros(sum(len(r) if x == FSCORE else 1 for x in m), np.float32)
    lib().orc_metrics_f32(d12.ctypes.data, d12.shape[0], d21.ctypes.data, d21.shape[0], m.ctypes.data, len(m),
                          r.ctypes.data, len(r), out.ctypes.data)
    return out
